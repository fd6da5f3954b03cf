"""Host-side checks (no GPU) of the feature transforms for every build_transform configuration: the fp64 oracle
(tests/features_batch_oracle.py) against torchaudio and against the reference's own per-utterance transform
(tests/golden/features_tiny.npz); the modules' tables, buffer names and module order; the per-utterance SpecAugment
span draws; the argument checks of the new C entry points."""
import os
import random

import numpy as np
import pytest
import torch

from tests import features_batch_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "features_tiny.npz")
GEOMS = [(512, 1, True), (400, 3, True), (512, 3, False)]
CONFIGS = [(ft, delta) + g for ft in ("logfbank", "mfcc", "melspec") for delta in (False, True) for g in GEOMS]


def golden():
    return np.load(GOLDEN)


def tag(ft, delta, n_fft, ds, ptd):
    return "%s.d%d.n%d.ds%d.p%d" % (ft, int(delta), n_fft, ds, int(ptd))


def oracle_batch(z, ft, delta, n_fft, ds, ptd):
    return O.batch_transform(z["x"].astype(np.float64), z["lens"], ft, int(z["size"]), n_fft=n_fft,
                             win_length=int(z["win"]), hop_length=int(z["hop"]), delta=delta, downsample=ds,
                             pad_to_divisible=ptd)


def melspec_bar(x, lens, n_fft, win, hop, delta, ds, C, ptd):
    """Per-element bar of the melspec rows: the frame's total power (over the +-4 frames a delta reads), laid out as
    the collated output."""
    rows = []
    for b, n in enumerate(lens):
        p = O.frame_power(x[b:b + 1, :n], n_fft, win, hop)[0]
        Fb = len(p)
        if delta:
            idx = np.clip(np.arange(Fb)[:, None] + np.arange(-4, 5)[None, :], 0, Fb - 1)
            pd = p[idx].max(axis=1)
            per = np.concatenate([np.repeat(p[None], C, 0), np.repeat(pd[None], 2 * C, 0)], axis=0)   # [3C, F]
        else:
            per = np.repeat(p[None], C, 0)
        per = per[None]
        if ds > 1:
            per = O.F.downsample(per, ds, ptd)
        rows.append(per[0].T)
    return O.seq_collate(rows)[0]


@pytest.mark.parametrize("ft,delta,n_fft,ds,ptd", CONFIGS)
def test_oracle_matches_the_reference_transform(ft, delta, n_fft, ds, ptd):
    z = golden()
    k = tag(ft, delta, n_fft, ds, ptd)
    want, want_len = z[k + ".xs"], z[k + ".xlen"]
    got, xlen = oracle_batch(z, ft, delta, n_fft, ds, ptd)
    assert got.shape == want.shape and np.array_equal(xlen, want_len)
    C = int(z["size"])
    assert got.shape[2] == C * (3 if delta else 1) * ds == int(z[k + ".input_size"])
    for b, T in enumerate(xlen):
        assert (want[b, T:] == 0).all() and (got[b, T:] == 0).all()
    if ft == "melspec":
        bar = melspec_bar(z["x"].astype(np.float64), z["lens"], n_fft, int(z["win"]), int(z["hop"]), delta, ds, C, ptd)
        assert (np.abs(got - want) <= 1e-6 * bar + 1e-30).all()
    else:
        assert np.abs(got - want).max() < 2e-4
    if ft == "logfbank" and not delta and ds == 1:
        assert (want[1, 14] == 0).all() and (got[1, 14] == 0).all()     # L_1 % hop == 0: its last frame is masked


def test_oracle_spans_reproduce_the_reference_masks():
    z = golden()
    C = int(z["size"])
    for i in range(2):
        ft, delta, n_fft, ds, ptd, tm, tn, fm, fn = [str(v) for v in z["masked%d.cfg" % i]]
        delta, n_fft, ds, ptd, tm, tn, fm, fn = int(delta), int(n_fft), int(ds), bool(int(ptd)), int(tm), int(tn), \
            int(fm), int(fn)
        clean, xlen = oracle_batch(z, ft, bool(delta), n_fft, ds, ptd)
        random.seed(int(z["mask_seed"]))
        tsp, fsp = O.reference_spans(xlen.tolist(), clean.shape[2], tm, tn, fm, fn)
        got = O.apply_spans(clean, tsp, fsp)
        want = z["masked%d.xs" % i]
        assert np.array_equal(xlen, z["masked%d.xlen" % i])
        assert np.array_equal(got == 0, want == 0)
        assert np.abs(got - want).max() < 2e-4
        assert (want == 0).mean() > (clean == 0).mean()                  # the masks did something
        assert clean.shape[2] == C * (3 if delta else 1) * ds


def test_batch_module_draws_the_reference_spans():
    from edgedict_b200.rnnt.features import draw_utterance_spans
    for T, W, args in [([6, 5, 4], 180, (3, 2, 8, 2)), ([18, 15, 11, 1], 20, (4, 2, 5, 1)), ([7, 9], 240, (0, 2, 5, 3)),
                       ([7, 9], 240, (5, 3, 0, 0)), ([40, 12, 33], 240, (50, 2, 5, 1))]:
        random.seed(7)
        want = O.reference_spans(T, W, *args)
        after = random.random()
        random.seed(7)
        got = draw_utterance_spans(T, W, *args)
        assert [[tuple(s) for s in r] for r in got[0]] == want[0] and [[tuple(s) for s in r] for r in got[1]] == want[1]
        assert random.random() == after                                  # the same number of draws
    with pytest.raises(ValueError):
        draw_utterance_spans([3, 0], 20, 2, 1, 0, 0)                    # randrange(0) as the reference hits it


@pytest.mark.parametrize("n_fft,win,hop", [(400, 400, 200), (512, 400, 200), (512, 320, 160)])
def test_oracle_matches_torchaudio(n_fft, win, hop):
    ta = pytest.importorskip("torchaudio")
    g = torch.Generator().manual_seed(n_fft + win)
    x = torch.randn(2, 3217, generator=g, dtype=torch.float64)
    kw = dict(n_fft=n_fft, win_length=win, hop_length=hop)
    ref = ta.transforms.MelSpectrogram(n_mels=80, **kw).double()(x).numpy()
    got = O.melspec(x.numpy(), 80, **kw)
    assert got.shape == ref.shape == (2, 80, 1 + 3217 // hop)
    # torchaudio builds its filterbank in fp32: the bar is fp32 round-off of the frame's total power
    assert (np.abs(got - ref) <= 1e-6 * O.frame_power(x.numpy(), n_fft, win, hop)[:, None, :]).all()
    ref = ta.transforms.MFCC(n_mfcc=40, log_mels=True, melkwargs=kw).double()(x).numpy()
    got = O.mfcc(x.numpy(), 40, **kw)
    assert got.shape == ref.shape and np.abs(got - ref).max() < 1e-4
    d = ta.functional.compute_deltas(torch.tensor(got))
    assert np.abs(O.compute_deltas(got) - d.numpy()).max() < 1e-9
    assert np.abs(O.cat_deltas(got)[:, 80:] - ta.functional.compute_deltas(d).numpy()).max() < 1e-9
    fb = ta.functional.melscale_fbanks(1 + n_fft // 2, 0.0, 8000.0, 128, 16000, norm=None, mel_scale="htk").numpy()
    mine = O.htk_mel_filterbank(n_fft, 128)
    assert np.abs(mine - fb).max() < 1e-4
    assert np.array_equal(mine.sum(0) == 0, fb.sum(0) == 0)              # the same filters cover no bin
    assert np.abs(O.create_dct(40, 128) - ta.functional.create_dct(40, 128, "ortho").numpy()).max() < 5e-6   # fp32 cos in torchaudio
    assert np.abs(O.hann_periodic(win) - torch.hann_window(win, dtype=torch.float64).numpy()).max() < 1e-15
    with pytest.raises(ValueError):
        O.mfcc(x.numpy(), 129, **kw)


def test_mfcc_n_fft_400_has_all_zero_filters():
    """With n_fft = 400 (the trainers' default) four of the 128 HTK filters cover no FFT bin: their mel power is exactly
    zero and the MFCC sees log(1e-6) there."""
    fb = O.htk_mel_filterbank(400, 128)
    assert (fb.sum(0) == 0).sum() == 4
    x = np.random.default_rng(0).standard_normal((1, 4000))
    assert (O.melspec(x, 128, 400)[:, fb.sum(0) == 0] == 0).all()


def test_module_tables_and_buffer_names():
    from edgedict_b200.rnnt import features as Fm
    m = Fm.MFCC(n_mfcc=40, log_mels=True, melkwargs=dict(n_fft=400, win_length=400, hop_length=200))
    assert list(m.state_dict()) == ["dct_mat", "MelSpectrogram.spectrogram.window", "MelSpectrogram.mel_scale.fb"]
    assert tuple(m.dct_mat.shape) == (128, 40) and tuple(m.MelSpectrogram.mel_scale.fb.shape) == (201, 128)
    # the GEMM operands are read as dense row-major tables
    assert m.dct_mat.is_contiguous() and m.MelSpectrogram.mel_scale.fb.is_contiguous()
    assert m.MelSpectrogram.spectrogram.dft_basis.is_contiguous()
    assert np.abs(m.dct_mat.numpy() - O.create_dct(40, 128)).max() < 1e-6
    assert np.abs(m.MelSpectrogram.mel_scale.fb.numpy() - O.htk_mel_filterbank(400, 128)).max() < 1e-4
    assert (m.MelSpectrogram.mel_scale.fb.sum(0) == 0).sum() == 4
    s = Fm.MelSpectrogram(n_mels=80, n_fft=512, win_length=400, hop_length=200)
    assert list(s.state_dict()) == ["spectrogram.window", "mel_scale.fb"]
    assert np.abs(s.spectrogram.window.numpy() - O.hann_periodic(400)).max() < 1e-6
    # the DFT basis is the periodic window centred in n_fft: frame @ basis == rfft(frame * window)
    frame = np.random.default_rng(1).standard_normal(512)
    w = np.zeros(512)
    w[56:456] = O.hann_periodic(400)
    spec = np.fft.rfft(frame * w)
    got = frame @ s.spectrogram.dft_basis.numpy().astype(np.float64)
    assert np.abs(got[:257] - spec.real).max() < 1e-4 and np.abs(got[257:] - spec.imag).max() < 1e-4
    ta = pytest.importorskip("torchaudio")
    ref = ta.transforms.MFCC(n_mfcc=40, log_mels=True, melkwargs=dict(n_fft=400, win_length=400, hop_length=200))
    assert list(ref.state_dict()) == list(m.state_dict())
    for k, v in ref.state_dict().items():
        assert v.shape == m.state_dict()[k].shape and (v - m.state_dict()[k]).abs().max() < 5e-6, k
    assert torch.equal(ref.state_dict()["MelSpectrogram.mel_scale.fb"], m.MelSpectrogram.mel_scale.fb)


def test_modules_refuse_what_they_do_not_implement():
    from edgedict_b200.rnnt import features as Fm
    with pytest.raises(ValueError):
        Fm.MFCC(n_mfcc=129, log_mels=True, melkwargs=dict(n_fft=400))
    with pytest.raises(NotImplementedError):
        Fm.MFCC(n_mfcc=40)                                              # log_mels=False: amplitude_to_DB is not built
    with pytest.raises(NotImplementedError):
        Fm.build_transform("spectrogram", 40)
    with pytest.raises(NotImplementedError):
        Fm.build_batch_transform("fbank", 40)
    for m in (Fm.MFCC(n_mfcc=20, log_mels=True), Fm.MelSpectrogram(n_mels=20), Fm.CatDeltas()):
        with pytest.raises(RuntimeError, match="CUDA"):
            m(torch.randn(1, 4000) if not isinstance(m, Fm.CatDeltas) else torch.randn(1, 20, 30))
    train, test, _ = Fm.build_batch_transform("mfcc", 20, dither=0)
    with pytest.raises(RuntimeError, match="CUDA"):
        test(torch.randn(2, 4000), torch.tensor([4000, 3000]))


@pytest.mark.parametrize("ft", ["logfbank", "mfcc", "melspec"])
def test_build_transform_module_order_and_input_size(ft):
    from edgedict_b200.rnnt import features as Fm
    first = {"logfbank": "FilterbankFeatures", "mfcc": "MFCC", "melspec": "MelSpectrogram"}[ft]
    for delta in (False, True):
        for ds in (1, 2, 3):
            for tm, fm in ((0, 0), (10, 0), (0, 5), (10, 5)):
                train, test, size = Fm.build_transform(ft, 40, delta=delta, downsample=ds, T_mask=tm, T_num_mask=2,
                                                       F_mask=fm, F_num_mask=1)
                want = [first] + (["CatDeltas"] if delta else []) + (["Downsample"] if ds > 1 else [])
                assert [type(m).__name__ for m in test] == want
                assert [type(m).__name__ for m in train] == want + (["TimeMasking"] if tm else []) + \
                    (["FrequencyMasking"] if fm else [])
                assert size == 40 * (3 if delta else 1) * ds
                btrain, btest, bsize = Fm.build_batch_transform(ft, 40, delta=delta, downsample=ds, T_mask=tm,
                                                                T_num_mask=2, F_mask=fm, F_num_mask=1)
                assert bsize == size == btest.input_size == btrain.input_size
                assert btrain.features is btest.features and type(btest.features).__name__ == first
    m = Fm.build_transform("mfcc", 80, n_fft=400)[1][0]
    assert m.n_mfcc == 80 and m.MelSpectrogram.n_mels == 128 and m.MelSpectrogram.hop_length == 200
    assert Fm.build_transform("melspec", 64, n_fft=400)[1][0].mel_scale.fb.shape == (201, 64)
    assert Fm.build_batch_transform("logfbank", 80, dither=0)[1].features.dither == 0


def test_new_entry_points_reject_bad_arguments_before_touching_the_device():
    """Status 2 (invalid value) before any CUDA call: null pointers, lengths outside (n_fft//2, L], shapes that do not
    hold every utterance's frames."""
    import ctypes
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    L = lib()
    p = 1 << 20
    lens = lambda *v: (ctypes.c_int * len(v))(*v)
    ok = lens(4000, 3000)
    assert L.eb_fe_preemph_pad_lens(None, ok, p, p, 2, 4000, 4400, 256, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad_lens(p, None, p, p, 2, 4000, 4400, 256, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad_lens(p, ok, None, p, 2, 4000, 4400, 256, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad_lens(p, ok, p, None, 2, 4000, 4400, 256, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad_lens(p, lens(4000, 256), p, p, 2, 4000, 4600, 256, 0.97, 1, None) == 2   # L_b <= pad
    assert L.eb_fe_preemph_pad_lens(p, lens(4001, 300), p, p, 2, 4000, 4600, 256, 0.97, 1, None) == 2   # L_b > L
    assert L.eb_fe_preemph_pad_lens(p, lens(4000, 0), p, p, 2, 4000, 4600, 256, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad_lens(p, ok, p, p, 2, 4000, 4400, 256, 0.97, 1, None) == 2   # Lp < L + 2*pad
    assert L.eb_fe_preemph_pad_lens(p, ok, p, p, 0, 4000, 4600, 256, 0.97, 1, None) == 2   # B <= 0
    assert L.eb_fe_log(None, 8, 1e-6, None) == 2
    assert L.eb_fe_log(p, -8, 1e-6, None) == 2
    assert L.eb_fe_log(p, 8, 0.0, None) == 2
    # eb_fe_finish: 4000 samples at hop 200 -> 21 frames, 7 rows at n_stack 3
    args = dict(feat=p, out=p, lens=ok, dev=p, B=2, R=23, hop=200, C=40, n=3, T=7, log=1, mask=1, delta=1, ptd=1)

    def fin(**change):
        a = dict(args, **change)
        return L.eb_fe_finish(a["feat"], a["out"], a["lens"], a["dev"], a["B"], a["R"], a["hop"], a["C"], a["n"],
                              a["T"], a["log"], a["mask"], a["delta"], a["ptd"], None)
    for change in [dict(feat=None), dict(out=None), dict(lens=None), dict(dev=None), dict(B=0), dict(R=0), dict(hop=0),
                   dict(C=0), dict(n=0), dict(T=0), dict(R=20), dict(T=6), dict(lens=lens(4000, 0)),
                   dict(lens=lens(4000, -5))]:
        assert fin(**change) == 2, change
    assert L.eb_fe_deltas(None, p, 2, 10, 40, None) == 2
    assert L.eb_fe_deltas(p, None, 2, 10, 40, None) == 2
    assert L.eb_fe_deltas(p, p, 0, 10, 40, None) == 2
    assert L.eb_fe_deltas(p, p, 2, 0, 40, None) == 2
    assert L.eb_fe_deltas(p, p, 2, 10, 0, None) == 2


def test_ops_refuse_bad_lengths_on_the_host():
    from edgedict_b200 import ops
    from edgedict_b200.rnnt import features as Fm
    with pytest.raises(RuntimeError, match="CUDA"):
        Fm.build_batch_transform("melspec", 20)[1](torch.zeros(2, 1000), [1000, 300])
    F, T = ops.fe_lengths([4000, 3999, 257], 200, 3, True)
    assert F == [21, 20, 2] and T == [7, 7, 1]
    assert ops.fe_lengths([4000, 3999, 257], 200, 3, False)[1] == [7, 6, 0]
