"""Per-utterance features of a padded batch (build_batch_transform -> csrc/frontend.cu) for every build_transform
configuration, against the fp64 oracle (tests/features_batch_oracle.py) and the reference's own per-utterance transform
(tests/golden/features_tiny.npz), plus the bitwise invariants of the batched path and two integrations.

Bars: per element, the first-order bound tests/features_fp64.py propagates through the fp64 restatement of the chain
on the module's own fp32 tables, in table mode (plus the effect of those tables' distance from the oracle's exact ones).
Against the reference's own fp32 features (the golden fixture), which carry their own error, the bar grows by
|oracle - golden|, measured per element: |device - golden| <= bar + |oracle - golden| by the triangle inequality.  The
melspec rows also print their ratio to the former bar, 1e-5 x the frame's total power sum_k P."""
import random

import numpy as np
import pytest
import torch

from tests import features_batch_oracle as O
from tests import features_fp64 as X
from tests.test_features_batch_host import CONFIGS, golden, melspec_bar, tag

pytestmark = pytest.mark.gpu


def _build(ft, size, n_fft=512, delta=False, ds=1, ptd=True, **kw):
    from edgedict_b200.rnnt.features import build_batch_transform
    train, test, n = build_batch_transform(ft, size, n_fft=n_fft, win_length=400, hop_length=200, delta=delta,
                                           downsample=ds, pad_to_divisible=ptd, dither=0, **kw)
    return train.cuda(), test.cuda(), n


def _bar(test, ft, x, lens, n_fft, C, delta, ds, ptd):
    """Per-element bar and where it holds (features_fp64.chain in table mode) for the module `test` on fp32 x [B, L]."""
    basis, fbT, dct, pre = X.module_tables(test)
    te = X.tables_err(ft, basis, fbT, dct, n_fft, C, pre)
    _, bar, ok = X.chain(x.cuda(), lens, ft, basis, fbT, n_fft, 200, ds, delta, ptd, preemph=pre, dct=dct, tables_err=te)
    return bar, ok


def _check(ft, got, want, bar, ok, x, lens, n_fft, delta, ds, C, ptd, what, extra=None):
    """Assert the propagated bar; return the worst error as a fraction of it."""
    if ft == "melspec":
        err = np.abs(np.asarray(got, np.float64) - want)
        old = 1e-5 * melspec_bar(x, lens, n_fft, 400, 200, delta, ds, C, ptd)
        print("%s %s worst error / former bar 1e-5 sum_k P = %.3g" % (what, ft, float(np.max(err / np.maximum(old, 1e-30)))))
    return X.report("%s %s d%d n%d ds%d p%d" % (what, ft, delta, n_fft, ds, ptd), got, want, bar, ok, extra)


@pytest.mark.parametrize("ft,delta,n_fft,ds,ptd", CONFIGS)
def test_golden_and_oracle_parity(ft, delta, n_fft, ds, ptd):
    z = golden()
    k = tag(ft, delta, n_fft, ds, ptd)
    C = int(z["size"])
    _, test, n = _build(ft, C, n_fft, delta, ds, ptd)
    x = z["x"]
    xs, xlen = test(torch.tensor(x).cuda(), torch.tensor(z["lens"]))
    xs = xs.cpu().numpy()
    assert xlen.dtype == torch.int32 and xlen.device.type == "cpu"
    assert np.array_equal(xlen.numpy(), z[k + ".xlen"]) and xs.shape == z[k + ".xs"].shape and xs.shape[2] == n
    for b, T in enumerate(xlen.tolist()):
        assert (xs[b, T:] == 0).all()
    bar, ok = _bar(test, ft, torch.tensor(x), z["lens"], n_fft, C, delta, ds, ptd)
    want, _ = O.batch_transform(x.astype(np.float64), z["lens"], ft, C, n_fft=n_fft, win_length=400, hop_length=200,
                                delta=delta, downsample=ds, pad_to_divisible=ptd)
    gold = z[k + ".xs"].astype(np.float64)
    _check(ft, xs, want, bar, ok, x.astype(np.float64), z["lens"], n_fft, delta, ds, C, ptd, "oracle")
    _check(ft, xs, gold, bar, ok, x.astype(np.float64), z["lens"], n_fft, delta, ds, C, ptd, "golden",
           extra=np.abs(want - gold))


def _speech_like(lens, seed):
    g = torch.Generator().manual_seed(seed)
    L = max(lens)
    t = torch.arange(L) / 16000.0
    x = torch.zeros(len(lens), L)
    for b, n in enumerate(lens):
        env = 0.5 + 0.5 * torch.sin(2 * np.pi * 3.0 * t[:n] + b)
        x[b, :n] = 0.05 * torch.randn(n, generator=g) + env * (0.4 * torch.sin(2 * np.pi * (150.0 + 40 * b) * t[:n]) +
                                                               0.1 * torch.sin(2 * np.pi * 2500.0 * t[:n]))
    return x


LONG_LENS = [16000, 256000, 71234, 143999, 200000, 33333, 111111, 255800]       # 1 - 16 s


@pytest.mark.parametrize("ft", ["logfbank", "mfcc", "melspec"])
@pytest.mark.parametrize("delta", [False, True])
def test_long_utterances_against_the_oracle(ft, delta):
    x = _speech_like(LONG_LENS, 3)
    _, test, _ = _build(ft, 80, 512, delta, 3, True)
    xs, xlen = test(x.cuda(), LONG_LENS)
    want, wlen = O.batch_transform(x.numpy().astype(np.float64), LONG_LENS, ft, 80, n_fft=512, win_length=400,
                                   hop_length=200, delta=delta, downsample=3, pad_to_divisible=True)
    assert np.array_equal(xlen.numpy(), wlen)
    bar, ok = _bar(test, ft, x, LONG_LENS, 512, 80, delta, 3, True)
    _check(ft, xs.cpu().numpy(), want, bar, ok, x.numpy().astype(np.float64), LONG_LENS, 512, delta, 3, 80, True,
           "8 x 1-16 s")


def test_masks_reproduce_the_reference_draws():
    z = golden()
    for i in range(2):
        ft, delta, n_fft, ds, ptd, tm, tn, fm, fn = [str(v) for v in z["masked%d.cfg" % i]]
        train, test, _ = _build(ft, int(z["size"]), int(n_fft), bool(int(delta)), int(ds), bool(int(ptd)),
                                T_mask=int(tm), T_num_mask=int(tn), F_mask=int(fm), F_num_mask=int(fn))
        x = torch.tensor(z["x"]).cuda()
        random.seed(int(z["mask_seed"]))
        got, xlen = train(x, torch.tensor(z["lens"]))
        want = z["masked%d.xs" % i]
        clean, _ = test(x, torch.tensor(z["lens"]))
        assert np.array_equal(xlen.numpy(), z["masked%d.xlen" % i])
        g, c = got.cpu().numpy(), clean.cpu().numpy()
        assert np.array_equal(g == 0, want == 0)
        assert ((g == c) | (g == 0)).all()                              # unmasked elements are the test transform's
        # the oracle with the same spans; the golden masked rows carry their own distance from it
        oc, olen = O.batch_transform(z["x"].astype(np.float64), z["lens"], ft, int(z["size"]), n_fft=int(n_fft),
                                     win_length=400, hop_length=200, delta=bool(int(delta)), downsample=int(ds),
                                     pad_to_divisible=bool(int(ptd)))
        random.seed(int(z["mask_seed"]))
        om = O.apply_spans(oc, *O.reference_spans(olen.tolist(), oc.shape[2], int(tm), int(tn), int(fm), int(fn)))
        bar, ok = _bar(test, ft, torch.tensor(z["x"]), z["lens"], int(n_fft), int(z["size"]), bool(int(delta)), int(ds),
                       bool(int(ptd)))
        X.report("masked%d %s vs golden" % (i, ft), g, want, bar, ok, np.abs(om - want))


@pytest.mark.parametrize("ft", ["logfbank", "mfcc", "melspec"])
def test_bitwise_invariants(ft):
    lens = [48000, 30117, 12800, 7201]
    x = _speech_like(lens, 11).cuda()
    _, test_d, _ = _build(ft, 40, 512, True, 3, True)
    _, test_s, _ = _build(ft, 40, 512, False, 3, True)
    train0, test0, _ = _build(ft, 40, 512, True, 3, True, T_mask=0, T_num_mask=2, F_mask=0, F_num_mask=1)
    _, test_f, _ = _build(ft, 40, 512, True, 3, False)
    xd, ld = test_d(x, lens)
    xs, ls = test_s(x, lens)
    xf, lf = test_f(x, lens)
    assert torch.equal(ld, ls)
    for b, n in enumerate(lens):
        T = int(ld[b])
        assert (xd[b, T:] == 0).all() and (xs[b, T:] == 0).all() and (xf[b, int(lf[b]):] == 0).all()
        # utterance b alone: its own length, its own batch of one
        alone, la = test_d(x[b:b + 1, :n].contiguous(), [n])
        assert int(la[0]) == T and torch.equal(alone[0], xd[b, :T])
        # the static channels of each stacked frame are the delta=False output
        d =xd[b].reshape(xd.shape[1], 3, 3, 40)                        # [T, stacked frame, (x, d1, d2), C]
        assert torch.equal(d[:, :, 0], xs[b].reshape(xs.shape[1], 3, 40))
        # pad_to_divisible=False: the leading floor(F_b / 3) rows of the padded output
        Tf = int(lf[b])
        assert Tf <= T and torch.equal(xf[b, :Tf], xd[b, :Tf])
    y0, l0 = train0(x, lens)
    assert torch.equal(y0, xd) and torch.equal(l0, ld)                  # no masks: train is test


def test_logfbank_equal_lengths_is_the_fused_frontend():
    from edgedict_b200.rnnt.features import LogMelFrontend
    x = _speech_like([40000] * 3, 5).cuda()
    for ptd in (True, False):
        _, test, _ = _build("logfbank", 80, 512, False, 3, ptd)
        got, xlen = test(x, [40000] * 3)
        want = LogMelFrontend(80, downsample=3, pad_to_divisible=ptd, dither=0).cuda()(x.clone())
        assert torch.equal(got, want) and (xlen == want.shape[1]).all()


def test_sequential_modules_match_the_batched_path():
    """build_transform's [B, C, T] module sequence (MFCC / MelSpectrogram, CatDeltas, Downsample) on one utterance is
    the batched module's output, transposed."""
    from edgedict_b200.rnnt.features import build_transform
    x = _speech_like([30117], 2).cuda()
    for ft in ("mfcc", "melspec"):
        for ptd in (True, False):
            seq = build_transform(ft, 40, delta=True, downsample=3, pad_to_divisible=ptd)[1].cuda()
            _, test, _ = _build(ft, 40, 512, True, 3, ptd)
            got = seq(x)
            want, _ = test(x, [30117])
            assert torch.equal(got.transpose(1, 2), want)


def test_transducer_loss_and_gradients_from_batched_features():
    """E4D1-sized transducer: loss and every gradient from build_batch_transform's features equal, bitwise, those from
    per-utterance features padded with zero_pad_concat (rnnt/dataset.py:202-211)."""
    from edgedict_b200.rnnt.models import Transducer
    from tests.util import E4D1_CFG
    lens = [64000, 41234, 52000]
    x = _speech_like(lens, 9).cuda()
    _, test, n = _build("mfcc", 40, 512, True, 2, True)
    assert n == E4D1_CFG["input_size"]
    xs, xlen = test(x, lens)
    feats = [test(x[b:b + 1, :L].contiguous(), [L])[0][0] for b, L in enumerate(lens)]
    padded = torch.zeros_like(xs)
    for b, f in enumerate(feats):
        padded[b, :len(f)] = f
    assert torch.equal(padded, xs)
    torch.manual_seed(0)
    m = Transducer(**E4D1_CFG).cuda()
    ys = torch.randint(4, 1024, (3, 20), dtype=torch.int32).cuda()
    ylen = torch.tensor([20, 17, 12], dtype=torch.int32)
    out = []
    for feats_in in (xs, padded):
        m.zero_grad()
        loss = m(feats_in, ys, xlen, ylen)
        loss.backward()
        out.append((loss.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    assert torch.equal(out[0][0], out[1][0]) and torch.isfinite(out[0][0])
    assert all(torch.equal(a, b) for a, b in zip(out[0][1], out[1][1]))


def test_stream_decoder_with_mfcc_delta_transform():
    """PytorchStreamDecoder driven by build_transform('mfcc', 80, delta=True, downsample=3, pad_to_divisible=False)'s
    test transform, chunk by chunk, emits the ids Transducer.greedy_decode finds over the concatenated chunk features."""
    from edgedict_b200.rnnt.features import build_transform
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    _, tf, n = build_transform("mfcc", 80, delta=True, downsample=3, pad_to_divisible=False)
    tf = tf.cuda()
    torch.manual_seed(4)
    m = Transducer(vocab_embed_size=16, vocab_size=32, input_size=n, enc_hidden_size=64, enc_layers=2, enc_dropout=0,
                   enc_proj_size=32, dec_hidden_size=32, dec_layers=1, dec_dropout=0, dec_proj_size=32,
                   joint_size=48).cuda().eval()

    class Tok:
        vocab_size = 32

        class tokenizer:
            @staticmethod
            def id_to_token(i):
                return "t%d</w>" % i

            @staticmethod
            def token_to_id(t):
                return -1                                               # no <unk> rule: greedy_decode has none

    dec = PytorchStreamDecoder(FLAGS=None, transducer=m, transform=tf, tokenizer=Tok())
    x = _speech_like([96000], 8)[0].cuda()
    chunks = [x[i:i + 12000][None] for i in range(0, 96000, 12000)]
    text = "".join(dec.decode(c) for c in chunks)
    feats = torch.cat([tf(c).transpose(1, 2) for c in chunks], dim=1)
    assert feats.shape[2] == n == 720
    ids, _ = m.greedy_decode(feats, torch.tensor([feats.shape[1]]))
    want = "".join("t%d " % int(i) for i in ids[0] if int(i) != 0)
    assert text == want
