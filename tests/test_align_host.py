"""Forced alignment without a GPU: the fp64 restatements (tests/align_oracle.py) against brute-force enumeration and
torchaudio, every malformed argument refused on the host, and the C entries' argument checks."""
import ctypes

import numpy as np
import pytest
import torch

from tests import align_oracle as ao


def _argmax_set(paths):
    best = max(s for _, s in paths)
    return best, {p for p, s in paths if s == best}


@pytest.mark.parametrize("T, U", [(1, 0), (1, 3), (4, 0), (2, 2), (3, 3), (5, 2), (4, 4), (6, 3)])
@pytest.mark.parametrize("kind", ["random", "two_values", "constant"])
def test_rnnt_restatement_is_the_best_path(T, U, kind):
    rng = np.random.default_rng(T * 100 + U)
    for _ in range(20):
        if kind == "random":
            lpb, lpl = (rng.standard_normal((T, U + 1)).astype(np.float32) - 2 for _ in range(2))
        elif kind == "two_values":
            lpb, lpl = (rng.choice(np.float32([-1.0, -2.0]), (T, U + 1)) for _ in range(2))
        else:
            lpb = lpl = np.full((T, U + 1), -1.5, np.float32)
        frames, logp, score = ao.rnnt_viterbi(lpb, lpl)
        best, winners = _argmax_set(ao.rnnt_all_paths(lpb, lpl))
        assert score == best
        assert tuple(frames) in winners
        assert np.all(np.diff(frames) >= 0) and (U == 0 or (frames.min() >= 0 and frames.max() < T))
        assert np.array_equal(logp, lpl[frames, np.arange(U)])


def test_rnnt_restatement_tie_rule():
    # every path scores the same: each cell reached by stay keeps it, so the backtrace walks back along the last
    # label's row to t = 0, and all labels are emitted at the first frame
    frames, _, _ = ao.rnnt_viterbi(np.zeros((5, 4), np.float32), np.zeros((5, 4), np.float32))
    assert frames.tolist() == [0, 0, 0]
    frames, _, score = ao.rnnt_viterbi(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32))
    assert frames.tolist() == [-1, -1] and score == -np.inf


@pytest.mark.parametrize("T, labels", [(1, []), (3, []), (1, [1]), (2, [1]), (3, [1, 2]), (4, [1, 1]), (3, [1, 1]),
                                       (2, [1, 1]), (5, [2, 1, 2]), (6, [1, 2, 2]), (6, [3, 3, 3])])
@pytest.mark.parametrize("kind", ["random", "two_values", "constant"])
def test_ctc_restatement_is_the_best_path(T, labels, kind):
    rng = np.random.default_rng(T * 10 + len(labels))
    V = 4
    for _ in range(20):
        if kind == "random":
            lp = rng.standard_normal((T, V)).astype(np.float32)
        elif kind == "two_values":
            lp = rng.choice(np.float32([-1.0, -2.0]), (T, V))
        else:
            lp = np.full((T, V), -1.0, np.float32)
        align, logp, score = ao.ctc_viterbi(lp, labels, 0)
        paths = ao.ctc_all_paths(lp, labels, 0)
        if not paths:
            assert score == -np.inf and align.tolist() == [-1] * T and np.all(logp == -np.inf)
            continue
        best, winners = _argmax_set(paths)
        assert score == best
        assert tuple(align) in winners
        assert np.array_equal(logp, lp[np.arange(T), align])


def test_ctc_restatement_tie_rules():
    lp = np.full((4, 3), -1.0, np.float32)
    # every path scores the same: the last label beats the equal final blank, and walking back each state keeps
    # itself while it can, so the path reaches its labels as early as the lattice allows
    assert ao.ctc_viterbi(lp, [1], 0)[0].tolist() == [1, 1, 1, 1]
    assert ao.ctc_viterbi(lp, [1, 2], 0)[0].tolist() == [1, 2, 2, 2]
    assert ao.ctc_viterbi(lp, [1, 1], 0)[0].tolist() == [1, 0, 1, 1]
    assert ao.ctc_viterbi(lp, [], 0)[0].tolist() == [0, 0, 0, 0]
    assert ao.ctc_viterbi(lp[:2], [1, 1], 0)[1].tolist() == [-np.inf, -np.inf]      # too short for the repeat
    assert ao.ctc_viterbi(lp, [5], 0)[0].tolist() == [-1] * 4                       # label outside [0, V)
    a, s, score = ao.ctc_viterbi(lp[:0], [], 0)
    assert a.size == 0 and score == 0.0


def test_ctc_restatement_matches_torchaudio_on_continuous_inputs():
    F = pytest.importorskip("torchaudio.functional")
    if not hasattr(F, "forced_align"):
        pytest.skip("torchaudio without forced_align")
    rng = np.random.default_rng(7)
    for i in range(150):
        T, V = int(rng.integers(1, 60)), int(rng.integers(3, 12))
        S = int(rng.integers(1, max(2, T // 2)))                      # torchaudio refuses empty targets
        labels = rng.integers(1, V, S)
        if i % 3 == 0 and S >= 2:
            labels[1] = labels[0]                                     # a repeat
        lp = torch.from_numpy(rng.standard_normal((T, V)).astype(np.float32)).log_softmax(-1)
        align, logp, _ = ao.ctc_viterbi(lp.numpy(), labels, 0)
        if align[0] < 0:
            continue
        ta, ts = F.forced_align(lp[None], torch.from_numpy(labels)[None].to(torch.int32), blank=0)
        assert ta[0].tolist() == align.tolist(), i
        assert np.array_equal(ts[0].numpy(), logp), i


# ---- host-side refusals ----------------------------------------------------------------------------------------------
def _ctc_args(**kw):
    B, T, V, S = 2, 6, 5, 3
    a = dict(log_probs=torch.randn(B, T, V).log_softmax(-1), targets=torch.randint(1, V, (B, S)),
             input_lengths=[T, T - 1], target_lengths=[S, 2], blank=0)
    a.update(kw)
    return a


@pytest.mark.parametrize("bad, exc", [
    (dict(log_probs=torch.randn(2, 6, 5, dtype=torch.float64)), TypeError),
    (dict(log_probs=[[0.0]]), TypeError),
    (dict(targets=torch.ones(2, 3)), TypeError),
    (dict(log_probs=torch.randn(6, 5)), ValueError),                     # batch first [B, T, V] only
    (dict(log_probs=torch.randn(0, 6, 5)), ValueError),
    (dict(targets=torch.ones(2, 3, 1, dtype=torch.long)), ValueError),
    (dict(targets=torch.ones(3, 3, dtype=torch.long)), ValueError),
    (dict(target_lengths=[4, 2]), ValueError),
    (dict(target_lengths=[-1, 2]), ValueError),
    (dict(target_lengths=[3]), ValueError),
    (dict(target_lengths=torch.tensor([3.0, 2.0])), TypeError),
    (dict(input_lengths=[7, 6]), ValueError),
    (dict(input_lengths=[6, -1]), ValueError),
    (dict(targets=torch.ones(6, dtype=torch.long)), ValueError),
    (dict(blank=5), ValueError),
    (dict(blank=-1), ValueError),
    (dict(log_probs=torch.randn(1, 1100, 5), targets=torch.ones(1, 1024, dtype=torch.long), input_lengths=[1100],
          target_lengths=[1024]), ValueError),
    (dict(), RuntimeError),                                              # valid, but CPU tensors: no CPU path
])
def test_ctc_forced_align_refuses_bad_arguments_on_the_host(bad, exc):
    from edgedict_b200.ctc import forced_align
    with pytest.raises(exc):
        forced_align(**_ctc_args(**bad))


def _rnnt_args(**kw):
    a = dict(acts=torch.randn(2, 5, 4, 6), labels=torch.ones(2, 3, dtype=torch.int32),
             act_lens=torch.tensor([5, 4], dtype=torch.int32), label_lens=torch.tensor([3, 1], dtype=torch.int32))
    a.update(kw)
    return a


@pytest.mark.parametrize("bad, exc", [
    (dict(labels=torch.ones(2, 3, dtype=torch.int64)), TypeError),
    (dict(act_lens=torch.tensor([5, 4])), TypeError),
    (dict(acts=torch.randn(2, 6, 5, 4).transpose(1, 2)), ValueError),   # not contiguous
    (dict(act_lens=torch.tensor([5], dtype=torch.int32)), ValueError),
    (dict(acts=torch.randn(2, 5, 4)), ValueError),
    (dict(act_lens=torch.tensor([4, 4], dtype=torch.int32)), ValueError),   # T != max length
    (dict(label_lens=torch.tensor([2, 1], dtype=torch.int32)), ValueError),  # U != max label length + 1
    (dict(), RuntimeError),
    (dict(acts=torch.randn(2, 5, 4, 6).half()), RuntimeError),          # CPU is refused before the dtype
])
def test_rnnt_forced_align_refuses_bad_arguments_on_the_host(bad, exc):
    from edgedict_b200.align import rnnt_forced_align
    with pytest.raises(exc):
        rnnt_forced_align(**_rnnt_args(**bad))


def test_model_align_refuses_bad_lengths_before_the_device():
    from edgedict_b200.rnnt.models import CTCEncoder
    m = CTCEncoder(vocab_size=8, input_size=4, enc_hidden_size=8, enc_layers=1, enc_dropout=0, proj_size=8)
    from edgedict_b200.rnnt import models
    with pytest.raises(ValueError):
        models._ctc_frames(10, [20, 30, 40], 2)
    assert models._ctc_frames(10, [20, 10], 2).tolist() == [10, 5]
    assert hasattr(m, "align") and hasattr(models.Transducer, "align")


# ---- C entries ---------------------------------------------------------------------------------------------------
def test_align_entry_points_refuse_bad_arguments_before_touching_the_device():
    from edgedict_b200._lib import lib
    L = lib()
    fake = ctypes.c_void_p(256)          # never dereferenced: every call below must return before any launch
    assert L.eb_rnnt_align_bytes(2, 10, 1025) == 0
    assert L.eb_rnnt_align_bytes(0, 10, 3) == 0
    assert L.eb_rnnt_align_bytes(2, 100, 129) == 0                       # decisions fit in shared memory
    assert L.eb_rnnt_align_bytes(2, 1000, 1024) == 2 * 1000 * 1024
    # the whole 227 KB opt-in shared memory holds delta, frames, (t, u) and the decisions: the kernel has no static part
    assert L.eb_rnnt_align_bytes(2, 1777, 129) == 0
    assert L.eb_rnnt_align_bytes(2, 1778, 129) == 2 * 1778 * 129

    def vit(**kw):
        a = dict(xl=fake, yl=fake, B=2, T=10, U=4, ds=4, ws=fake, dec=None, fr=fake, lp=fake, sc=fake)
        a.update(kw)
        return L.eb_rnnt_viterbi(a["xl"], a["yl"], a["B"], a["T"], a["U"], a["ds"], a["ws"], a["dec"], a["fr"],
                                 a["lp"], a["sc"], None)

    for kw in (dict(U=1025), dict(U=0), dict(T=0), dict(B=0), dict(ds=2), dict(xl=None), dict(yl=None),
               dict(ws=None), dict(fr=None), dict(lp=None), dict(sc=None),
               dict(T=1000, U=1024)):                                    # decisions do not fit: a buffer is needed
        assert vit(**kw) == 2, kw

    assert L.eb_ctc_align_workspace_size(2, 10, 1024) == 0
    assert L.eb_ctc_align_workspace_size(0, 10, 3) == 0
    assert L.eb_ctc_align_workspace_size(2, 10, 3) == 0                  # back-pointers fit in shared memory
    assert L.eb_ctc_align_workspace_size(2, 2000, 1023) == 2 * 2000 * 2047
    # states, labels, four control ints and the back-pointers in 227 KB, with no static shared memory beside them
    assert L.eb_ctc_align_workspace_size(2, 499, 223) == 0
    assert L.eb_ctc_align_workspace_size(2, 500, 223) == 2 * 500 * 447
    assert L.eb_ctc_align_workspace_size(2, 1148, 99) == 0               # exactly 227 KB
    assert L.eb_ctc_align_workspace_size(2, 1149, 99) == 2 * 1149 * 199

    def ali(**kw):
        a = dict(lp=fake, sb=50, st=5, B=2, T=10, V=5, targets=fake, nt=6, off=fake, tl=fake, il=fake, S=3, blank=0,
                 ws=None, al=fake, fl=fake)
        a.update(kw)
        return L.eb_ctc_align(a["lp"], a["sb"], a["st"], a["B"], a["T"], a["V"], a["targets"], a["nt"], a["off"],
                              a["tl"], a["il"], a["S"], a["blank"], a["ws"], a["al"], a["fl"], None)

    for kw in (dict(S=1024), dict(S=-1), dict(blank=5), dict(blank=-1), dict(B=0), dict(B=70000), dict(T=-1),
               dict(V=0), dict(lp=None), dict(off=None), dict(tl=None), dict(il=None), dict(al=None), dict(fl=None),
               dict(targets=None), dict(nt=-1), dict(sb=-1), dict(st=-5),
               dict(T=2000, S=1023)):                                    # back-pointers do not fit: a buffer is needed
        assert ali(**kw) == 2, kw
