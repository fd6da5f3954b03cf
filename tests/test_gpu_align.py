"""Forced alignment on the device (eb_rnnt_viterbi, eb_ctc_align and their Python interfaces).

Teacher-forced and bitwise: the log-probs the kernels read are taken from the workspace (or are the input, for CTC) and
the fp64 restatements of tests/align_oracle.py run on exactly those values; frames, alignments, per-label / per-frame
log-probs and scores must match bit for bit.  Then exact ties, invariants (score against the loss, path sums, batch
independence, repeatability) and the models against the fp64 oracles."""
import numpy as np
import pytest
import torch

from tests import align_oracle as ao

pytestmark = pytest.mark.gpu

f32, f64 = torch.float32, torch.float64


def _np(t):
    return t.detach().cpu().numpy()


def _ws_logprobs(ws, B, T, U, dtype):
    """lpb, lpl [B, T, U] from the loss workspace: its second and third arrays of n = B*T*U values."""
    n = B * T * U
    w = ws.view(dtype)
    return _np(w[n:2 * n].view(B, T, U)), _np(w[2 * n:3 * n].view(B, T, U))


def _path_sum(lpb, lpl, frames):
    """The log-probs of the path `frames` describes, summed in fp64 in path order."""
    T, U1 = lpb.shape
    acc, u = 0.0, 0
    for t in range(T):
        while u < U1 - 1 and frames[u] == t:
            acc += float(lpl[t, u])
            u += 1
        acc += float(lpb[t, u])
    return acc


def _rnnt_problem(B, T, U1, V, dtype, blank, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        acts = torch.randn(B, T, U1, V, generator=g, dtype=f64) * 2
    elif kind == "constant":
        acts = torch.zeros(B, T, U1, V, dtype=f64)
    else:                                                    # two values per row: many exact ties
        acts = torch.randint(0, 2, (B, T, U1, V), generator=g).to(f64)
    labels = torch.randint(0, V - 1, (B, max(U1 - 1, 0)), generator=g, dtype=torch.int32)
    labels += (labels >= blank).to(torch.int32)
    xlen = torch.randint(1, T + 1, (B,), generator=g, dtype=torch.int32)
    ylen = torch.randint(0, U1, (B,), generator=g, dtype=torch.int32)
    xlen[0], ylen[0] = T, U1 - 1
    if B > 2:
        ylen[1] = 0
    return acts.to(dtype).cuda(), labels.cuda(), xlen, ylen


def _check_rnnt(frames, logp, score, lpb, lpl, xlen, ylen, costs=None):
    frames, logp, score = _np(frames), _np(logp), _np(score)
    for b in range(len(xlen)):
        Tb, Ub = int(xlen[b]), int(ylen[b]) + 1
        rf, rl, rs = ao.rnnt_viterbi(lpb[b, :Tb, :Ub], lpl[b, :Tb, :Ub])
        assert np.array_equal(frames[b, :Ub - 1], rf), b
        assert np.array_equal(logp[b, :Ub - 1], rl), b
        assert np.all(frames[b, Ub - 1:] == -1) and np.all(logp[b, Ub - 1:] == 0), b
        assert score[b] == score.dtype.type(rs), (b, score[b], rs)
        assert _path_sum(lpb[b, :Tb, :Ub], lpl[b, :Tb, :Ub], rf) == rs
        if costs is not None:                                # the best path is one of the paths the loss sums
            assert score[b] <= -costs[b] + 1e-5 * abs(costs[b]) + 1e-5, (b, score[b], costs[b])


RNNT_CASES = [
    (1, 1, 1, 5, f32, 0, "random"),
    (3, 17, 5, 11, f32, 0, "random"),
    (40, 60, 9, 16, f32, 0, "random"),
    (5, 40, 7, 13, f32, 12, "random"),                      # blank = V - 1
    (4, 30, 6, 9, f64, 0, "random"),
    (3, 1000, 20, 8, f32, 0, "random"),
    (2, 100, 1024, 4, f32, 0, "random"),                    # a full CTA, decisions in shared memory; the wide lattice
    (2, 300, 1024, 4, f32, 3, "random"),                    # a full CTA, decisions in the caller's buffer
    (1, 1000, 1024, 2, f32, 0, "random"),
    (2, 50, 1024, 3, f64, 0, "random"),
    (2, 1777, 129, 5, f32, 0, "random"),                   # the last T' whose decisions fit in shared memory
    (2, 1778, 129, 5, f32, 0, "random"),                   # one more: staged from the caller's buffer in 4 bands
    (3, 20, 6, 7, f32, 0, "constant"),
    (3, 30, 8, 5, f32, 0, "two_values"),
    (2, 25, 5, 4, f64, 0, "two_values"),
]


@pytest.mark.parametrize("B, T, U1, V, dtype, blank, kind", RNNT_CASES)
def test_rnnt_viterbi_teacher_forced_bitwise(B, T, U1, V, dtype, blank, kind):
    from edgedict_b200 import ops
    from edgedict_b200.align import rnnt_forced_align
    acts, labels, xlen, ylen = _rnnt_problem(B, T, U1, V, dtype, blank, kind, B * 1000 + T + U1)
    xl, yl = xlen.cuda(), ylen.cuda()
    costs, ws = ops.rnnt_loss_fwd(acts, labels, xl, yl, blank, need_beta=False)
    costs = _np(costs)
    out = ops.rnnt_viterbi(xl, yl, B, T, U1, ws, dtype)
    lpb, lpl = _ws_logprobs(ws, B, T, U1, dtype)
    _check_rnnt(*out, lpb, lpl, xlen, ylen, costs)
    again = rnnt_forced_align(acts, labels, xlen, ylen, blank=blank)
    for a, b in zip(out, again):
        assert torch.equal(a, b)
    if kind == "constant":                                   # every path ties: all labels at the first frame
        assert np.all(_np(out[0])[0] == 0)


def test_rnnt_viterbi_is_per_utterance_and_repeatable():
    from edgedict_b200.align import rnnt_forced_align
    acts, labels, xlen, ylen = _rnnt_problem(6, 80, 12, 10, f32, 0, "random", 5)
    full = rnnt_forced_align(acts, labels, xlen, ylen)
    again = rnnt_forced_align(acts, labels, xlen, ylen)
    for a, b in zip(full, again):
        assert torch.equal(a, b)
    from edgedict_b200 import ops
    for b in range(6):                                        # utterance b alone, over the same padded lattice
        xl, yl = xlen[b:b + 1].cuda(), ylen[b:b + 1].cuda()
        _, ws = ops.rnnt_loss_fwd(acts[b:b + 1].contiguous(), labels[b:b + 1], xl, yl, 0, need_beta=False)
        fr, lp, sc = ops.rnnt_viterbi(xl, yl, 1, 80, 12, ws, f32)
        assert torch.equal(fr[0], full[0][b]) and torch.equal(lp[0], full[1][b]) and torch.equal(sc[0], full[2][b])


def test_rnnt_viterbi_no_frames_has_no_alignment():
    from edgedict_b200 import ops
    acts, labels, xlen, ylen = _rnnt_problem(3, 10, 4, 6, f32, 0, "random", 9)
    xl, yl = xlen.cuda(), ylen.cuda()
    _, ws = ops.rnnt_loss_fwd(acts, labels, xl, yl, 0, need_beta=False)
    xl[2] = 0                                                 # the workspace is not read for utterance 2
    frames, logp, score = ops.rnnt_viterbi(xl, yl, 3, 10, 4, ws, f32)
    assert float(score[2]) == -np.inf and bool((frames[2] == -1).all()) and bool((logp[2] == -np.inf).all())


# ---- CTC -------------------------------------------------------------------------------------------------------------
def _ctc_problem(B, T, V, S, blank, kind, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "constant":
        lp = torch.full((B, T, V), -float(np.log(V)))
    elif kind == "two_values":
        lp = torch.randint(0, 2, (B, T, V), generator=g).float().log_softmax(-1)
    else:
        lp = (torch.randn(B, T, V, generator=g) * 2).log_softmax(-1)
    labels = torch.randint(0, V - 1, (B, S), generator=g)
    labels += (labels >= blank).long()
    tl = torch.randint(0, S + 1, (B,), generator=g)
    tl[0] = S
    il = torch.full((B,), T, dtype=torch.long)
    for b in range(1, B):
        il[b] = int(torch.randint(min(T, 2 * int(tl[b]) + 1), T + 1, (1,), generator=g))
    return lp, labels, il, tl


def _check_ctc(al, fl, lp, labels, il, tl, blank, costs=None):
    al, fl = _np(al), _np(fl)
    for b in range(lp.shape[0]):
        Tb, Sb = int(il[b]), int(tl[b])
        ra, rl, rs = ao.ctc_viterbi(_np(lp[b, :Tb]), _np(labels[b, :Sb]), blank)
        if rs == -np.inf:
            assert np.all(al[b] == -1) and np.all(fl[b] == -np.inf), b
            continue
        assert np.array_equal(al[b, :Tb], ra), b
        assert np.array_equal(fl[b, :Tb], rl), b
        assert np.all(al[b, Tb:] == -1) and np.all(fl[b, Tb:] == 0), b
        acc = 0.0
        for x in fl[b, :Tb]:
            acc += float(x)
        assert acc == rs, b
        if costs is not None:
            assert rs <= -costs[b] + 1e-5 * abs(costs[b]) + 1e-5, (b, rs, costs[b])


CTC_CASES = [
    (4, 50, 6, 5, 0, "random", "padded"),
    (3, 200, 30, 0, 0, "random", "padded"),                # S = 0
    (5, 100, 10, 20, 0, "random", "concat"),               # back-pointers in shared memory
    (3, 120, 3, 40, 0, "random", "padded"),                # many repeated labels
    (2, 2000, 40, 511, 0, "random", "strided"),            # 1023 states, two per thread
    (2, 1100, 40, 512, 0, "random", "padded"),             # 1025 states, four per thread
    (2, 2000, 60, 1023, 0, "random", "concat"),
    (2, 499, 40, 223, 0, "random", "padded"),              # back-pointers fit in shared memory, 439 bytes spare
    (2, 500, 40, 223, 0, "random", "padded"),              # 8 bytes over: staged from the caller's buffer
    (2, 1148, 40, 99, 0, "random", "concat"),              # exactly the 227 KB opt-in limit
    (2, 1149, 40, 99, 0, "random", "concat"),              # one frame more: staged
    (4, 70, 9, 6, 8, "random", "strided"),                 # blank = V - 1
    (3, 40, 5, 6, 0, "constant", "padded"),
    (4, 60, 6, 8, 0, "two_values", "padded"),
]


@pytest.mark.parametrize("B, T, V, S, blank, kind, layout", CTC_CASES)
def test_ctc_align_teacher_forced_bitwise(B, T, V, S, blank, kind, layout):
    from edgedict_b200.ctc import ctc_loss, forced_align
    lp, labels, il, tl = _ctc_problem(B, T, V, S, blank, kind, B * 100 + T + S)
    if layout == "strided":                                   # a [T, B, V] tensor seen batch first
        dev = lp.transpose(0, 1).contiguous().cuda().transpose(0, 1)
    else:
        dev = lp.cuda()
    tg = labels if layout != "concat" else torch.cat([labels[b, :int(tl[b])] for b in range(B)])
    al, fl = forced_align(dev, tg.cuda(), il, tl, blank=blank)
    assert al.dtype == tg.dtype and al.shape == (B, T) and fl.dtype == f32
    costs = _np(ctc_loss(dev.transpose(0, 1), tg.cuda(), il, tl, blank=blank, reduction="none"))
    _check_ctc(al, fl, lp, labels, il, tl, blank, costs)
    al2, fl2 = forced_align(dev, tg.cuda(), il, tl, blank=blank)
    assert torch.equal(al, al2) and torch.equal(fl, fl2)


def test_ctc_align_edge_utterances_and_batch_independence():
    from edgedict_b200.ctc import forced_align
    B, T, V = 6, 30, 7
    lp, labels, il, tl = _ctc_problem(B, T, V, 8, 0, "random", 3)
    labels[1, :4] = torch.tensor([2, 2, 2, 2])
    tl[1], il[1] = 4, 6                                       # needs 7 frames for 2 2 2 2: no alignment
    tl[2], il[2] = max(int(tl[2]), 1), 0                      # no frames, labels: no alignment
    tl[3], il[3] = 0, 0                                       # no frames, no labels: aligned, nothing to say
    labels[4, 0], tl[4] = V, max(int(tl[4]), 1)               # a label outside [0, V)
    al, fl = forced_align(lp.cuda(), labels.cuda(), il, tl)
    _check_ctc(al, fl, lp, labels, il, tl, 0)
    for b in (1, 2, 4):
        assert bool((al[b] == -1).all()) and bool((fl[b] == -np.inf).all())
    assert bool((al[3] == -1).all()) and bool((fl[3] == 0).all())
    for b in range(B):
        a1, f1 = forced_align(lp[b:b + 1].cuda(), labels[b:b + 1].cuda(), il[b:b + 1], tl[b:b + 1])
        assert torch.equal(a1[0], al[b]) and torch.equal(f1[0], fl[b])


# ---- models against the fp64 oracles ---------------------------------------------------------------------------------
TINY = dict(vocab_embed_size=16, vocab_size=64, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0,
            enc_proj_size=40, dec_hidden_size=32, dec_layers=1, dec_dropout=0, dec_proj_size=24, joint_size=56)
E6D2 = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
            enc_proj_size=640, dec_hidden_size=256, dec_layers=2, dec_dropout=0.0, dec_proj_size=256, joint_size=640)


def _capture_viterbi(monkeypatch):
    """Record the workspace Transducer.align hands to the Viterbi kernel."""
    from edgedict_b200 import ops
    seen = {}
    real = ops.rnnt_viterbi

    def spy(xlen, ylen, B, T, U, ws, dtype):
        out = real(xlen, ylen, B, T, U, ws, dtype)
        seen.update(ws=ws.clone(), dims=(B, T, U), dtype=dtype)
        return out

    monkeypatch.setattr(ops, "rnnt_viterbi", spy)
    return seen


@pytest.mark.parametrize("dims, precision, module", [("tiny", "fp32", "LSTM"), ("tiny", "bf16", "LSTM"),
                                                     ("e6d2", "fp32", "LSTM"), ("e6d2", "bf16", "LSTM"),
                                                     ("tiny", "fp32", "GRU"), ("tiny", "bf16", "peaked")])
def test_transducer_align_against_fp64_oracle(monkeypatch, dims, precision, module):
    from edgedict_b200.rnnt.models import Transducer
    from oracle import model_torch as mt
    cfg, B, T, U = (TINY, 3, 23, 6) if dims == "tiny" else (E6D2, 4, 200, 32)
    torch.manual_seed(11)
    m = Transducer(module_type="GRU" if module == "GRU" else "LSTM", **cfg)
    if module == "peaked":                                    # one alignment dominates every other
        with torch.no_grad():
            m.joint.joint[2].weight.mul_(30)
            m.joint.joint[2].bias.mul_(30)
    m = m.cuda().set_precision(precision)
    g = torch.Generator().manual_seed(12)
    xs = torch.randn(B, T, cfg["input_size"], generator=g)
    ys = torch.randint(1, cfg["vocab_size"], (B, U), generator=g, dtype=torch.int32)
    xlen = torch.tensor([T] + [T - 3 * k - 1 for k in range(1, B)], dtype=torch.int32)
    ylen = torch.tensor([U] + [max(U - 2 * k - 1, 0) for k in range(1, B)], dtype=torch.int32)
    seen = _capture_viterbi(monkeypatch)
    frames, logps, nscore = m.align(xs.cuda(), ys.cuda(), xlen, ylen)
    Bw, Tw, Uw = seen["dims"]
    lpb, lpl = _ws_logprobs(seen["ws"], Bw, Tw, Uw, seen["dtype"])
    # fp64 oracle log-probs of the same model
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    with torch.no_grad():
        enc = mt.encoder_gru if module == "GRU" else mt.encoder
        h_enc, _ = enc(sd, xs.double())
        h_dec, _ = mt.decoder(sd, ys)
        lp = torch.log_softmax(mt.joint(sd, h_enc, h_dec), -1)
    xl = _np(mt.scale_length(lp.shape[1], xlen))
    score = _np(-nscore)
    for b in range(B):
        Tb, Ub = int(xl[b]), int(ylen[b]) + 1
        ob = _np(lp[b, :Tb, :Ub, 0])
        ol = np.zeros((Tb, Ub))
        ol[:, :Ub - 1] = _np(lp[b, :Tb, torch.arange(Ub - 1), ys[b, :Ub - 1].long()].reshape(Tb, Ub - 1))
        # teacher-forced: bit for bit over the values the kernel read
        rf, rl, rs = ao.rnnt_viterbi(lpb[b, :Tb, :Ub], lpl[b, :Tb, :Ub])
        assert np.array_equal(frames[b], rf) and np.array_equal(logps[b], rl)
        assert score[b] == np.float32(rs)
        # against the fp64 optimum, within the measured per-cell error along a path
        eps = max(np.abs(lpb[b, :Tb, :Ub] - ob).max(), np.abs(lpl[b, :Tb, :Ub - 1] - ol[:, :Ub - 1]).max()
                  if Ub > 1 else 0.0)
        of, _, opt = ao.rnnt_viterbi(ob, ol)
        got = _path_sum(ob, ol, frames[b])
        bar = 2 * (Tb + Ub) * eps
        print("  %s %s %s b=%d eps %.3g: fp64 optimum %.6f, device path %.6f (bar %.3g)"
              % (dims, precision, module, b, eps, opt, got, bar))
        assert got >= opt - bar and got <= opt
        if module == "peaked":
            assert np.array_equal(frames[b], of)


@pytest.mark.parametrize("dims, precision", [("tiny", "fp32"), ("tiny", "bf16"), ("e6d2", "fp32"), ("e6d2", "bf16"),
                                             ("tiny", "peaked")])
def test_ctc_encoder_align_against_fp64_oracle(dims, precision):
    from edgedict_b200.rnnt.models import CTCEncoder
    from oracle import ctc as oc
    from oracle import model_torch as mt
    if dims == "tiny":
        cfg, B, T, S = dict(vocab_size=32, input_size=24, enc_hidden_size=48, enc_layers=2, enc_dropout=0,
                            proj_size=40), 3, 40, 6
    else:
        cfg, B, T, S = dict(vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0,
                            proj_size=640), 4, 200, 32
    torch.manual_seed(21)
    m = CTCEncoder(**cfg)
    if precision == "peaked":
        with torch.no_grad():
            m.tovocab[0].weight.mul_(30)
            m.tovocab[0].bias.mul_(30)
    m = m.cuda().set_precision("bf16" if precision == "bf16" else "fp32")
    g = torch.Generator().manual_seed(22)
    xs = torch.randn(B, T, cfg["input_size"], generator=g)
    ys = torch.randint(1, cfg["vocab_size"], (B, S), generator=g)
    xlen = torch.tensor([T] + [T - 5 * k for k in range(1, B)])
    ylen = torch.tensor([S] + [S - 2 * k for k in range(1, B)])
    al, fl = m.align(xs.cuda(), ys.cuda(), xlen, ylen)
    lp_dev = _np(m(xs.cuda()))
    sd = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    with torch.no_grad():
        lp = _np(oc.ctc_encoder_forward(sd, xs.double()))
    xl = _np(mt.scale_length(lp.shape[1], xlen))
    al, fl = _np(al), _np(fl)
    for b in range(B):
        Tb, Sb = int(xl[b]), int(ylen[b])
        labels = _np(ys[b, :Sb])
        ra, rl, _ = ao.ctc_viterbi(lp_dev[b, :Tb], labels, 0)
        assert np.array_equal(al[b, :Tb], ra) and np.array_equal(fl[b, :Tb], rl)
        eps = float(np.abs(lp_dev[b, :Tb] - lp[b, :Tb]).max())
        oa, _, opt = ao.ctc_viterbi(lp[b, :Tb], labels, 0)
        got = float(lp[b, np.arange(Tb), al[b, :Tb]].sum())
        bar = 2 * Tb * eps
        print("  CTC %s %s b=%d eps %.3g: fp64 optimum %.6f, device path %.6f (bar %.3g)"
              % (dims, precision, b, eps, opt, got, bar))
        assert got >= opt - bar and got <= opt + 1e-9 * abs(opt)
        if precision == "peaked":
            assert np.array_equal(al[b, :Tb], oa)
