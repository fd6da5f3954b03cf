"""Teacher-forced fp64 parity of the decode program kernel (csrc/decode.cu, decode_program_kernel), per phase and per
element: LSTM, LINEAR, LN, PAIR, COPY and ARGMAX run as one-phase programs through eb_decode_run, then a whole
StreamEngine chunk and a GreedyEngine run, layer by layer and frame by frame.  Every reference is computed in fp64 from
the kernel's own inputs, so errors do not compound and a failure names one (row, column).

Error model (first order, per element; derived from decode.cu):
  products        3xTF32: x = hi + lo with hi = tf32_rna(x) (11 significant bits) and lo = tf32_rna(x - hi) (11 more),
                  a*b = a_lo b_hi + a_hi b_lo + a_hi b_hi with the lo*lo term dropped: about 3 * 2^-22 |a||b| per
                  product, counted as 6 UTC on sum_k |x_k||w_k|.
  accumulation    n_add UTC sum_k |x_k||w_k| (UTC = 2^-23 per tensor-core add).  n_add is the longest fp32 chain of
                  tile_mma: the 16-wide k steps of all K segments of a tile are dealt round-robin to 8 warps (step_ctr
                  continues across the K1 and K2 segments), each step adds 3 MMAs x 2 into the same accumulator, then
                  tile_reduce adds the 8 warp partials in order (`_n_add`).  The epilogue adds b1 (and b2) with one
                  fp32 rounding each, then LINEAR's tanh (EPS_LIBM absolute).
  LSTM cell       fwd_ref's propagation (test_gpu_lstm_recurrence_fp64) with T = 1 and EPS_LIBM for expf / tanhf; the
                  cell state of the encoder's n steps per chunk is recursed in fp64 with its bar alongside.
  LN              the two-pass mean and variance in fp32 (`ln_ref`): the lane chains of ceil(H/32) adds plus 5 shuffle
                  adds, the cancellation in z - mu for rows with a large mean, rsqrtf (2 ulp), and the affine epilogue.
  chunk level     the bars of teacher-forced inputs are zero; where a frame's input is not visible (the predictor state
                  between two output frames, greedy's frames), it is recomputed in fp64 and its bar propagated through
                  |W| into the next phase.

Every matrix-phase test also proves it could tell 3xTF32 from plain TF32: it computes on the host, in fp64 from
TF32-rounded operands, the error plain TF32 products would make, and asserts that it exceeds the test's own bar at least
8x somewhere.  Each matrix test plants one "TF32-adversarial" row and output column (all of one sign, each value 0.45
TF32 ulp above a TF32 value, so the TF32 rounding errors add up instead of cancelling).

Every phase runs with max_ctas in {0, 1, 3, 17}: the outputs must be bitwise identical, since each element's summation
order is fixed by the warp split and tile_reduce, not by the grid.  max_ctas = 1 runs every tile through the grid-stride
loop of one CTA and reuses its shared memory from tile to tile.  Outputs are filled with NaN before each run, so a tile
that is skipped shows.

pytest -s prints the worst err/bar of every phase and shape next to the element where it occurs, and the power-check
ratio.  DESIGN.md (verification table, greedy / streaming decode) records the measured figures."""
import numpy as np
import pytest
import torch

from tests.test_gpu_lstm_recurrence_fp64 import EPS_LIBM, U24, UTC, _report, fwd_ref

pytestmark = pytest.mark.gpu

f32, f64, i32 = torch.float32, torch.float64, torch.int32
DEV = "cuda"
CTAS = (0, 1, 3, 17)              # 0: one CTA per SM (the engines' default)
POWER = 8.0                       # plain TF32 must exceed the bar by this much somewhere
LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
RAGGED = dict(vocab_embed_size=24, vocab_size=77, input_size=37, enc_hidden_size=100, enc_layers=3, enc_dropout=0.0,
              enc_proj_size=70, dec_hidden_size=60, dec_layers=2, dec_dropout=0.0, dec_proj_size=45, joint_size=91)


# ---- running programs -------------------------------------------------------------------------------------------------
def _run(phases, max_ctas=0):
    from edgedict_b200._lib import check, lib
    from edgedict_b200.stream_engine import EbPhase
    arr = (EbPhase * len(phases))(*phases)
    prog = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(DEV)
    bar = torch.zeros(64, dtype=i32, device=DEV)
    check(lib().eb_decode_run(prog.data_ptr(), len(phases), bar.data_ptr(), max_ctas,
                              torch.cuda.current_stream().cuda_stream), "eb_decode_run")
    torch.cuda.synchronize()


def _bits(t):
    return t.contiguous().view(i32) if t.dtype == f32 else t


def _run_all(phases, outs, reset):
    """Run the program once per max_ctas in CTAS, each time after reset(); the outputs must be bitwise identical.
    Returns copies of the outputs of the full-grid run."""
    first = None
    for mc in CTAS:
        reset()
        _run(phases, mc)
        snap = [o.clone() for o in outs]
        if first is None:
            first = snap
            continue
        for k, (a, b) in enumerate(zip(first, snap)):
            diff = (_bits(a) != _bits(b)).nonzero()
            assert diff.numel() == 0, "output %d: max_ctas=%d differs from the full grid at %s" % (
                k, mc, diff[:4].tolist())
    return first


# ---- error model ------------------------------------------------------------------------------------------------------
def _n_add(*Ks):
    """Longest fp32 chain of one tile_mma output over K segments Ks, plus the 3xTF32 product error as 6 UTC."""
    steps = sum(-(-k // 16) for k in Ks)
    return 6 * -(-steps // 8) + 8 + 6


def _tf32(x):
    """cvt.rna.tf32.f32 on the host: round to 10 explicit mantissa bits, ties away from zero."""
    u = x.detach().float().cpu().contiguous().numpy().view(np.uint32)
    return torch.from_numpy(((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)).to(x.device)


def _adversarial(shape, scale, gen):
    """Positive values 0.45 TF32 ulp above a TF32 value: tf32_rna rounds every one of them down by the same share."""
    t = _tf32(0.5 + 0.5 * torch.rand(shape, generator=gen)).double()          # TF32 values in [0.5, 1)
    return ((t + 0.45 * 2.0 ** -11) * scale).float()


def _power(name, pairs, bar):
    """pairs: [(x [R,K], w [N,K])] the operands of one product sum; bar [R,N] the test's bar of that sum.  Asserts that
    plain TF32 products would err by more than POWER x bar somewhere."""
    exact = sum(x.double() @ w.double().t() for x, w in pairs)
    tf = sum(_tf32(x).double() @ _tf32(w).double().t() for x, w in pairs)
    r = float(((tf - exact).abs() / bar).max())
    print("  %-34s plain-TF32 err / bar: %.1f" % (name, r))
    assert r >= POWER, "%s: the bar cannot tell 3xTF32 from plain TF32 (ratio %.2f)" % (name, r)


def linear_ref(x1, w1, b, x2=None, w2=None, tanh=False, dx1=None, dx2=None):
    """fp64 y = act(x1 W1^T (+ x2 W2^T) + b) with its bar; dx1 / dx2 are bars the operands already carry."""
    x1, w1 = x1.double(), w1.double()
    v = x1 @ w1.t()
    A = x1.abs() @ w1.abs().t()
    Ks = [w1.shape[1]]
    prop = 0.0 if dx1 is None else dx1 @ w1.abs().t()
    if x2 is not None:
        x2, w2 = x2.double(), w2.double()
        v = v + x2 @ w2.t()
        A = A + x2.abs() @ w2.abs().t()
        Ks.append(w2.shape[1])
        if dx2 is not None:
            prop = prop + dx2 @ w2.abs().t()
    bar = _n_add(*Ks) * UTC * A + prop
    if b is not None:
        b = b.double()
        bar = bar + U24 * (v.abs() + b.abs())
        v = v + b
    if tanh:
        v = torch.tanh(v)
        bar = (1 - v * v) * bar + EPS_LIBM + U24 * v.abs()
    return v, bar


def lstm_ref(x1, w1, x2, w2, b1, b2, c, dx1=None, dx2=None, dc=None):
    """One LSTM phase step in fp64 (gate rows i|f|g|o of W1 [4H,K1], W2 [4H,K2]) through fwd_ref with T = 1.
    Returns (c, dc, y, dy) [S,H]; dx1 / dx2 / dc are bars the inputs already carry."""
    x1, w1, x2, w2, b1, b2 = (a.double() for a in (x1, w1, x2, w2, b1, b2))
    hin = torch.cat([x1, x2], 1)
    w = torch.cat([w1, w2], 1)
    S = hin.shape[0]
    xg = (b1 + b2).expand(S, -1)
    # the epilogue adds b1 then b2: one more rounding than fwd_ref's single bias add
    dpre = 2 * U24 * (hin.abs() @ w.abs().t() + b1.abs() + b2.abs())
    if dx1 is not None:
        dpre = dpre + dx1 @ w1.abs().t()
    if dx2 is not None:
        dpre = dpre + dx2 @ w2.abs().t()
    r = fwd_ref(xg[:, None], w, hin[:, None], c.double()[:, None], _n_add(w1.shape[1], w2.shape[1]), UTC, EPS_LIBM,
                dpre[:, None], 0.0 if dc is None else dc[:, None])
    return r["c"][0][:, 0], r["c"][1][:, 0], r["y"][0][:, 0], r["y"][1][:, 0]


def ln_ref(z32, w, b):
    """LayerNorm (eps 1e-5) of the fp32 rows z32 [R,H] as phase_ln forms them, in fp64 with the bar of its fp32
    two-pass evaluation."""
    z, w, b = z32.double(), w.double(), b.double()
    H = z.shape[1]
    n = -(-H // 32) + 5                                       # lane chain + butterfly
    mu = z.mean(1, keepdim=True)
    dmu = n * U24 * z.abs().sum(1, keepdim=True) / H + U24 * mu.abs()
    d = z - mu
    dd = dmu + U24 * d.abs()
    q = (d * d).sum(1, keepdim=True)
    dq = (2 * d.abs() * dd + dd * dd).sum(1, keepdim=True) + (n + 1) * U24 * q
    var = q / H + 1e-5
    dvar = dq / H + 2 * U24 * var
    rs = var.rsqrt()
    drs = rs * (0.5 * dvar / var + 4 * U24)                  # rsqrtf: 2 ulp
    y = d * rs * w + b
    dy = w.abs() * (dd * rs + d.abs() * drs) + 3 * U24 * ((d * rs * w).abs() + b.abs())
    return y, dy


def argmax_rule(x, unk):
    """torch.argmax of every row of a CPU copy (NaN ranks first, the lowest index wins), then the <unk> rule of
    rnnt/stream.py:105-108: where the token is unk, its logit := 0 and argmax again."""
    x = x.detach().cpu().clone()
    p = torch.argmax(x, 1)
    if unk >= 0:
        hit = p == unk
        if hit.any():
            x2 = x[hit]
            x2[:, unk] = 0
            p[hit] = torch.argmax(x2, 1)
    return p


def may_win(z, bar, unk):
    """[R,V] bool: the tokens the argmax with the <unk> rule may return for logits anywhere in z +- bar."""
    def top(z, bar):
        return (z + bar) >= (z - bar).max(1, keepdim=True).values
    m1 = top(z, bar)
    out = m1.clone()
    if unk >= 0:
        out[:, unk] = False
        z2, b2 = z.clone(), bar.clone()
        z2[:, unk] = 0
        b2[:, unk] = 0
        out |= top(z2, b2) & m1[:, unk:unk + 1]
    return out


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=f32, device=DEV)


# ---- LSTM ---------------------------------------------------------------------------------------------------------------
# S, H, K1, K2, mode.  plain: dense rows; strided: the encoder's x1 = X + t I, ldx1 = ni I (t = 1 of ni = 3) and
# x2 = y_{t-1} with ldx2 = ni H; offset: x1 one float past a 16-byte boundary with ldx1 = K1 + 4; embed: F_EMBED rows
# with repeated tokens and F_MASKED with a mix of blank and non-blank tokens (K2 = H: the masked rows copy x2).
LSTM_CASES = [
    (1, 8, 1, 3, "plain"),
    (63, 12, 5, 17, "strided"),
    (64, 20, 17, 20, "embed"),
    (65, 100, 240, 100, "strided"),
    (130, 512, 3, 640, "offset"),
    (200, 1024, 640, 1024, "strided"),
    (200, 100, 240, 100, "embed"),
    (70, 12, 1, 12, "embed"),
    (130, 20, 640, 5, "offset"),
]


@pytest.mark.parametrize("S,H,K1,K2,mode", LSTM_CASES)
def test_lstm_phase(S, H, K1, K2, mode):
    from edgedict_b200.stream_engine import EbPhase, F_EMBED, F_MASKED, PH_LSTM, _ptr
    gen = torch.Generator().manual_seed(S * 7 + H + K1 + K2)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, generator=gen) * sc).to(DEV)
    G = 4 * H
    w1, w2 = rnd(G, K1, sc=1.5 / K1 ** 0.5), rnd(G, K2, sc=1.5 / K2 ** 0.5)
    b1, b2 = rnd(G, sc=0.5), rnd(G, sc=0.5)
    c0 = rnd(S, H, sc=1.5)
    scale = 2.0 ** -round(np.log2(0.3 * (K1 + K2)))          # the adversarial pre-activation stays O(1)
    for g in range(4):                                        # unit 0: every gate row
        w1[g * H] = _adversarial(K1, scale, gen).to(DEV)
        w2[g * H] = _adversarial(K2, scale, gen).to(DEV)
    ni, t, blank, flags = 3, 1, 2, 0
    if mode == "embed":
        Vt = 9
        table = rnd(Vt, K1)
        tok = torch.randint(0, Vt, (S,), generator=gen).to(DEV).int()
        tok[::3] = blank                                      # masked rows
        tok[0] = 5
        table[5] = _adversarial(K1, 1.0, gen).to(DEV)
        x1v = table[tok.long()]
        x1, ldx1, flags = table, K1, F_EMBED | F_MASKED
        hbuf = rnd(S, K2)
        hbuf[0] = _adversarial(K2, 1.0, gen).to(DEV)
        x2, ldx2, x2v = hbuf, K2, hbuf
    elif mode == "strided":
        X = rnd(S, ni, K1)
        X[0, t] = _adversarial(K1, 1.0, gen).to(DEV)
        Y = rnd(S, ni, K2)
        Y[0, t - 1] = _adversarial(K2, 1.0, gen).to(DEV)
        x1, ldx1, x1v = X.view(-1)[t * K1:], ni * K1, X[:, t]
        x2, ldx2, x2v = Y.view(-1)[(t - 1) * K2:], ni * K2, Y[:, t - 1]
    else:
        off = 1 if mode == "offset" else 0
        ldx1 = K1 + 4 * off
        buf = rnd(S * ldx1 + 4)
        x1v = buf[off:off + S * ldx1].view(S, ldx1)[:, :K1]
        x1v[0] = _adversarial(K1, 1.0, gen).to(DEV)
        x1 = buf[off:]
        x2 = rnd(S, K2)
        x2[0] = _adversarial(K2, 1.0, gen).to(DEV)
        ldx2, x2v = K2, x2
    ldy = ni * H if mode == "strided" else H
    ybuf = _nan(S, ldy)
    yoff = t * H if mode == "strided" else 0
    y2 = _nan(S, H)
    c = c0.clone()
    tok_in = tok if mode == "embed" else None
    ph = EbPhase(type=PH_LSTM, S=S, N=H, K1=K1, K2=K2, flags=flags, x1=_ptr(x1), ldx1=ldx1, x2=_ptr(x2), ldx2=ldx2,
                 w1=_ptr(w1), ldw1=K1, w2=_ptr(w2), ldw2=K2, b1=_ptr(b1), b2=_ptr(b2), c=_ptr(c),
                 y=_ptr(ybuf, yoff), ldy=ldy, y2=_ptr(y2), tok_in=_ptr(tok_in), aux=blank)

    def reset():
        c.copy_(c0)
        ybuf.fill_(float("nan"))
        y2.fill_(float("nan"))

    cg, yb, y2g = _run_all([ph], [c, ybuf, y2], reset)
    y = yb[:, yoff:yoff + H]
    rest = torch.cat([yb[:, :yoff], yb[:, yoff + H:]], 1)
    assert torch.isnan(rest).all(), "LSTM wrote outside its y columns"
    assert torch.equal(_bits(y2g), _bits(y)), "y2 is not a bitwise copy of y"
    cr, dc, yr, dy = lstm_ref(x1v, w1, x2v, w2, b1, b2, c0)
    name = "lstm S=%d H=%d K=%d+%d %s" % (S, H, K1, K2, mode)
    act = torch.ones(S, dtype=torch.bool, device=DEV)
    if mode == "embed":
        act = tok != blank
        m = ~act
        assert m.any() and act.any()
        assert torch.equal(_bits(cg[m]), _bits(c0[m])), "masked rows changed c"
        assert torch.equal(_bits(y[m]), _bits(x2v[m][:, :H])), "masked rows did not copy h"
    _report(name, [("c", cg[act], cr[act], dc[act]), ("y", y[act], yr[act], dy[act])])
    pre_bar = _n_add(K1, K2) * UTC * (torch.cat([x1v, x2v], 1).double().abs() @ torch.cat([w1, w2], 1).double().abs().t())
    _power(name, [(x1v, w1), (x2v, w2)], pre_bar)


# ---- LINEAR ---------------------------------------------------------------------------------------------------------------
# S, N, K1, K2 (0: no second segment), tanh, x1_div, pad of ldx1 beyond K1
LINEAR_CASES = [
    (1, 1, 1, 0, False, 0, 0),
    (31, 33, 3, 5, True, 1, 2),
    (33, 1025, 17, 0, False, 3, 0),
    (1025, 31, 240, 17, True, 8, 4),
    (130, 1025, 640, 640, True, 0, 0),          # the joint hidden layer at E6D2: K1 = E, K2 = D
    (65, 1024, 640, 0, False, 0, 1),            # the output layer
    (200, 33, 5, 1, False, 3, 3),
    (31, 1, 640, 3, True, 8, 0),
]


@pytest.mark.parametrize("S,N,K1,K2,tanh,x1_div,pad", LINEAR_CASES)
def test_linear_phase(S, N, K1, K2, tanh, x1_div, pad):
    from edgedict_b200.stream_engine import EbPhase, F_TANH, PH_LINEAR, _ptr
    gen = torch.Generator().manual_seed(S + 3 * N + 5 * K1 + K2 + x1_div)
    rnd = lambda *s, sc=1.0: (torch.randn(*s, generator=gen) * sc).to(DEV)
    ldx1 = K1 + pad
    x1b = rnd(S, ldx1)                            # row r reads x1[r / x1_div]: the rows past S / x1_div differ
    x1b[0, :K1] = _adversarial(K1, 1.0, gen).to(DEV)
    w1 = rnd(N, K1, sc=1.0 / K1 ** 0.5)
    scale = 2.0 ** -round(np.log2(0.3 * (K1 + K2)))
    w1[0] = _adversarial(K1, scale, gen).to(DEV)
    b = rnd(N, sc=0.3)
    x2 = w2 = None
    if K2:
        x2 = rnd(S, K2)
        x2[0] = _adversarial(K2, 1.0, gen).to(DEV)
        w2 = rnd(N, K2, sc=1.0 / K2 ** 0.5)
        w2[0] = _adversarial(K2, scale, gen).to(DEV)
    y = _nan(S, N)
    ph = EbPhase(type=PH_LINEAR, S=S, N=N, K1=K1, K2=K2, flags=F_TANH if tanh else 0, x1=_ptr(x1b), ldx1=ldx1,
                 x1_div=x1_div, x2=_ptr(x2), ldx2=K2, w1=_ptr(w1), ldw1=K1, w2=_ptr(w2), ldw2=K2, b1=_ptr(b),
                 y=_ptr(y), ldy=N)
    (yg,) = _run_all([ph], [y], lambda: y.fill_(float("nan")))
    x1v = x1b[torch.arange(S, device=DEV) // max(x1_div, 1), :K1]
    yr, dy = linear_ref(x1v, w1, b, x2, w2, tanh)
    name = "linear S=%d N=%d K=%d+%d%s div=%d" % (S, N, K1, K2, " tanh" if tanh else "", x1_div)
    _report(name, [("y", yg, yr, dy)])
    pairs = [(x1v, w1)] + ([(x2, w2)] if K2 else [])
    _power(name, pairs, linear_ref(x1v, w1, None, x2, w2)[1])


# ---- LN, PAIR, COPY -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [12, 240, 1024, 1500])
@pytest.mark.parametrize("res", [False, True])
def test_ln_phase(H, res):
    """Rows: random; constant (var = 0: rs = rsqrt(eps) ~ 316 magnifies any error of the mean, and 0.75 * H is exact in
    fp32, so the result must be b bitwise); mean 1e3 - 1e4 with spread 1 (z - mu cancels); variance ~ eps."""
    from edgedict_b200.stream_engine import EbPhase, PH_LN, _ptr
    gen = torch.Generator().manual_seed(H + res)
    R = 77
    x1 = torch.randn(R, H, generator=gen) * 1.7
    x1[10:20] = 0.5 if res else 0.75
    x1[20:40] = torch.logspace(3, 4, 20)[:, None] + torch.randn(20, H, generator=gen)
    x1[40:60] = 0.3 + torch.randn(20, H, generator=gen) * torch.logspace(-3.5, -2, 20)[:, None]
    x2 = None
    if res:
        x2 = torch.randn(R, H, generator=gen)
        x2[10:20] = 0.25
        x2[20:60] = 0.0
        x2 = x2.to(DEV)
    x1 = x1.to(DEV)
    w = (torch.randn(H, generator=gen) * 0.5 + 1).to(DEV)
    b = (torch.randn(H, generator=gen) * 0.2).to(DEV)
    y = _nan(R, H + 3)
    ph = EbPhase(type=PH_LN, S=R, N=H, x1=_ptr(x1), ldx1=H, x2=_ptr(x2), ldx2=H, w1=_ptr(w), b1=_ptr(b), y=_ptr(y),
                 ldy=H + 3)
    (yg,) = _run_all([ph], [y], lambda: y.fill_(float("nan")))
    assert torch.isnan(yg[:, H:]).all()
    yg = yg[:, :H]
    z32 = x1 + x2 if res else x1
    assert torch.equal(_bits(yg[10:20]), _bits(b.expand(10, H))), "constant rows must give b bitwise"
    yr, dy = ln_ref(z32, w, b)
    name = "ln H=%d%s" % (H, " +res" if res else "")
    _report(name, [("random", yg[:10], yr[:10], dy[:10]), ("mean1e3+", yg[20:40], yr[20:40], dy[20:40]),
                   ("var~eps", yg[40:60], yr[40:60], dy[40:60]), ("rest", yg[60:], yr[60:], dy[60:])])


@pytest.mark.parametrize("aux", [2, 4, 6])
@pytest.mark.parametrize("H", [5, 100, 1024])
def test_pair_and_copy_phases(aux, H):
    from edgedict_b200.stream_engine import EbPhase, PH_COPY, PH_PAIR, _ptr
    gen = torch.Generator().manual_seed(aux * 100 + H)
    S = 67
    x = (torch.randn(S, aux, H, generator=gen) * 3).to(DEV)
    y = _nan(S, aux // 2, H)
    y2 = _nan(S * aux, H)
    phases = [EbPhase(type=PH_PAIR, S=S, N=H, aux=aux, x1=_ptr(x), y=_ptr(y)),
              EbPhase(type=PH_COPY, S=S * aux, N=H, x1=_ptr(x), y=_ptr(y2))]

    def reset():
        y.fill_(float("nan"))
        y2.fill_(float("nan"))

    yg, cg = _run_all(phases, [y, y2], reset)
    want = 0.5 * (x[:, 0::2] + x[:, 1::2])                   # fp32, as the kernel rounds it
    assert torch.equal(_bits(yg), _bits(want)), "PAIR differs from 0.5f * (a + b)"
    assert torch.equal(_bits(cg), _bits(x.view(S * aux, H))), "COPY is not bitwise"


# ---- ARGMAX ---------------------------------------------------------------------------------------------------------------
TIES = [(0, 32), (5, 32), (0, 1), (7, 1), (9, 64)]          # row r: equal maxima at a and a + d (d = 32: the same lane)


def _argmax_rows(V, unk, gen):
    """Random rows plus: exact ties in one lane (v, v + 32) and across lanes (v, v + 1); unk the maximum with a positive
    runner-up; unk the maximum with every other logit negative."""
    x = torch.randn(40, V, generator=gen) * 3
    if V >= 2:
        for r, (a, d) in enumerate(TIES):
            if a + d < V:
                x[r, a] = x[r, a + d] = x[r].max() + 1.0
        x[10, unk] = x[10].max() + 2.0                        # unk wins, runner-up positive
        x[11] = -(torch.rand(V, generator=gen) + 0.5)         # unk wins, every other logit negative: token stays unk
        x[11, unk] = 1.0
        x[12] = -(torch.rand(V, generator=gen) + 0.5)
        x[12, unk] = -0.1                                     # all negative, unk the maximum
        x[13, unk] = x[13].max() + 1.0
        x[13, V - 1] = x[13, unk] - 0.5                       # the runner-up in the last column
    return x


@pytest.mark.parametrize("V", [1, 31, 33, 1024, 1025])
def test_argmax_phase_ties_and_unk_rule(V):
    from edgedict_b200.stream_engine import EbPhase, PH_ARGMAX, _ptr
    gen = torch.Generator().manual_seed(V)
    unk = min(3, V - 1)
    x = _argmax_rows(V, unk, gen).to(DEV)
    S, HL, col = x.shape[0], 3, 1
    tok = torch.full((S,), -5, dtype=i32, device=DEV)
    hist = torch.full((S, HL), -7, dtype=i32, device=DEV)
    ph = EbPhase(type=PH_ARGMAX, S=S, N=V, x1=_ptr(x), ldx1=V, aux=0, aux2=unk, tok_out=_ptr(tok), hist=_ptr(hist),
                 hist_ld=HL, hist_col=col)

    def reset():
        tok.fill_(-5)
        hist.fill_(-7)

    tg, hg = _run_all([ph], [tok, hist], reset)
    want = argmax_rule(x, unk)
    bad = (tg.cpu().long() != want).nonzero().flatten().tolist()
    assert not bad, "rows %s: kernel %s, torch %s" % (bad[:5], tg.cpu()[bad[:5]].tolist(), want[bad[:5]].tolist())
    assert torch.equal(hg[:, col], tg) and (hg[:, [0, 2]] == -7).all(), "hist column"
    if V > 1:
        assert all(int(want[r]) == a for r, (a, d) in enumerate(TIES) if a + d < V), "the tie rows"
        assert want[10] != unk and want[11] == unk and want[12] == unk and want[13] == V - 1, "the unk rows"
    print("  argmax V=%d: %d rows token for token (ties, unk rule)" % (V, S))


@pytest.mark.parametrize("V", [1, 31, 33, 1025])
def test_argmax_phase_nan_and_neg_inf_rows(V):
    """Rows all NaN, NaN at some positions, all -inf, -inf with one NaN: the token follows torch.argmax (the first
    NaN, index 0 for an all -inf row) and lies in [0, V).  A one-phase program: nothing consumes these tokens."""
    from edgedict_b200.stream_engine import EbPhase, PH_ARGMAX, _ptr
    nan, inf = float("nan"), float("inf")
    gen = torch.Generator().manual_seed(V + 1)
    x = torch.randn(9, V, generator=gen)
    x[0] = nan
    x[1] = -inf
    x[2, V // 2] = nan
    x[3, V - 1] = nan
    x[4, ::5] = nan
    x[5] = -inf
    x[5, V - 1] = nan
    x[6, min(3, V - 1)] = nan                                 # the unk logit is NaN: := 0, then argmax again
    x[7] = -inf
    x[7, V // 3] = 2.0
    x = x.to(DEV)
    for unk in (-1, min(3, V - 1)):
        tok = torch.full((9,), -5, dtype=i32, device=DEV)
        ph = EbPhase(type=PH_ARGMAX, S=9, N=V, x1=_ptr(x), ldx1=V, aux=0, aux2=unk, tok_out=_ptr(tok))
        (tg,) = _run_all([ph], [tok], lambda: tok.fill_(-5))
        tg = tg.cpu().long()
        assert ((tg >= 0) & (tg < V)).all(), "unk=%d: token out of range: %s" % (unk, tg.tolist())
        assert torch.equal(tg, argmax_rule(x, unk)), "unk=%d: kernel %s, torch %s" % (
            unk, tg.tolist(), argmax_rule(x, unk).tolist())


@pytest.mark.parametrize("V", [1, 33, 1024, 1025])
def test_argmax_phase_logp(V):
    """F_LOGP (GreedyEngine: aux2 = -1) against the fp64 log_softmax(x)[pred], accumulated into a nonzero y; logits
    spread over +-80, some rows with the maximum in the last column."""
    from edgedict_b200.stream_engine import EbPhase, F_LOGP, PH_ARGMAX, _ptr
    gen = torch.Generator().manual_seed(V + 2)
    S = 70
    x = (torch.rand(S, V, generator=gen) * 160 - 80)
    x[:20] = torch.randn(20, V, generator=gen) * 2                 # many terms of similar size
    x[20:30, V - 1] = x[20:30].max(1).values + torch.rand(10, generator=gen)
    x[30:35, V - 1] = x[30:35].max(1).values - 0.3
    x = x.to(DEV)
    y0 = (torch.randn(S, generator=gen) * 5).to(DEV)
    y, tok = y0.clone(), torch.zeros(S, dtype=i32, device=DEV)
    ph = EbPhase(type=PH_ARGMAX, S=S, N=V, flags=F_LOGP, x1=_ptr(x), ldx1=V, aux=0, aux2=-1, tok_out=_ptr(tok), y=_ptr(y))

    def reset():
        y.copy_(y0)
        tok.fill_(-5)

    yg, tg = _run_all([ph], [y, tok], reset)
    assert torch.equal(tg.cpu().long(), argmax_rule(x, -1))
    xd = x.double()
    best = xd.gather(1, tg.long()[:, None])
    a = xd - best
    e = a.exp()
    s = e.sum(1)
    n = -(-V // 32) + 5
    ds = (e * (2.0 ** -22 + U24 * a.abs())).sum(1) + n * U24 * s
    yr = y0.double() - s.log()
    bar = ds / s + 2 * U24 * s.log().abs() + 2.0 ** -22 + U24 * (yr.abs() + y0.double().abs())
    _report("argmax logp V=%d" % V, [("y", yg, yr, bar)])


# ---- chunk level: StreamEngine and GreedyEngine -----------------------------------------------------------------------------
def _scaled(cfg, seed):
    """Random-init weights x 2: at x 1 the joint emits blanks only."""
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    m = Transducer(output_loss=False, **cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(2.0)
    return m.cuda()


class _Pred:
    """fp64 predictor steps with bars (the predictor phases: embedding, Ld masked LSTM layers, COPY, projection)."""

    def __init__(self, m):
        sd = {k: v.detach().double() for k, v in m.state_dict().items()}
        self.sd, self.Ld = sd, m.decoder.lstm.num_layers
        self.emb, self.wp, self.bp = sd["decoder.embed.weight"], sd["decoder.proj.weight"], sd["decoder.proj.bias"]
        self.w1, self.b1 = sd["joint.joint.0.weight"], sd["joint.joint.0.bias"]
        self.w2, self.b2 = sd["joint.joint.2.weight"], sd["joint.joint.2.bias"]

    def step(self, tok, st):
        """st = (h, dh, c, dc) [Ld,R,Hd] -> (new state, dec_x, its bar) for tokens tok [R]."""
        h, dh, c, dc = st
        x, dx = self.emb[tok.long()], None
        hs, dhs, cs, dcs = [], [], [], []
        for k in range(self.Ld):
            g = lambda n: self.sd["decoder.lstm.%s_l%d" % (n, k)]
            ck, dck, yk, dyk = lstm_ref(x, g("weight_ih"), h[k], g("weight_hh"), g("bias_ih"), g("bias_hh"), c[k],
                                        dx1=dx, dx2=dh[k], dc=dc[k])
            for lst, v in zip((hs, dhs, cs, dcs), (yk, dyk, ck, dck)):
                lst.append(v)
            x, dx = yk, dyk
        dx_out, ddx = linear_ref(x, self.wp, self.bp, dx1=dx)
        return (torch.stack(hs), torch.stack(dhs), torch.stack(cs), torch.stack(dcs)), dx_out, ddx

    def joint(self, enc, dec_x, ddec):
        E = enc.shape[1]
        return linear_ref(enc, self.w1[:, :E], self.b1, dec_x, self.w1[:, E:], tanh=True, dx2=ddec)

    def logits(self, hid, dhid=None):
        return linear_ref(hid, self.w2, self.b2, dx1=dhid)


def _frames(P, enc_out, hist, st, dec_x, ddec, blank, unk, hidden=None, logits=None):
    """The joint -> argmax -> masked predictor step of every output frame, in fp64 from the device's encoder output and
    the state before the first frame (value, bar), following the device's tokens.  hidden / logits are the device's
    buffers after the last frame (teacher-forced there).  Returns (state, dec_x, ddec, items, undecided rows of each
    frame, rows, fp64 log p of the tokens with its bar)."""
    R, n_out = hist.shape
    items, und, lp, dlp = [], [], 0.0, 0.0
    for k in range(n_out):
        tok = hist[:, k]
        hid, dhid = P.joint(enc_out[:, k], dec_x, ddec)
        if k == n_out - 1 and hidden is not None:
            items.append(("hidden", hidden, hid, dhid))
            z, dz = P.logits(hidden)                       # teacher-forced from the device's hidden
            items.append(("logits", logits, z, dz))
            assert torch.equal(tok.cpu().long(), argmax_rule(logits, unk)), "token != argmax of the device logits"
        else:
            z, dz = P.logits(hid, dhid)
        ok = may_win(z, dz, unk)
        assert ok.gather(1, tok.long()[:, None]).all(), "frame %d rows %s: token outside the fp64 argmax set" % (
            k, (~ok.gather(1, tok.long()[:, None])[:, 0]).nonzero().flatten()[:5].tolist())
        und.append(int((ok.sum(1) > 1).sum()))
        lsm = z - z.logsumexp(1, keepdim=True)
        lp = lp + lsm.gather(1, tok.long()[:, None])[:, 0]
        dlp = dlp + 2 * dz.max(1).values + 4 * U24 * (lsm.gather(1, tok.long()[:, None])[:, 0].abs() + z.abs().max(1).values)
        nb = tok != blank
        if nb.any():
            nst, nx, ndx = P.step(tok, st)
            st = tuple(torch.where(nb[None, :, None], a, b) for a, b in zip(nst, st))
            dec_x, ddec = torch.where(nb[:, None], nx, dec_x), torch.where(nb[:, None], ndx, ddec)
    return st, dec_x, ddec, items, und, R * n_out, lp, dlp


@pytest.mark.parametrize("cfg,S,n,chunks", [("large", 130, 2, 12), ("ragged", 67, 4, 12)])
def test_stream_engine_chunks_teacher_forced(cfg, S, n, chunks):
    """Each chunk against fp64 recomputed from the device's own inputs: the input LN, every encoder layer's LSTM steps
    (x from the device's buffer of the layer below, h_{t-1} from its own y), the cell state recursed over the chunk's
    steps, the LN (+ residual), the time reduction, the projection, the joint, the tokens and the predictor state.
    large: E6D2_LARGE dims, weights x 2, S = 130 (three row tiles), one output frame per chunk; ragged: S = 67, n = 4,
    two output frames.  Then the same chunks with max_ctas in {1, 3, 17} give the same bits."""
    from edgedict_b200.stream_engine import StreamEngine
    model = _scaled(LARGE if cfg == "large" else RAGGED, seed=10)
    F = model.encoder.norm.weight.shape[0]
    g = torch.Generator().manual_seed(5)
    xs = torch.randn(chunks, S, n, F, generator=g).to(DEV)
    eng = StreamEngine(model, S, n)
    P = _Pred(model)
    sd = P.sd
    enc = model.encoder
    L, red = len(enc.lstm.lstms), enc.lstm.time_reductions
    worst_items = {}
    und = rows = emitted = 0
    states, hists = [], []
    for ci in range(chunks):
        st0 = eng.state()
        states.append(st0)
        hist = eng.step(xs[ci]).clone()
        hists.append(hist)
        items = []
        a0r, da0 = ln_ref(xs[ci].reshape(S * n, F), sd["encoder.norm.weight"], sd["encoder.norm.bias"])
        items.append(("a0", eng.a0.view(S * n, F), a0r, da0))
        X, ni, bi = eng.a0, n, 0
        for i in range(L):
            yL, zL = eng._bufs[bi], eng._bufs[bi + 1]
            bi += 2
            g_ = lambda nm: sd["encoder.lstm.lstms.%d.%s_l0" % (i, nm)]
            c, dc = st0["enc_c"][i].double(), None
            for t in range(ni):
                hin = st0["enc_h"][i] if t == 0 else yL[:, t - 1]
                c, dc, yr, dy = lstm_ref(X[:, t], g_("weight_ih"), hin, g_("weight_hh"), g_("bias_ih"), g_("bias_hh"), c,
                                         dc=dc)
                items.append(("L%d y t%d" % (i, t), yL[:, t], yr, dy))
            items.append(("L%d c" % i, eng.enc_c[i], c, dc))
            assert torch.equal(_bits(eng.enc_h[i]), _bits(yL[:, ni - 1])), "enc_h is not the last step's y"
            H = yL.shape[2]
            z32 = (yL + X) if i > 0 else yL
            zr, dz = ln_ref(z32.reshape(-1, H), sd["encoder.lstm.projs.%d.0.weight" % i],
                            sd["encoder.lstm.projs.%d.0.bias" % i])
            items.append(("L%d ln" % i, zL.reshape(-1, H), zr, dz))
            X = zL
            if i in red:
                zp = eng._bufs[bi]
                bi += 1
                assert torch.equal(_bits(zp), _bits(0.5 * (zL[:, 0::2] + zL[:, 1::2]))), "PAIR"
                X, ni = zp, ni // 2
        er, de = linear_ref(X.reshape(S * ni, -1), sd["encoder.proj.weight"], sd["encoder.proj.bias"])
        items.append(("enc_out", eng.enc_out.reshape(S * ni, -1), er, de))
        h0, c0, x0 = st0["dec_h"].double(), st0["dec_c"].double(), st0["dec_x"].double()
        st = (h0, torch.zeros_like(h0), c0, torch.zeros_like(c0))
        fin, dx, ddx, fit, u, r, _, _ = _frames(P, eng.enc_out, hist, st, x0, torch.zeros_like(x0), eng.blank, eng.unk,
                                                eng.hidden, eng.logits)
        items += fit
        und, rows, emitted = und + sum(u), rows + r, emitted + int((hist != eng.blank).sum())
        items += [("dec_h", eng.dec_h, fin[0], fin[1]), ("dec_c", eng.dec_c, fin[2], fin[3]),
                  ("dec_x", eng.dec_x, dx, ddx)]
        quiet = (hist == eng.blank).all(1)                    # streams whose predictor never stepped: bitwise unchanged
        for k in ("dec_h", "dec_c"):
            assert torch.equal(_bits(getattr(eng, k)[:, quiet]), _bits(st0[k][:, quiet])), k + " of a blank stream"
        assert torch.equal(_bits(eng.dec_x[quiet]), _bits(st0["dec_x"][quiet])), "dec_x of a blank stream"
        assert torch.equal(eng.tok, hist[:, -1])
        for label, got, ref, bar in items:                    # keep the worst chunk of every item for the report
            ratio = float(((got.double() - ref).abs() / (bar + 2.0 ** -120)).max())
            if label not in worst_items or ratio > worst_items[label][0]:
                worst_items[label] = (ratio, got.clone(), ref, bar)
    _report("stream %s S=%d n=%d" % (cfg, S, n), [(k, v[1], v[2], v[3]) for k, v in worst_items.items()])
    print("  stream %s: %d of %d frame tokens emitted, %d inside the logits' bar" % (cfg, emitted, rows, und))
    assert emitted > rows // 20 and und <= rows // 50
    # max_ctas invariance: the same chunks from the same states
    for mc in CTAS[1:]:
        e2 = StreamEngine(model, S, n, max_ctas=mc)
        for ci in (0, chunks - 1):
            e2.load_state(states[ci])
            h2 = e2.step(xs[ci])
            assert torch.equal(h2, hists[ci]), "max_ctas=%d chunk %d tokens" % (mc, ci)
            e1 = StreamEngine(model, S, n, state=states[ci])
            e1.step(xs[ci])
            for k in StreamEngine.STATE:
                assert torch.equal(_bits(getattr(e2, k)), _bits(getattr(e1, k))), "max_ctas=%d chunk %d %s" % (mc, ci, k)
            for a, b in zip(e2._bufs + [e2.enc_out, e2.logits], e1._bufs + [e1.enc_out, e1.logits]):
                assert torch.equal(_bits(a), _bits(b)), "max_ctas=%d chunk %d buffers" % (mc, ci)


def test_greedy_engine_teacher_forced():
    """GreedyEngine on B = 70 (two row tiles), T' = 6: the priming step and every frame in fp64 from the device's
    encoder output with the predictor's bars propagated from frame to frame; the tokens, log p, the last frame's hidden
    and logits, and the final predictor state.  Then max_ctas in {1, 3, 17} give the same bits."""
    from edgedict_b200.rnnt.tokenizer import BOS
    from edgedict_b200.stream_engine import GreedyEngine
    model = _scaled(RAGGED, seed=3)
    B, T = 70, 6
    E = model.encoder.proj.weight.shape[0]
    g = torch.Generator().manual_seed(9)
    h_enc = (torch.randn(B, T, E, generator=g) * 2).to(DEV)
    eng = GreedyEngine(model, B, T)
    hist, logp = (a.clone() for a in eng.run(h_enc))
    P = _Pred(model)
    Ld, Hd = model.decoder.lstm.num_layers, model.decoder.lstm.hidden_size
    z = torch.zeros(Ld, B, Hd, dtype=f64, device=DEV)
    st, dx, ddx = P.step(torch.full((B,), BOS, dtype=i32, device=DEV), (z, z, z, z))
    fin, dx, ddx, items, und, rows, lp, dlp = _frames(P, h_enc, hist, st, dx, ddx, eng.blank, -1, eng.hidden, eng.logits)
    emitted = int((hist != eng.blank).sum())
    _report("greedy B=%d T=%d" % (B, T), items + [
        ("logp", logp, lp, dlp + U24 * T * lp.abs() + T * 2.0 ** -20),
        ("dec_h", eng.dec_h, fin[0], fin[1]), ("dec_c", eng.dec_c, fin[2], fin[3]), ("dec_x", eng.dec_x, dx, ddx)])
    # the predictor's bars are propagated worst-case from frame to frame, so later frames leave more tokens undecided
    print("  greedy: %d of %d tokens emitted, inside the logits' bar per frame: %s" % (emitted, rows, und))
    assert emitted > rows // 20 and und[0] + und[1] <= B // 25
    for mc in CTAS[1:]:
        e2 = GreedyEngine(model, B, T, max_ctas=mc)
        h2, l2 = e2.run(h_enc)
        assert torch.equal(h2, hist) and torch.equal(_bits(l2), _bits(logp)), "max_ctas=%d" % mc
        for k in ("dec_h", "dec_c", "dec_x", "hidden", "logits"):
            assert torch.equal(_bits(getattr(e2, k)), _bits(getattr(eng, k))), "max_ctas=%d %s" % (mc, k)
