"""GPU parity of the individual kernels (through the C-ABI) against plain torch fp32/fp64 CPU
references of the same op and the oracle's LSTM restatement."""
import numpy as np
import pytest
import torch

from tests.util import rel_err

pytestmark = pytest.mark.gpu


def _r(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (65, 70, 33), (128, 64, 16), (200, 1024, 320), (37, 5, 130)])
def test_gemm_f32_all_layouts(M, N, K):
    from edgedict_b200 import ops
    x, w, dy = _r(M, K, seed=1), _r(N, K, seed=2), _r(M, N, seed=3)
    b = _r(N, seed=4)
    xd, wd, dyd, bd = x.cuda(), w.cuda(), dy.cuda(), b.cuda()
    assert rel_err(ops.mm_nt(xd, wd, bd).cpu(), x.double() @ w.double().t() + b.double()) < 1e-5
    assert rel_err(ops.mm_nn(dyd, wd).cpu(), dy.double() @ w.double()) < 1e-5
    assert rel_err(ops.mm_tn(dyd, xd).cpu(), dy.double().t() @ x.double()) < 1e-5
    # accumulate + strided (column-slice) weight view
    if K >= 4:
        k0 = K // 2
        y = ops.mm_nt(xd[:, :k0].contiguous(), wd[:, :k0], None)
        assert rel_err(y.cpu(), x[:, :k0].double() @ w[:, :k0].double().t()) < 1e-5
    acc = torch.ones(N, K, device="cuda")
    ops.mm_tn(dyd, xd, out=acc, accumulate=True)
    assert rel_err(acc.cpu(), 1 + dy.double().t() @ x.double()) < 1e-5


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 640), (300, 136, 72), (1000, 1024, 240), (129, 8, 8)])
def test_gemm_bf16_tcgen05_all_layouts(M, N, K):
    """bf16 operands (rounded identically on both sides), fp32 accumulation: error is summation
    order only."""
    from edgedict_b200 import ops
    x, w, dy = _r(M, K, seed=1).bfloat16(), _r(N, K, seed=2).bfloat16(), _r(M, N, seed=3).bfloat16()
    b = _r(N, seed=4)
    xd, wd, dyd, bd = x.cuda(), w.cuda(), dy.cuda(), b.cuda()
    ref = x.double() @ w.double().t() + b.double()
    y = ops.gemm_bf16(xd, 0, wd, 0, M, N, K, bias=bd)
    assert rel_err(y.cpu(), ref) < 2e-5
    y16 = ops.gemm_bf16(xd, 0, wd, 0, M, N, K, bias=bd, out_bf16=True)
    assert y16.dtype == torch.bfloat16 and rel_err(y16.float().cpu(), ref) < 1e-2
    if K % 8 == 0 and N % 8 == 0:
        dx = ops.gemm_bf16(dyd, 0, wd, 1, M, K, N)                        # dy[M,N] @ w[N,K]
        assert rel_err(dx.cpu(), dy.double() @ w.double()) < 2e-5
    if N % 8 == 0 and K % 8 == 0:
        dw = ops.gemm_bf16(dyd, 1, xd, 1, N, K, M)                        # dy^T @ x, both MN-major
        assert rel_err(dw.cpu(), dy.double().t() @ x.double()) < 2e-5
        acc = torch.full((N, K), 2.0, device="cuda")
        ops.gemm_bf16(dyd, 1, xd, 1, N, K, M, out=acc, accumulate=True)
        assert rel_err(acc.cpu(), 2 + dy.double().t() @ x.double()) < 2e-5
    if M % 8 == 0:
        # A MN-major, B K-major:  (x^T)^T ... C[K? ] -- use A = x^T stored [K, M]
        xt = x.t().contiguous().cuda()                                    # [K, M]: contraction K rows
        y2 = ops.gemm_bf16(xt, 1, wd, 0, M, N, K)
        assert rel_err(y2.cpu(), x.double() @ w.double().t()) < 2e-5


def test_gemm_bf16_persistent_many_tiles():
    from edgedict_b200 import ops
    M, N, K = 128 * 40 + 17, 1024, 640                                   # > 132 tiles (one per SM), ragged M
    x, w = _r(M, K, seed=7).bfloat16(), _r(N, K, seed=8).bfloat16()
    y = ops.gemm_bf16(x.cuda(), 0, w.cuda(), 0, M, N, K)
    ref = x.float() @ w.float().t()
    assert rel_err(y.cpu(), ref) < 2e-5


def test_gemm_bf16_wide_tiles_overhanging_the_last_columns():
    """N = 256 k + 128 with many row blocks selects 128x256 tiles whose last column tile hangs over N (the joint's
    d-hidden GEMM, N = 640): out-of-range columns are never stored, in-range chunks keep the vector path."""
    from edgedict_b200 import ops
    M, N, K = 128 * 4 * 148 + 77, 384, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    dy = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w_nt = torch.randn(N, K, device="cuda", generator=g).bfloat16()          # B K-major
    w_nn = torch.randn(K, N, device="cuda", generator=g).bfloat16()          # B MN-major
    guard = torch.full((M + 1, N), 7.0, device="cuda").bfloat16()
    y = ops.gemm_bf16(dy, 0, w_nt, 0, M, N, K, out=guard[:M])
    ref = dy.float() @ w_nt.float().t()
    assert rel_err(y.float().cpu(), ref.cpu()) < 1e-2 and (guard[M] == 7.0).all()
    y2 = ops.gemm_bf16(dy, 0, w_nn, 1, M, N, K)                              # fp32 out
    assert rel_err(y2.cpu(), (dy.float() @ w_nn.float()).cpu()) < 2e-5
    hid = torch.tanh(torch.randn(M, N, device="cuda", generator=g)).bfloat16()
    y3 = ops.gemm_bf16_dtanh(dy, w_nn, True, hid, M, N, K)
    assert rel_err(y3.float().cpu(), ((dy.float() @ w_nn.float()) * (1 - hid.float() ** 2)).cpu()) < 1e-2


@pytest.mark.parametrize("M,N,K", [(1024, 640, 64 * 700 + 24), (320, 384, 64 * 97), (128, 128, 64 * 361)])
def test_gemm_bf16_split_k_weight_gradients(M, N, K):
    """fp32-output products with few output tiles and a long contraction split K across CTAs: each split's partial tile
    goes to the workspace sized by eb_gemm_bf16_partials and splitk_reduce_kernel adds the splits in order.  Both operands
    MN-major (the weight-gradient layout), with / without bias and accumulate, against fp64; a shrunk workspace (fewer
    splits, and for the last shape 20 splits of 19 k-blocks over 361, so that the last split is empty) and no workspace
    (no split) give the same product; repeated launches give the same bits."""
    from edgedict_b200 import ops
    from edgedict_b200._lib import lib, check
    g = torch.Generator(device="cuda").manual_seed(M + K)
    a = (torch.randn(K, M, device="cuda", generator=g) * 0.1).bfloat16()       # A^T stored [K, M]
    b = torch.randn(K, N, device="cuda", generator=g).bfloat16()               # B stored [K, N]
    bias = torch.randn(N, device="cuda", generator=g)
    want = a.double().t() @ b.double()
    planned = int(lib().eb_gemm_bf16_partials(1, 0, 0, M, N, K, 0))
    assert planned >= 2 * M * N, "this shape must take the split-K path"
    y = ops.gemm_bf16(a, 1, b, 1, M, N, K)
    assert rel_err(y.cpu(), want.cpu()) < 2e-5
    assert torch.equal(ops.gemm_bf16(a, 1, b, 1, M, N, K), y)
    yb = ops.gemm_bf16(a, 1, b, 1, M, N, K, bias=bias)
    assert rel_err(yb.cpu(), (want + bias.double()).cpu()) < 2e-5
    base = torch.randn(M, N, device="cuda", generator=g)
    acc = base.clone()
    ops.gemm_bf16(a, 1, b, 1, M, N, K, out=acc, accumulate=True)
    assert rel_err(acc.cpu(), (want + base.double()).cpu()) < 2e-5

    def with_ws(floats):
        out = torch.full((M, N), 7.0, device="cuda")
        ws = torch.empty(max(floats, 1), device="cuda")
        check(lib().eb_gemm_bf16_ex(a.data_ptr(), 1, b.data_ptr(), 1, out.data_ptr(), 0, bias.data_ptr(), 0, M, N, K, 0,
                                    ws.data_ptr() if floats else None, floats, None), "eb_gemm_bf16_ex")
        torch.cuda.synchronize()
        return out
    shrunk = 20 if K == 64 * 361 else 2
    assert planned >= shrunk * M * N
    # fewer splits = longer fp32 accumulation chains per element (no workspace: one chain over all of K, up to 45 k
    # terms): the rounding grows with the chain, so chains beyond 16 k terms get a wider bar
    for splits, floats in ((shrunk, shrunk * M * N), (1, 0)):
        bar = 2e-5 if K // splits <= 16384 else 1e-4
        assert rel_err(with_ws(floats).cpu(), (want + bias.double()).cpu()) < bar, splits


@pytest.mark.parametrize("rows,H,res", [(7, 12, False), (33, 240, False), (64, 320, True), (19, 1024, True), (5, 1500, True),
                                        (300, 256, False), (2000, 512, True), (4100, 1024, False), (3, 128, True)])
def test_layernorm_fwd_bwd(rows, H, res):
    from edgedict_b200 import ops
    x, r = _r(rows, H, seed=1), (_r(rows, H, seed=2) if res else None)
    g, b, dy = _r(H, seed=3) + 1, _r(H, seed=4), _r(rows, H, seed=5)
    xt = x.double().requires_grad_(True)
    rt = r.double().requires_grad_(True) if res else None
    gt, bt = g.double().requires_grad_(True), b.double().requires_grad_(True)
    ref = torch.nn.functional.layer_norm(xt + rt if res else xt, (H,), gt, bt, 1e-5)
    ref.backward(dy.double())
    y, _, mean, rstd = ops.layernorm_fwd(x.cuda(), r.cuda() if res else None, g.cuda(), b.cuda())
    assert rel_err(y.cpu(), ref.detach()) < 1e-5
    dz, dg, db = ops.layernorm_bwd(dy.cuda(), x.cuda(), r.cuda() if res else None, g.cuda(), mean, rstd)
    assert rel_err(dz.cpu(), xt.grad) < 1e-5
    assert rel_err(dg.cpu(), gt.grad) < 1e-5 and rel_err(db.cpu(), bt.grad) < 1e-5


@pytest.mark.parametrize("T", [1, 2, 7, 10])
def test_time_reduction(T):
    from edgedict_b200 import ops
    from oracle import model_torch as mt
    x = _r(3, T, 5, seed=T).requires_grad_(True)
    ref = mt.time_reduction(x)
    dy = _r(*ref.shape, seed=9)
    ref.backward(dy)
    y, _ = ops.time_reduce_fwd(x.detach().cuda())
    assert torch.equal(y.cpu(), ref.detach())
    assert torch.allclose(ops.time_reduce_bwd(dy.cuda(), T).cpu(), x.grad)


def test_embedding_fwd_bwd():
    from edgedict_b200 import ops
    W = _r(20, 6, seed=1)
    ids = torch.tensor([[4, 1, 7], [1, 19, 4]], dtype=torch.int32)
    for prep in (True, False):
        full = torch.cat([torch.full((2, 1), 2), ids.long()], 1) if prep else ids.long()
        Wt = W.clone().requires_grad_(True)
        ref = torch.nn.functional.embedding(full, Wt, padding_idx=1)
        dout = _r(*ref.shape, seed=3)
        ref.backward(dout)
        out = ops.embedding_fwd(ids.cuda(), W.cuda(), prep, 2)
        assert torch.equal(out.cpu(), ref.detach())
        dW = ops.embedding_bwd(ids.cuda(), dout.cuda(), 20, prep, 2, 1)
        assert torch.allclose(dW.cpu(), Wt.grad, atol=1e-6)
    out = ops.embedding_fwd(torch.zeros(3, 0, dtype=torch.int64).cuda(), W.cuda(), True, 2)     # greedy priming
    assert out.shape == (3, 1, 6) and torch.equal(out.cpu(), W[2].expand(3, 1, 6))


@pytest.mark.parametrize("use16", [False, True])
def test_joint_hidden_fwd_bwd(use16):
    from edgedict_b200 import ops
    B, T, U, J = 2, 5, 4, 24
    ep, dp = _r(B, T, J, seed=1).requires_grad_(True), _r(B, U, J, seed=2).requires_grad_(True)
    ref = torch.tanh(ep[:, :, None, :] + dp[:, None, :, :])
    dh = _r(B, T, U, J, seed=3)
    ref.backward(dh)
    hid = ops.joint_hidden_fwd(ep.detach().cuda(), dp.detach().cuda(), use16)
    tol = 1e-2 if use16 else 1e-6
    assert rel_err(hid.float().cpu(), ref.detach()) < tol
    dhd = dh.cuda().bfloat16() if use16 else dh.cuda().clone()
    dep, ddp = ops.joint_hidden_bwd(dhd, hid)
    assert rel_err(dep.cpu(), ep.grad) < (3e-2 if use16 else 1e-5)
    assert rel_err(ddp.cpu(), dp.grad) < (3e-2 if use16 else 1e-5)


def test_colsum_cast_transpose_adam():
    from edgedict_b200 import ops
    from edgedict_b200._lib import lib, check
    x = _r(1000, 37, seed=1)
    assert rel_err(ops.colsum(x.cuda()).cpu(), x.double().sum(0)) < 1e-5
    assert rel_err(ops.colsum(x.cuda().bfloat16()).cpu(), x.bfloat16().double().sum(0)) < 1e-5
    v = _r(1003, seed=2)
    assert torch.equal(ops.cast_bf16(v.cuda()).cpu(), v.bfloat16())
    y = torch.empty(37, 1000, dtype=torch.bfloat16, device="cuda")
    check(lib().eb_transpose_to_bf16(x.cuda().data_ptr(), 0, y.data_ptr(), 1000, 37, None), "transpose")
    assert torch.equal(y.cpu(), x.t().bfloat16())
    # Adam: three steps against torch.optim.Adam
    p = _r(777, seed=3)
    pt = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=1e-2, betas=(0.9, 0.999), eps=1e-8)
    pd, m, vv = p.cuda(), torch.zeros(777, device="cuda"), torch.zeros(777, device="cuda")
    for step in range(1, 4):
        g = _r(777, seed=10 + step)
        pt.grad = g.clone()
        opt.step()
        ops.adam_step(pd, g.cuda(), m, vv, 1e-2, 0.9, 0.999, 1e-8, 0.0, step)
    assert rel_err(pd.cpu(), pt.detach()) < 1e-5


@pytest.mark.parametrize("B,T,I,H", [(2, 5, 6, 8), (3, 9, 12, 24), (33, 4, 8, 16), (2, 12, 64, 320), (4, 6, 32, 1024)])
def test_lstm_layer_fwd_bwd_vs_oracle(B, T, I, H):
    """Persistent LSTM kernels vs the oracle's explicit cell loop (fp64 on CPU), including
    non-zero initial states and gradients flowing into the final states."""
    from edgedict_b200 import functional as Fn
    from oracle import model_torch as mt
    k = 1.0 / np.sqrt(H)
    w_ih, w_hh = (torch.rand(4 * H, I) * 2 - 1) * k, (torch.rand(4 * H, H) * 2 - 1) * k
    b_ih, b_hh = (torch.rand(4 * H) * 2 - 1) * k, (torch.rand(4 * H) * 2 - 1) * k
    x, h0, c0 = _r(B, T, I, seed=1), _r(B, H, seed=2, scale=0.5), _r(B, H, seed=3, scale=0.5)
    dy, dh, dc = _r(B, T, H, seed=4), _r(B, H, seed=5), _r(B, H, seed=6)
    ref_in = [t.double().requires_grad_(True) for t in (x, h0, c0, w_ih, w_hh, b_ih, b_hh)]
    y, hT, cT = mt.lstm_layer(*ref_in, fast=False)
    ((y * dy.double()).sum() + (hT * dh.double()).sum() + (cT * dc.double()).sum()).backward()
    dev_in = [t.clone().cuda().requires_grad_(True) for t in (x, h0, c0, w_ih, w_hh, b_ih, b_hh)]
    yd, hTd, cTd = Fn.LSTMLayer.apply(*dev_in, "fp32")
    assert rel_err(yd.detach().cpu(), y.detach()) < 1e-5
    assert rel_err(hTd.detach().cpu(), hT.detach()) < 1e-5 and rel_err(cTd.detach().cpu(), cT.detach()) < 1e-5
    ((yd * dy.cuda()).sum() + (hTd * dh.cuda()).sum() + (cTd * dc.cuda()).sum()).backward()
    for name, a, r in zip("x h0 c0 w_ih w_hh b_ih b_hh".split(), dev_in, ref_in):
        assert rel_err(a.grad.cpu(), r.grad) < 2e-5, name
    # zero initial state path (h0 = c0 = None) as in training
    y2, _, _ = Fn.LSTMLayer.apply(dev_in[0].detach(), None, None, *[t.detach() for t in dev_in[3:]], "fp32")
    y2r, _, _ = mt.lstm_layer(x.double(), torch.zeros(B, H).double(), torch.zeros(B, H).double(),
                              *[t.detach() for t in ref_in[3:]])
    assert rel_err(y2.cpu(), y2r) < 1e-5


@pytest.mark.parametrize("B,T,I,H", [(4, 6, 32, 64), (32, 9, 64, 256), (7, 5, 24, 320), (32, 4, 64, 1024), (40, 3, 16, 128)])
def test_lstm_tensor_core_layer_vs_oracle(B, T, I, H):
    """bf16-mode persistent LSTM (mma.sync, weights resident in registers, cluster/DSMEM reduce in
    BPTT) vs the fp64 oracle evaluated with the SAME bf16-rounded weights.  Remaining difference:
    h_{t-1} and dG_t are exchanged in bf16 (documented tolerance 2e-2 / 5e-2)."""
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    from oracle import model_torch as mt
    assert ops.lstm_tc_supported(B, H)
    k = 1.0 / np.sqrt(H)
    rb = lambda t: t.bfloat16().float()
    w_ih, w_hh = rb((torch.rand(4 * H, I) * 2 - 1) * k), rb((torch.rand(4 * H, H) * 2 - 1) * k)
    b_ih, b_hh = (torch.rand(4 * H) * 2 - 1) * k, (torch.rand(4 * H) * 2 - 1) * k
    x, h0, c0 = rb(_r(B, T, I, seed=1)), _r(B, H, seed=2, scale=0.5), _r(B, H, seed=3, scale=0.5)
    dy, dh, dc = _r(B, T, H, seed=4), _r(B, H, seed=5), _r(B, H, seed=6)
    ref_in = [t.double().requires_grad_(True) for t in (x, h0, c0, w_ih, w_hh, b_ih, b_hh)]
    y, hT, cT = mt.lstm_layer(*ref_in, fast=False)
    ((y * dy.double()).sum() + (hT * dh.double()).sum() + (cT * dc.double()).sum()).backward()
    dev_in = [t.clone().cuda().requires_grad_(True) for t in (x, h0, c0, w_ih, w_hh, b_ih, b_hh)]
    yd, hTd, cTd = Fn.LSTMLayer.apply(*dev_in, "bf16")
    assert rel_err(yd.detach().cpu(), y.detach()) < 2e-2
    assert rel_err(hTd.detach().cpu(), hT.detach()) < 2e-2 and rel_err(cTd.detach().cpu(), cT.detach()) < 2e-2
    ((yd * dy.cuda()).sum() + (hTd * dh.cuda()).sum() + (cTd * dc.cuda()).sum()).backward()
    for name, a, r in zip("x h0 c0 w_ih w_hh b_ih b_hh".split(), dev_in, ref_in):
        assert rel_err(a.grad.cpu(), r.grad) < 5e-2, name


@pytest.mark.parametrize("B,H,lens", [(32, 256, [5, 5, 3]), (7, 1024, [4, 2]), (40, 128, [3, 3, 3, 1]), (32, 512, [6])])
def test_lstm_bptt_one_launch_over_chunk_major_buffers(B, H, lens):
    """eb_lstm_tc_bwd_chunks (one launch walking the wavefront's chunk-major buffers) == eb_lstm_tc_bwd once per chunk with
    the (dh, dc) carry, bit for bit: same kernel, same arithmetic, only the row addressing differs.  B = 40 crosses the
    32-row batch tile."""
    from edgedict_b200 import ops
    from edgedict_b200.functional import _Chunks
    g = torch.Generator(device="cuda").manual_seed(3)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    k = _Chunks(B, lens)
    T = sum(lens)
    whhT16 = (rn(H, 4 * H) / np.sqrt(H)).bfloat16()
    gates = torch.sigmoid(rn(k.rows, 4 * H))
    gates[:, 2 * H:3 * H] = torch.tanh(rn(k.rows, H))                  # the cell candidate is a tanh
    cseq, dy = rn(k.rows, H), rn(k.rows, H)
    one = torch.full((k.rows + 1, 4 * H), 7.0, device="cuda").bfloat16()
    _, dh1, dc1 = ops.lstm_tc_bwd_chunks(dy, gates, cseq, whhT16, lens, B, one[:k.rows])
    ref = torch.empty(k.rows, 4 * H, device="cuda").bfloat16()
    dh = dc = None
    for c in range(len(lens) - 1, -1, -1):
        c_prev = k.blk(cseq, c - 1)[:, -1].contiguous() if c else None
        _, dh, dc = ops.lstm_tc_bwd(k.blk(dy, c), k.blk(gates, c), k.blk(cseq, c), c_prev, whhT16, dh, dc, out=k.blk(ref, c))
    torch.cuda.synchronize()
    assert torch.equal(one[:k.rows], ref) and (one[k.rows] == 7.0).all()
    assert torch.equal(dh1, dh) and torch.equal(dc1, dc)


@pytest.mark.parametrize("B,T,U,J", [(3, 70, 9, 640), (2, 33, 129, 72), (5, 32, 4, 128), (1, 250, 17, 320)])
def test_joint_dpre_reduce_shapes(B, T, U, J):
    """eb_joint_dpre_reduce (dep = sum over u, ddp = sum over t of the bf16 d-pre-activation) vs torch in fp64 at shapes
    with many frames / ragged column counts."""
    from edgedict_b200 import ops
    d = _r(B, T, U, J, seed=21).bfloat16().cuda()
    dep, ddp = ops.joint_dpre_reduce(d)
    ref = d.double().cpu()
    assert rel_err(dep.cpu(), ref.sum(2)) < 1e-5
    assert rel_err(ddp.cpu(), ref.sum(1)) < 1e-5


@pytest.mark.parametrize("M,N,K", [(300, 128, 64), (1000, 640, 256), (257, 72, 96)])
def test_gemm_dtanh_epilogue_and_dpre_reductions(M, N, K):
    """eb_gemm_bf16_dtanh: (A B) * (1 - hid^2) in the GEMM epilogue (full and edge tiles), then eb_joint_dpre_reduce."""
    from edgedict_b200 import ops
    a = (_r(M, K, seed=1) / 4).bfloat16().cuda()
    w = (_r(K, N, seed=2) / 4).bfloat16().cuda()
    hid = torch.tanh(_r(M, N, seed=3)).bfloat16().cuda()
    got = ops.gemm_bf16_dtanh(a, w, True, hid, M, N, K).float().cpu()
    ref = (a.float().cpu() @ w.float().cpu()) * (1 - hid.float().cpu() ** 2)
    assert rel_err(got, ref) < 1e-2                       # bf16 output rounding
    if N % 8 == 0 and M % 4 == 0:
        B, T = 2, 2
        U = M // 4
        d4 = got.bfloat16().cuda().view(B, T, U, N)
        dep, ddp = ops.joint_dpre_reduce(d4)
        assert rel_err(dep.cpu(), d4.float().cpu().sum(2)) < 1e-5
        assert rel_err(ddp.cpu(), d4.float().cpu().sum(1)) < 1e-5


@pytest.mark.parametrize("B,T,H", [(32, 9, 256), (5, 7, 512), (40, 4, 768), (32, 6, 1024)])
def test_lstm_c4_cluster_kernels_vs_oracle(B, T, H):
    """csrc/lstm_c4.cu directly (cluster / wgmma forward with both save layouts, wgmma BPTT) against an explicit fp64
    cell loop on the same bf16-rounded recurrent weights; remaining difference: h_{t-1} / dG_t exchanged in bf16 and
    the saved gates kept in bf16 (documented tolerances as for lstm_tc: 2e-2 forward, 5e-2 gradients)."""
    from edgedict_b200 import ops
    if not ops.lstm_c4_supported(B, H):
        pytest.skip("clusters of the lstm_c4 kernels are not co-resident on this GPU")
    torch.manual_seed(B + T)
    k = 1.0 / np.sqrt(H)
    w = ((torch.rand(4 * H, H) * 2 - 1) * k).bfloat16()
    xg = torch.randn(B, T, 4 * H)
    h0, c0 = torch.randn(B, H) * 0.5, torch.randn(B, H) * 0.5
    dy, dhT, dcT = torch.randn(B, T, H), torch.randn(B, H), torch.randn(B, H)
    # fp64 reference with autograd
    xr, hr, cr = xg.double().requires_grad_(True), h0.double().requires_grad_(True), c0.double().requires_grad_(True)
    wd = w.double()
    h, c, ys = hr, cr, []
    for t in range(T):
        g = xr[:, t] + h @ wd.t()
        i, f, gg, o = g[:, :H].sigmoid(), g[:, H:2 * H].sigmoid(), g[:, 2 * H:3 * H].tanh(), g[:, 3 * H:].sigmoid()
        c = f * c + i * gg
        h = o * c.tanh()
        ys.append(h)
    y = torch.stack(ys, 1)
    ((y * dy.double()).sum() + (h * dhT.double()).sum() + (c * dcT.double()).sum()).backward()
    dev = "cuda"
    wg, whT = w.to(dev), w.t().contiguous().to(dev)
    y1, hp, hT, cT, gs, cs = ops.lstm_c4_fwd(xg.to(dev), wg, h0.to(dev), c0.to(dev), True)
    assert rel_err(y1.cpu(), y.detach()) < 2e-2 and rel_err(hT.cpu(), h.detach()) < 2e-2 and rel_err(cT.cpu(), c.detach()) < 2e-2
    want_hp = torch.cat([h0[:, None], y.detach().float()[:, :-1]], 1)
    assert rel_err(hp.float().cpu(), want_hp) < 2e-2
    # standard-layout saves feed the mma.sync BPTT kernel, the CTA-private ones the wgmma BPTT kernel
    y2, _, _, _, gstd, cstd = ops.lstm_c4_fwd(xg.to(dev), wg, h0.to(dev), c0.to(dev), True, std_saves=True)
    assert torch.equal(y1, y2)
    for name, (dg, dh0, dc0) in (("tc_bwd", ops.lstm_tc_bwd(dy.to(dev), gstd, cstd, c0.to(dev), whT, dhT.to(dev), dcT.to(dev))),
                                 ("c4_bwd", ops.lstm_c4_bwd(dy.to(dev), gs, cs, c0.to(dev), whT, dhT.to(dev), dcT.to(dev)))):
        assert rel_err(dg.float().cpu(), xr.grad) < 5e-2, name
        assert rel_err(dh0.cpu(), hr.grad) < 5e-2 and rel_err(dc0.cpu(), cr.grad) < 5e-2, name
