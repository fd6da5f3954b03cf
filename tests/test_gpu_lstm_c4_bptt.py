"""eb_lstm_c4_bwd_chunks, the K-split wgmma BPTT kernel in clusters of 16, against an fp64 cell loop, against
eb_lstm_tc_bwd_chunks on identical inputs, and against itself (the same bits on every launch)."""
import numpy as np
import pytest
import torch

from tests.util import rel_err

pytestmark = pytest.mark.gpu


def _need(H):
    from edgedict_b200 import ops
    if not ops.lstm_c4_bwd_chunks_supported(H):
        pytest.skip("clusters of 16 of the lstm_c4 BPTT kernel are not co-resident on this GPU")


@pytest.mark.parametrize("H", [256, 512, 1024])
@pytest.mark.parametrize("B,lens", [(5, [7]), (32, [4, 3, 2]), (40, [2, 5, 1, 3])])
def test_lstm_c4_bwd_chunks_vs_fp64_cell_loop(B, lens, H):
    """Forward through eb_lstm_c4_fwd (standard-layout fp32 saves), the saves scattered into the wavefront's chunk-major
    layout, BPTT through eb_lstm_c4_bwd_chunks with c0 / dh_T / dc_T, against autograd on an fp64 cell loop with the same
    bf16-rounded W_hh.  Tolerance as for the other bf16 BPTT kernels (dG_t is exchanged in bf16).  B = 40 crosses the
    32-row batch tile."""
    from edgedict_b200 import ops
    from edgedict_b200.functional import _Chunks
    _need(H)
    T = sum(lens)
    torch.manual_seed(B + T + H)
    k = 1.0 / np.sqrt(H)
    w = ((torch.rand(4 * H, H) * 2 - 1) * k).bfloat16()
    xg = torch.randn(B, T, 4 * H)
    h0, c0 = torch.randn(B, H) * 0.5, torch.randn(B, H) * 0.5
    dy, dhT, dcT = torch.randn(B, T, H), torch.randn(B, H), torch.randn(B, H)
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
    _, _, _, _, gstd, cstd = ops.lstm_c4_fwd(xg.to(dev), w.to(dev), h0.to(dev), c0.to(dev), True, std_saves=True)
    ck = _Chunks(B, lens)
    dg = torch.empty(ck.rows, 4 * H, dtype=torch.bfloat16, device=dev)
    _, dh0, dc0 = ops.lstm_c4_bwd_chunks(ck.scatter(dy.to(dev)), ck.scatter(gstd), ck.scatter(cstd),
                                         w.t().contiguous().to(dev), lens, B, dg, c0.to(dev), dhT.to(dev), dcT.to(dev))
    assert rel_err(ck.gather(dg).float().cpu(), xr.grad) < 5e-2
    assert rel_err(dh0.cpu(), hr.grad) < 5e-2 and rel_err(dc0.cpu(), cr.grad) < 5e-2


@pytest.mark.parametrize("B,H,lens", [(32, 1024, [40, 40, 37]), (7, 256, [9, 4]), (40, 512, [6, 6, 6, 6, 6, 5, 5, 5])])
def test_lstm_c4_bwd_chunks_matches_tc_kernel_and_itself(B, H, lens):
    """Same inputs through eb_lstm_tc_bwd_chunks: only the summation order of dh = W_hh^T dG differs, so the two agree
    within bf16 rounding; two launches of the new kernel give the same bits, and rows outside the buffer are untouched."""
    from edgedict_b200 import ops
    from edgedict_b200.functional import _Chunks
    _need(H)
    g = torch.Generator(device="cuda").manual_seed(5)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    k = _Chunks(B, lens)
    whhT16 = (rn(H, 4 * H) / np.sqrt(H)).bfloat16()
    gates = torch.sigmoid(rn(k.rows, 4 * H))
    gates[:, 2 * H:3 * H] = torch.tanh(rn(k.rows, H))
    cseq, dy = rn(k.rows, H), rn(k.rows, H)
    ref = torch.empty(k.rows, 4 * H, device="cuda").bfloat16()
    _, dh_r, dc_r = ops.lstm_tc_bwd_chunks(dy, gates, cseq, whhT16, lens, B, ref)
    one = torch.full((k.rows + 1, 4 * H), 7.0, device="cuda").bfloat16()
    _, dh1, dc1 = ops.lstm_c4_bwd_chunks(dy, gates, cseq, whhT16, lens, B, one[:k.rows])
    two = torch.empty(k.rows, 4 * H, device="cuda").bfloat16()
    _, dh2, dc2 = ops.lstm_c4_bwd_chunks(dy, gates, cseq, whhT16, lens, B, two)
    torch.cuda.synchronize()
    assert (one[k.rows] == 7.0).all()
    assert torch.equal(one[:k.rows], two) and torch.equal(dh1, dh2) and torch.equal(dc1, dc2)
    assert rel_err(one[:k.rows].float().cpu(), ref.float().cpu()) < 1e-2
    assert rel_err(dh1.cpu(), dh_r.cpu()) < 1e-2 and rel_err(dc1.cpu(), dc_r.cpu()) < 1e-2


def _tc_cluster_size(H):
    """The cluster size eb_lstm_tc_bwd picks (lstm_tc.cu pick_cs): the largest of 8 / 4 / 2 whose clusters all fit."""
    from edgedict_b200._lib import lib
    for cs in (8, 4, 2):
        if lib().eb_lstm_tc_max_clusters(H, cs) >= H // (8 * cs):
            return cs
    return 0


@pytest.mark.parametrize("B,H,lens", [(32, 1024, [167] * 5 + [165]), (40, 1024, [30, 20])])
def test_lstm_c4_bwd_chunks_same_bits_as_tc_kernel_in_clusters_of_2(B, H, lens):
    """When eb_lstm_tc_bwd runs clusters of 2 (an H100 at H = 1024), its dh sums run over the same 16 groups of H/4
    contraction indices, each accumulated over the same k16 steps, then in two halves of 8: the K-split kernel uses that
    order, so the two kernels give the same bits, and a training step gives the same bits with either."""
    from edgedict_b200 import ops
    from edgedict_b200.functional import _Chunks
    _need(H)
    if _tc_cluster_size(H) != 2:
        pytest.skip("eb_lstm_tc_bwd does not run clusters of 2 at this size on this GPU")
    g = torch.Generator(device="cuda").manual_seed(3)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)
    k = _Chunks(B, lens)
    whhT16 = (rn(H, 4 * H) / np.sqrt(H)).bfloat16()
    gates = torch.sigmoid(rn(k.rows, 4 * H))
    gates[:, 2 * H:3 * H] = torch.tanh(rn(k.rows, H))
    cseq, dy = rn(k.rows, H), rn(k.rows, H)
    a = torch.empty(k.rows, 4 * H, device="cuda").bfloat16()
    b = torch.empty_like(a)
    _, dha, dca = ops.lstm_tc_bwd_chunks(dy, gates, cseq, whhT16, lens, B, a)
    _, dhb, dcb = ops.lstm_c4_bwd_chunks(dy, gates, cseq, whhT16, lens, B, b)
    torch.cuda.synchronize()
    assert torch.equal(a, b) and torch.equal(dha, dhb) and torch.equal(dca, dcb)
