"""eb_colsum on bf16 rows (N % 8 == 0): the exact summation order, bit for bit.  Row lane k (0 <= k < 512) adds rows
k, k + 512, k + 1024, ... in order in fp32, then a fixed-shape tree adds the 512 lane sums (at stride st = 256 ... 1,
lane k < st adds lane k + st).  The bias gradients of the training step depend on this order for their bits, however
the lanes are spread over CTAs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _colsum_in_order(x16):
    x = x16.float().cpu().numpy()
    rows, N = x.shape
    lanes = np.zeros((512, N), dtype=np.float32)
    for r0 in range(0, rows, 512):
        blk = x[r0:r0 + 512]
        lanes[:blk.shape[0]] = lanes[:blk.shape[0]] + blk          # fp32 adds, one row per lane at a time
    st = 256
    while st:
        lanes[:st] = lanes[:st] + lanes[st:2 * st]
        st //= 2
    return lanes[0]


@pytest.mark.parametrize("rows,N", [(1, 8), (300, 24), (512, 16), (4096 + 7, 40), (3 * 512 * 8 + 511, 1024),
                                    (512 * 8 * 5, 64), (20000, 4096)])
def test_colsum_bf16_bits_follow_the_lane_order(rows, N):
    from edgedict_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(rows + N)
    x = (torch.randn(rows, N, device="cuda", generator=g) * 3).bfloat16()
    got = ops.colsum(x).cpu().numpy()
    want = _colsum_in_order(x)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), float(np.abs(got - want).max())


def test_colsum_bf16_accumulates_into_out():
    from edgedict_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(2000, 32, device="cuda", generator=g).bfloat16()
    base = torch.randn(32, device="cuda", generator=g)
    out = ops.colsum(x, out=base.clone()).cpu().numpy()
    want = base.cpu().numpy() + _colsum_in_order(x)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))
