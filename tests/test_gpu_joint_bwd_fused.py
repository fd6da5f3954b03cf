"""The loss gradient of the joint's bf16 backward with the output layer's bias gradient folded in, bit for bit:

    eb_rnnt_loss_bwd_bf16_db  d loss / d logits (bf16) and the bias gradient db[c] += sum over rows of them.  The
                              d logits must be eb_rnnt_loss_bwd_bf16's bits, and db must be eb_colsum's bits on those
                              d logits (its lane order: tests/test_gpu_colsum_order.py), accumulated into db.

Every output goes into a NaN-filled buffer with guard elements on both sides, and the guards must stay NaN.  The cases
cover ragged lengths (padded cells, whose d logits are zero and still take part in the column sum), cell counts that
are not a multiple of the 512 row lanes, vocabularies other than 1024 with V % 8 == 0, fewer cells than lanes, and the
E6D2 training shape itself."""
import numpy as np
import pytest
import torch

from tests.test_gpu_joint_loss_fused import _lattice, _lib, _lse, _p, _stream, _ws

pytestmark = pytest.mark.gpu

bf16 = torch.bfloat16
NAN = float("nan")
G = 8                      # guard elements on each side: keeps the 16-byte alignment of the slice between them


def _guarded(n, dtype):
    buf = torch.full((n + 2 * G,), NAN, dtype=dtype, device="cuda")
    return buf, buf[G:G + n]


def _guards_intact(name, buf):
    assert bool(buf[:G].isnan().all()) and bool(buf[-G:].isnan().all()), name + ": a guard element was written"


def _bits_equal(name, got, want):
    got, want = got.contiguous(), want.contiguous()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    iv = torch.int16 if got.dtype == bf16 else torch.int32
    diff = got.view(iv) != want.view(iv)
    assert not bool(diff.any()), "%s: %d of %d elements differ" % (name, int(diff.sum()), diff.numel())


# name: (B, T, U, V, J, blank, xlen, ylen, per-batch gscale)
LOSS_CASES = {
    # bench vocabulary, ragged (xlen = 1, ylen = 0), 3*24*21 = 1512 cells: not a multiple of 512
    "v1024_ragged": (3, 24, 21, 1024, 640, 0, [24, 17, 1], [20, 11, 0], False),
    # V % 256 != 0, blank in the last column group, per-utterance upstream gradient
    "v1000_blank_last": (2, 19, 13, 1000, 128, 999, [19, 12], [12, 5], True),
    # V = 136: a warp's threads span two row lanes; blank = 128
    "v136_blank128": (2, 23, 11, 136, 72, 128, [23, 9], [10, 10], False),
    # fewer cells (3*4*5 = 60) than row lanes: most lanes own no row
    "v72_few_cells": (3, 4, 5, 72, 8, 71, [4, 2, 1], [4, 0, 2], False),
    # several groups of 8 cells per lane, with a partial last group
    "v256_many_groups": (4, 97, 33, 256, 64, 3, [97, 60, 97, 5], [32, 32, 7, 0], True),
    # the E6D2 training step: B = 32, T' = 500 frames after time reduction, U + 1 = 129, V = 1024, J = 640
    "e6d2": (32, 500, 129, 1024, 640, 0, None, None, False),
}


def _loss_case(name):
    B, T, U, V, J, blank, xl, yl, per_batch = LOSS_CASES[name]
    seed = sum(map(ord, name))
    rng = np.random.RandomState(seed)
    if xl is None:
        xl, yl = [T] * B, [U - 1] * B
    g = torch.Generator(device="cuda").manual_seed(seed)
    n = B * T * U
    hid = (torch.rand(n, J, device="cuda", generator=g) * 2 - 1).to(bf16)
    w2 = (torch.randn(V, J, device="cuda", generator=g) * (3.0 * (3.0 / J) ** 0.5)).to(bf16)
    b2 = torch.randn(V, device="cuda", generator=g)
    lab = rng.randint(0, V, size=(B, U - 1)).astype(np.int32)
    lab[lab == blank] = (blank + 1) % V
    c = dict(B=B, T=T, U=U, V=V, J=J, blank=blank, hid=hid, w2=w2, b2=b2,
             lab_d=torch.as_tensor(lab, device="cuda"), xlen_d=torch.as_tensor(np.asarray(xl, np.int32), device="cuda"),
             ylen_d=torch.as_tensor(np.asarray(yl, np.int32), device="cuda"))
    gscale = (torch.rand(B, device="cuda", generator=g) + 0.5) if per_batch else torch.ones(1, device="cuda")
    return c, gscale


def _grad_args(c, ws, gscale):
    return (_p(c["lab_d"]), _p(c["xlen_d"]), _p(c["ylen_d"]), c["B"], c["T"], c["U"], c["V"], c["blank"], _p(ws),
            _p(gscale), int(gscale.numel() > 1), 1.0 / c["B"])


@pytest.mark.parametrize("name", list(LOSS_CASES))
def test_loss_gradient_with_bias_gradient_matches_gradient_then_colsum(name):
    from edgedict_b200 import ops
    c, gscale = _loss_case(name)
    B, T, U, V = c["B"], c["T"], c["U"], c["V"]
    n = B * T * U
    ws = _ws(c)
    logits = _lse(c, ws)
    _lattice(c, ws)
    del c["hid"]
    args = _grad_args(c, ws, gscale)
    # the existing entry, in place as JointLoss runs it, then eb_colsum on its d logits into a non-zero db
    ref = logits.clone()
    assert _lib().eb_rnnt_loss_bwd_bf16(_p(ref), _p(ref), *args, _stream()) == 0
    g = torch.Generator(device="cuda").manual_seed(n)
    db0 = torch.randn(V, device="cuda", generator=g)
    db_ref = ops.colsum(ref.view(n, V), out=db0.clone())

    part_buf, part = _guarded(512 * V, torch.float32)
    db_buf, db = _guarded(V, torch.float32)
    db.copy_(db0)
    # in place over the logits
    dl = logits.clone()
    assert _lib().eb_rnnt_loss_bwd_bf16_db(_p(dl), _p(dl), *args, _p(part), _p(db), _stream()) == 0
    torch.cuda.synchronize()
    _guards_intact(name + " part", part_buf)
    _guards_intact(name + " db", db_buf)
    _bits_equal(name + " d logits in place", dl, ref)
    _bits_equal(name + " db", db, db_ref)
    del dl
    # into a separate NaN-filled buffer: every element is written, padded cells with zeros
    out_buf, out = _guarded(n * V, bf16)
    db.copy_(db0)
    part.fill_(NAN)
    assert _lib().eb_rnnt_loss_bwd_bf16_db(_p(logits), _p(out), *args, _p(part), _p(db), _stream()) == 0
    torch.cuda.synchronize()
    _guards_intact(name + " d logits", out_buf)
    _bits_equal(name + " d logits out of place", out.view(B, T, U, V), ref)
    _bits_equal(name + " db (out of place)", db, db_ref)


def test_ops_wrapper_returns_the_column_sum_of_its_d_logits():
    """ops.rnnt_loss_bwd_bf16_db: db from zero is eb_colsum's column sum of the d logits it leaves in place."""
    from edgedict_b200 import ops
    c, gscale = _loss_case("v1024_ragged")
    B, T, U, V = c["B"], c["T"], c["U"], c["V"]
    ws = _ws(c)
    logits = _lse(c, ws)
    _lattice(c, ws)
    ref = logits.clone()
    ops.rnnt_loss_bwd_bf16(ref, c["lab_d"], c["xlen_d"], c["ylen_d"], c["blank"], ws, gscale, 1.0 / B)
    dl, db = ops.rnnt_loss_bwd_bf16_db(logits, c["lab_d"], c["xlen_d"], c["ylen_d"], c["blank"], ws, gscale, 1.0 / B)
    assert dl.data_ptr() == logits.data_ptr()
    _bits_equal("d logits", dl, ref)
    _bits_equal("db", db, ops.colsum(ref.view(-1, V)))


def test_loss_gradient_with_bias_gradient_rejects_what_it_cannot_run():
    """V % 8 != 0, misaligned pointers and missing buffers are refused before any launch."""
    L = _lib()
    buf = torch.zeros(4096, dtype=torch.float32, device="cuda")
    p = buf.data_ptr()
    lens = torch.ones(2, dtype=torch.int32, device="cuda")
    base = [p, p, lens.data_ptr(), lens.data_ptr(), lens.data_ptr(), 2, 3, 4, 16, 0, p, None, 0, 1.0, p, p, None]
    assert L.eb_rnnt_loss_bwd_bf16_db(*base[:8], 12, *base[9:]) == 2                       # V % 8
    for i in (0, 1, 14):                                                                      # logits, grads, part
        a = list(base)
        a[i] = p + 8
        assert L.eb_rnnt_loss_bwd_bf16_db(*a) == 2, i
    for i in (0, 1, 10, 14, 15):
        a = list(base)
        a[i] = None
        assert L.eb_rnnt_loss_bwd_bf16_db(*a) == 2, i
