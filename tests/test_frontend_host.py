"""The front end without a GPU: the fp64 restatement (tests/frontend_oracle.py) against the reference's own FrontEnd
(tests/golden/frontend_tiny.npz), the engine's seeded construction against the reference's weights bit for bit, the
length arithmetic, the refusals before any device work, and the argument checks of the C entries."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import frontend_oracle as fo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
TAGS = ["train", "pre", "dflt"]
SAMPLE_ABOVE, SAMPLE_STEP = 4096, 31          # tests/golden/make_golden_frontend.py


def _seeded(tag):
    from edgedict_b200.rnnt.models import FrontEnd
    z = np.load(os.path.join(GOLDEN, "frontend_tiny.npz"))
    params = [tuple(int(v) for v in r) for r in z[tag + ".params"]]
    torch.manual_seed(int(z[tag + ".seed"]))
    return z, params, FrontEnd(params, bias=bool(z[tag + ".bias"]))


@pytest.mark.parametrize("tag", TAGS)
def test_seeded_frontend_equals_the_reference_state_dict(tag):
    z, _, m = _seeded(tag)
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in z[tag + ".keys"]]
    for k, t in sd.items():
        assert hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest() == str(z[tag + ".sha." + k]), k


@pytest.mark.parametrize("tag", TAGS)
def test_restatement_reproduces_the_reference(tag):
    z, params, m = _seeded(tag)
    out, grads = fo.forward_and_grads(m.state_dict(), z["x"], params, z[tag + ".R"])
    np.testing.assert_allclose(out.numpy(), z[tag + ".out"], rtol=0, atol=2e-5)
    for k, _ in m.named_parameters():
        g = grads[k].numpy().reshape(-1)
        g = g if g.size <= SAMPLE_ABOVE else g[::SAMPLE_STEP]
        want = z[tag + ".grad." + k]
        np.testing.assert_allclose(g, want, rtol=0, atol=1e-5 * np.abs(want).max(), err_msg=k)


@pytest.mark.parametrize("tag", TAGS)
def test_bf16_restatement_without_rounding_is_the_fp64_restatement(tag):
    """The bf16-mode restatement with every rounding switched off is bit for bit the fp64 one; with the roundings on it
    moves the output and every gradient but the LayerNorm bias's (the sum of R), by no more than bf16 operands can."""
    z, params, m = _seeded(tag)
    sd = m.state_dict()
    out, grads = fo.forward_and_grads(sd, z["x"], params, z[tag + ".R"])
    out0, grads0 = fo.forward_and_grads(sd, z["x"], params, z[tag + ".R"], bf16=True, rounding=False)
    assert torch.equal(out0, out)
    for k, _ in m.named_parameters():
        assert torch.equal(grads0[k], grads[k]), k
    out1, grads1 = fo.forward_and_grads(sd, z["x"], params, z[tag + ".R"], bf16=True)
    for k, a, b in [("out", out1, out)] + [(k, grads1[k], grads[k]) for k, _ in m.named_parameters()]:
        rel = float((a - b).abs().max() / b.abs().max())
        assert (rel > 0 or k == "layer_norm.bias") and rel < 5e-2, (k, rel)


def test_length_arithmetic():
    from edgedict_b200.functional import conv_out_len
    from edgedict_b200.rnnt.models import FrontEnd
    train = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3
    assert FrontEnd(train).output_length(16 * 16000) == 399
    for T in (1, 2, 7, 100, 1001):
        for k, s in ((10, 5), (8, 4), (4, 2), (3, 2), (2, 2), (2, 3)):
            want = torch.nn.functional.conv1d(torch.zeros(1, 1, T), torch.zeros(1, 1, k), stride=s,
                                              padding=k - 1).shape[-1] - (k - 1)
            assert conv_out_len(T, k, s) == want


def test_frontend_lengths_is_the_trainers_rule():
    from edgedict_b200.rnnt.models import frontend_lengths
    xlen = torch.tensor([224000, 210345, 201600, 199999])
    T = 349
    want = torch.floor(xlen.float() / (xlen.max().item() / T)).int()
    got = frontend_lengths(xlen, T)
    assert got.dtype == torch.int32 and torch.equal(got, want) and int(got.max()) == T


def test_refusals_before_device_work():
    from edgedict_b200.rnnt.models import DilatedConvBlock, FrontEnd
    m = FrontEnd()
    with pytest.raises(ValueError):
        m(torch.zeros(2, 4000))                                   # a CPU tensor
    with pytest.raises(ValueError):
        m(torch.zeros(2, 4000, dtype=torch.float64))
    if torch.cuda.is_available():                                 # (only reachable with a device)
        with pytest.raises(ValueError):
            m(torch.zeros(2, 4000, dtype=torch.float16, device="cuda"))
        with pytest.raises(ValueError):
            FrontEnd([(10, 5, 16), (1, 1, 32)]).cuda()(torch.zeros(2, 4000, device="cuda"))
        with pytest.raises(ValueError):
            FrontEnd().cuda()(torch.zeros(2, 30, device="cuda"))
        with pytest.raises(ValueError):
            FrontEnd([(10, 5, 24), (3, 2, 128)]).cuda().set_precision("bf16")(torch.zeros(2, 4000, device="cuda"))
    with pytest.raises(ValueError):
        FrontEnd([(10, 5, 16), (1, 1, 32)]).output_length(4000)   # k == 1
    with pytest.raises(ValueError):
        FrontEnd().output_length(30)                               # a layer without output frames
    with pytest.raises(ValueError):
        DilatedConvBlock(16, 32, 3, stride=2)(torch.zeros(1, 16, 50))


def _lib():
    from edgedict_b200._lib import lib, LIB_PATH
    if not os.path.exists(LIB_PATH):
        pytest.skip("libedgedict_b200.so is not built")
    return lib()


def test_c_entries_reject_bad_arguments():
    L = _lib()
    P = ctypes.c_void_p
    dummy = P(256)
    INVALID = 2
    assert L.eb_conv_rows_per_split(128) == 256 and L.eb_conv_rows_per_split(0) == 0
    # first layer: T must be the conv's output length, k >= 2
    assert L.eb_conv1d_first_fwd(dummy, dummy, None, dummy, 2, 4000, 32, 10, 5, 100, None) == INVALID
    assert L.eb_conv1d_first_fwd(dummy, dummy, None, dummy, 2, 4000, 32, 1, 1, 4000, None) == INVALID
    assert L.eb_conv1d_first_fwd(None, dummy, None, dummy, 2, 4000, 32, 10, 5, 799, None) == INVALID
    # split count must match the rows
    assert L.eb_conv1d_first_dw(dummy, dummy, dummy, 3, 256, 2, 4000, 32, 10, 5, 799, None) == INVALID
    assert L.eb_gn_stats(dummy, 10, 2, 5, 4, dummy, dummy, dummy, 1e-5, None) == INVALID        # ustride < T*C
    assert L.eb_gn_stats(None, 20, 2, 5, 4, dummy, dummy, dummy, 1e-5, None) == INVALID
    assert L.eb_gn_apply(dummy, 20, 2, 5, 4, dummy, dummy, None, None, dummy, 0, 2, 6, 12, None) == INVALID
    assert L.eb_gn_apply(dummy, 20, 2, 5, 4, dummy, dummy, None, None, dummy, 0, 2, 8, 10, None) == INVALID
    assert L.eb_gn_bwd(dummy, 20, 2, 5, 4, dummy, dummy, None, dummy, 20, dummy, dummy, dummy, None, None, 20, None,
                       None) == INVALID                                                      # no dy output
    # the tensor-core conv: channel counts multiple of 16, aligned operands, even row pitch
    assert L.eb_conv1d_bf16(dummy, 100, 2, 24, 0, dummy, 3, 128, None, dummy, 128, 50, None) == INVALID
    assert L.eb_conv1d_bf16(dummy, 100, 2, 32, 0, dummy, 3, 120, None, dummy, 128, 50, None) == INVALID
    assert L.eb_conv1d_bf16(P(258), 100, 2, 32, 0, dummy, 3, 128, None, dummy, 128, 50, None) == INVALID
    assert L.eb_conv1d_bf16(dummy, 100, 2, 32, 0, dummy, 3, 128, None, dummy, 127, 50, None) == INVALID
    assert L.eb_gemm_f32_splitk(dummy, 1, 1, dummy, 1, 1, dummy, 4, 4, 100, 0, None) == INVALID
    assert L.eb_gemm_f32_splitk(dummy, 1, 1, dummy, 1, 1, dummy, 4, 4, 10 ** 8, 1, None) == INVALID
