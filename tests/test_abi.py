"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol
the headers declare; the Python mirror keeps the reference's interface (names, state_dict keys,
seeded initialisation, error behaviour).  No compute calls (no GPU needed)."""
import os
import re

import numpy as np
import pytest
import torch

from tests.util import E4D1_CFG, load_e4d1

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    from edgedict_b200 import build
    return build.build()


def _declared(header):
    src = open(os.path.join(ROOT, "include", header)).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return set(re.findall(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\([^;{]*\)\s*;", src)) - {"defined"}


def test_library_exports_every_declared_symbol(built):
    import ctypes
    h = ctypes.CDLL(built)
    names = _declared("edgedict_b200.h") | _declared("rnnt.h")
    assert len(names) > 25
    for n in sorted(names):
        assert hasattr(h, n), "missing export: " + n
    from edgedict_b200 import _lib
    assert set(_lib.SIGNATURES) == names, set(_lib.SIGNATURES) ^ names
    _lib.lib()


def test_version_and_status_strings(built):
    from edgedict_b200._lib import lib
    L = lib()
    assert L.get_warprnnt_version() == 1                  # rnnt_entrypoint.cpp:14-16
    assert L.rnntGetStatusString(0) == b"no error"
    assert L.rnntGetStatusString(2) == b"invalid value"
    import ctypes as C
    sz = C.c_size_t(0)
    assert L.get_workspace_size(4, 3, 2, True, C.byref(sz), 4) == 0 and sz.value >= 2 * (3 * 4 * 3 + 2) * 4
    assert L.get_workspace_size(0, 3, 2, True, C.byref(sz), 4) == 2      # INVALID_VALUE


def test_state_dict_keys_and_seeded_init_match_reference():
    from edgedict_b200.rnnt.models import Transducer
    z = load_e4d1()
    torch.manual_seed(10)
    m = Transducer(output_loss=False, **E4D1_CFG)
    sd = m.state_dict()
    assert list(sd.keys()) == [str(k) for k in z["sd_keys"]]
    sums = np.array([float(v.double().sum()) for v in sd.values()])
    abss = np.array([float(v.double().abs().sum()) for v in sd.values()])
    assert np.allclose(sums, z["sd_sum"], rtol=0, atol=1e-9)
    assert np.allclose(abss, z["sd_abs"], rtol=0, atol=1e-9)


def test_interface_surface():
    from edgedict_b200.rnnt import models
    from edgedict_b200.rnnt.tokenizer import NUL, PAD, BOS, UNK
    assert (NUL, PAD, BOS, UNK) == (0, 1, 2, 3)
    m = models.Transducer(**E4D1_CFG)
    for attr in ("encoder", "decoder", "joint", "blank", "loss_fn", "forward", "scale_length", "greedy_decode"):
        assert hasattr(m, attr)
    with pytest.raises(ValueError):
        models.Transducer(module_type="RNN", **E4D1_CFG)
    xl = m.scale_length(torch.zeros(2, 100, 41, 8), torch.tensor([200, 180], dtype=torch.int32))
    assert xl.tolist() == [100, 90] and xl.dtype == torch.int32
    ck = {"state_dict": {"model.encoder.norm.weight": 1, "model.joint.joint.0.bias": 2}}
    assert models.convert_lightning2normal(ck) == {"model": {"encoder.norm.weight": 1, "joint.joint.0.bias": 2}}
    assert models.convert_lightning2normal({"model": 3}) == {"model": 3}


def test_loss_certify_inputs_and_cpu_refusal():
    from edgedict_b200.warprnnt_pytorch import RNNTLoss, rnnt_loss
    acts = torch.zeros(2, 4, 3, 5)
    labels = torch.zeros(2, 2, dtype=torch.int32)
    tl = torch.tensor([4, 4], dtype=torch.int32)
    ul = torch.tensor([2, 2], dtype=torch.int32)
    with pytest.raises(TypeError):
        rnnt_loss(acts, labels.long(), tl, ul)
    with pytest.raises(ValueError, match="Input length mismatch"):
        rnnt_loss(acts, labels, torch.tensor([3, 3], dtype=torch.int32), ul)
    with pytest.raises(ValueError, match="Output length mismatch"):
        rnnt_loss(acts, labels, tl, torch.tensor([1, 1], dtype=torch.int32))
    with pytest.raises(ValueError):
        rnnt_loss(acts.transpose(1, 2), labels, tl, ul)
    with pytest.raises(RuntimeError, match="CUDA-only"):
        RNNTLoss()(acts, labels, tl, ul)               # no silent CPU path


def test_model_refuses_cpu_tensors():
    from edgedict_b200.rnnt.models import Encoder
    enc = Encoder(8, 16, 1, 0, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        enc(torch.zeros(1, 4, 8))


def test_entry_points_reject_bad_arguments_before_touching_the_device(built):
    """Error behaviour of the C ABI (status 2 = invalid value, as rnntStatus_t RNNT_STATUS_INVALID_VALUE): argument
    checks run before any CUDA call, so they are testable without a GPU."""
    from edgedict_b200._lib import lib
    L = lib()
    p = 1 << 20                                               # a plausible, aligned, never dereferenced address
    assert L.eb_gemm_bf16(None, 0, p, 0, p, 0, None, 0, 8, 8, 8, None) == 2
    assert L.eb_gemm_bf16(p, 0, p, 0, p, 0, None, 0, 8, 8, 12, None) == 2            # K-major rows must be 16-byte multiples
    assert L.eb_gemm_bf16(p + 2, 0, p, 0, p, 0, None, 0, 8, 8, 8, None) == 2         # misaligned operand
    assert L.eb_gemm_bf16_ex(p, 1, p, 0, p, 0, None, 0, 8, 8, 8, 1, None, 0, None) == 2   # co-resident config: K-major only
    # the epilogue stores column pairs as float2 (fp32 C) / __nv_bfloat162 (bf16 C)
    for c_bf16, off in ((0, 4), (0, 2), (0, 1), (1, 2), (1, 1)):
        assert L.eb_gemm_bf16(p, 0, p, 0, p + off, c_bf16, None, 0, 8, 8, 8, None) == 2, (c_bf16, off)
        assert L.eb_gemm_bf16(p, 1, p, 1, p + off, c_bf16, None, 1, 8, 8, 8, None) == 2, (c_bf16, off)
        assert L.eb_gemm_bf16_ex(p, 0, p, 0, p + off, c_bf16, None, 0, 8, 8, 8, 1, None, 0, None) == 2, (c_bf16, off)
    assert L.eb_gemm_bf16_dtanh(p, 0, p, 1, p, None, 8, 8, 8, None) == 2             # needs the hidden activations
    assert L.eb_gemm_bf16_dtanh(p, 0, p, 1, p, p, 8, 6, 8, None) == 2                # N % 4
    assert L.eb_joint_dpre_reduce(None, p, p, 1, 1, 1, 8, None) == 2
    assert L.eb_joint_dpre_reduce(p, p, p, 1, 1, 1, 12, None) == 2                   # J % 8
    assert L.eb_joint_logits_lse(p, p, None, p, p, p, p, p, p, p, 1, 1, 1, 8, 12, 0, None) == 2   # J % 8
    assert L.eb_joint_logits_lse(p, p, None, p, p, p, p, p, p, p, 1, 1, 1, 8, 8, 9, None) == 2    # blank >= V
    # the bf16 joint kernels load and store 16 bytes at a time: every operand must be 16-byte aligned
    for off in (2, 4, 8):
        assert L.eb_joint_dpre_reduce(p, p, p + off, 1, 1, 1, 8, None) == 2, off          # ddp
        assert L.eb_joint_dpre_reduce(p, p + off, p, 1, 1, 1, 8, None) == 2, off          # dep
        for i in range(3):
            a = [p, p, p]
            a[i] += off
            assert L.eb_joint_hidden_fwd(a[0], a[1], a[2], 1, 1, 1, 1, 8, None) == 2, (i, off)
        for i in range(4):
            a = [p, p, p, p]
            a[i] += off
            assert L.eb_joint_hidden_bwd(a[0], a[1], 1, a[2], a[3], 1, 1, 1, 8, None) == 2, (i, off)
    assert L.eb_joint_hidden_fwd(p, p, p, 1, 1, 1, 1, 12, None) == 2                  # J % 8
    assert L.eb_joint_hidden_bwd(p, p, 1, p, p, 1, 1, 1, 12, None) == 2
    # LayerNorm backward rejects what the forward rejects
    assert L.eb_layernorm_fwd(p, None, p, p, p, None, p, p, 0, 64, 1e-5, None) == 2
    assert L.eb_layernorm_bwd(p, p, None, p, p, p, p, p, p, 0, 64, None) == 2          # rows <= 0
    assert L.eb_layernorm_bwd(p, p, None, p, p, p, p, p, p, -3, 64, None) == 2
    assert L.eb_layernorm_bwd(p, p, None, p, p, p, p, p, p, 4, 0, None) == 2           # H <= 0
    assert L.eb_layernorm_bwd(p, p, None, p, p, p, p, p, p, 4, 2049, None) == 2
    assert L.eb_layernorm_fwd(p, None, p, p, p, None, p, p, 4, 2049, 1e-5, None) == 2
    # NULL operands and negative sizes; the optional y_bf16 / out_bf16 copies stay optional (an empty output returns
    # 0 without a launch, which is also what these calls with the copies omitted would reach on a GPU)
    assert L.eb_time_reduce_fwd(None, p, None, 2, 3, 4, None) == 2
    assert L.eb_time_reduce_fwd(p, None, p, 2, 3, 4, None) == 2
    assert L.eb_time_reduce_fwd(p, p, None, -1, 3, 4, None) == 2
    assert L.eb_time_reduce_fwd(p, p, None, 2, -3, 4, None) == 2
    assert L.eb_time_reduce_fwd(p, p, None, 2, 3, -4, None) == 2
    assert L.eb_time_reduce_fwd(None, None, None, 2, 0, 4, None) == 0                # empty: nothing to do
    assert L.eb_time_reduce_bwd(None, p, 2, 3, 4, None) == 2
    assert L.eb_time_reduce_bwd(p, None, 2, 3, 4, None) == 2
    assert L.eb_time_reduce_bwd(p, p, 2, -3, 4, None) == 2
    assert L.eb_embedding_fwd(None, 0, p, p, None, 2, 3, 4, 1, 2, None) == 2
    assert L.eb_embedding_fwd(p, 0, None, p, None, 2, 3, 4, 1, 2, None) == 2
    assert L.eb_embedding_fwd(p, 1, p, None, p, 2, 3, 4, 0, 2, None) == 2
    assert L.eb_embedding_fwd(p, 0, p, p, None, -2, 3, 4, 1, 2, None) == 2
    assert L.eb_embedding_fwd(p, 0, p, p, None, 2, -3, 4, 1, 2, None) == 2
    assert L.eb_embedding_fwd(p, 0, p, p, None, 2, 3, -4, 1, 2, None) == 2
    assert L.eb_embedding_fwd(p, 0, p, p, None, 2, 3, 4, 1, -1, None) == 2           # BOS row < 0
    assert L.eb_embedding_bwd(None, 0, p, p, 2, 3, 4, 1, 2, 1, None) == 2
    assert L.eb_embedding_bwd(p, 0, None, p, 2, 3, 4, 1, 2, 1, None) == 2
    assert L.eb_embedding_bwd(p, 0, p, None, 2, 3, 4, 1, 2, 1, None) == 2
    assert L.eb_embedding_bwd(p, 0, p, p, 2, -3, 4, 1, 2, 1, None) == 2
    assert L.eb_embedding_bwd(p, 0, p, p, 2, 3, 4, 1, -2, 1, None) == 2
    assert L.eb_transpose_to_bf16(None, 0, p, 8, 8, None) == 2
    assert L.eb_transpose_to_bf16(p, 1, None, 8, 8, None) == 2
    assert L.eb_transpose_to_bf16(p, 0, p, -8, 8, None) == 2
    assert L.eb_transpose_to_bf16(p, 0, p, 8, -8, None) == 2
    assert L.eb_transpose_to_bf16(None, 0, None, 0, 8, None) == 0                    # empty: nothing to do
    assert L.eb_sumsq(None, 8, p, None) == 2
    assert L.eb_sumsq(p, 8, None, None) == 2
    assert L.eb_sumsq(p, -8, p, None) == 2
    assert L.eb_fe_preemph_pad(None, p, 1, 100, 400, 8, 0.97, 1, None) == 2
    assert L.eb_fe_preemph_pad(p, p, 1, 100, 100, 8, 0.97, 1, None) == 2             # Lp < L + 2*pad
    assert L.eb_fe_power(p, None, 4, 4, None) == 2
    assert L.eb_fe_log_stack(p, p, 1, 3, 5, 5, 8, 1, 5, 1, None) == 2                # rows_per_utt < n_frames
    assert L.eb_lstm_tc_supported(32, 1024) == 1 and L.eb_lstm_tc_supported(32, 1000) == 0
    assert L.eb_lstm_tc_supported(32, 2048) == 0 and L.eb_lstm_tc_scratch_bytes(32, 1000) == 0
    assert L.eb_lstm_tc_fwd(None, p, None, None, p, p, p, p, None, None, p, 4, 3, 64, None) == 2
    assert L.eb_lstm_tc_fwd(p, p, None, None, p, p, p, p, None, None, p, 4, 0, 64, None) == 2     # T <= 0
    assert L.eb_lstm_tc_bwd(p, p, p, None, p, None, None, p, p, p, p, 4, 3, 96, None) == 2        # H % 64
    import ctypes
    lens = (ctypes.c_int * 9)(3, 3, 3, 3, 3, 3, 3, 3, 3)
    assert L.eb_lstm_tc_bwd_chunks(p, p, p, None, p, None, None, p, p, p, p, 4, lens, 9, 64, None) == 2   # more than 8 chunks
    assert L.eb_lstm_tc_bwd_chunks(p, p, p, None, p, None, None, p, p, p, p, 4, None, 2, 64, None) == 2   # no chunk lengths
    lens0 = (ctypes.c_int * 2)(3, 0)
    assert L.eb_lstm_tc_bwd_chunks(p, p, p, None, p, None, None, p, p, p, p, 4, lens0, 2, 64, None) == 2  # empty chunk
    assert L.eb_lstm_tc_bwd_chunks(p, p, p, None, p, None, None, p, p, p, p, 4, lens, 2, 96, None) == 2   # H % 64
    # the two loss backward entries reject what eb_rnnt_loss_fwd rejects: the kernels would dereference the missing
    # lengths / labels on the device, and a blank outside [0, V) would silently drop its gradient term
    good = dict(labels=p, xlen=p, ylen=p, B=2, maxT=3, maxU=4, V=8, blank=0)
    bad = [dict(xlen=None), dict(ylen=None), dict(labels=None), dict(B=0), dict(maxT=0), dict(maxU=0), dict(V=0),
           dict(B=-1), dict(V=-8), dict(blank=-1), dict(blank=8), dict(maxU=1025)]
    for change in bad:
        a = dict(good, **change)
        args = (a["labels"], a["xlen"], a["ylen"], a["B"], a["maxT"], a["maxU"], a["V"], a["blank"])
        assert L.eb_rnnt_loss_bwd_bf16(p, p, *args, p, None, 0, 1.0, None) == 2, change
        for dtype_size, out_bf16 in ((4, 0), (4, 1), (8, 0)):
            assert L.eb_rnnt_loss_bwd(p, p, out_bf16, *args, dtype_size, p, None, 0, 1.0, None) == 2, (change, dtype_size)
        assert L.eb_rnnt_loss_fwd(p, a["labels"], a["xlen"], a["ylen"], *args[3:], 4, p, None, 1, None) == 2, change
