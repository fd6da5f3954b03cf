"""ctypes loader for libedgedict_b200.so (the C-ABI declared in include/edgedict_b200.h and
include/rnnt.h).  There is NO fallback: if the library is missing or a call fails, we raise."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libedgedict_b200.so")

_lib = None

P, I, L, F, D, Z = C.c_void_p, C.c_int, C.c_long, C.c_float, C.c_double, C.c_size_t

OPT_MAX_GROUPS = 16


class OptHyper(C.Structure):
    """eb_opt_hyper: the per-group optimizer hyperparameters, passed by value."""
    _fields_ = [(k, D * OPT_MAX_GROUPS) for k in ("lr", "wd", "b1", "b2", "eps")]


# name -> (restype, argtypes); mirrors include/edgedict_b200.h one to one
SIGNATURES = {
    "eb_rnnt_workspace_bytes": (Z, [I, I, I, I]),
    "eb_rnnt_loss_fwd": (I, [P, P, P, P, I, I, I, I, I, I, P, P, I, P]),
    "eb_rnnt_loss_bwd": (I, [P, P, I, P, P, P, I, I, I, I, I, I, P, P, I, D, P]),
    "eb_rnnt_loss_lattice": (I, [P, P, I, I, I, P, P, I, P]),
    "eb_rnnt_loss_bwd_bf16": (I, [P, P, P, P, P, I, I, I, I, I, P, P, I, D, P]),
    "eb_rnnt_loss_bwd_bf16_db": (I, [P, P, P, P, P, I, I, I, I, I, P, P, I, D, P, P, P]),
    "eb_rnnt_loss_bwd_fe": (I, [P, P, I, P, P, P, I, I, I, I, I, I, P, P, I, D, D, P]),
    "eb_rnnt_loss_bwd_bf16_fe": (I, [P, P, P, P, P, I, I, I, I, I, P, P, I, D, D, P]),
    "eb_rnnt_loss_bwd_bf16_db_fe": (I, [P, P, P, P, P, I, I, I, I, I, P, P, I, D, P, P, D, P]),
    "eb_joint_logits_lse": (I, [P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, P]),
    "eb_lm_logits_ce": (I, [P, P, P, P, P, I, P, P, L, I, I, P]),
    "eb_lm_ce_rows": (I, [P, P, I, P, P, L, I, P]),
    "eb_lm_ce_loss": (I, [P, P, P, I, L, L, I, I, P, P, P, P]),
    "eb_lm_ce_bwd": (I, [P, P, I, P, P, I, L, L, I, P, I, P, P]),
    "eb_rnnt_workspace_views": (I, [P, I, I, I, I, P, P, P, P, P]),
    "eb_rnnt_align_bytes": (Z, [I, I, I]),
    "eb_rnnt_viterbi": (I, [P, P, I, I, I, I, P, P, P, P, P, P]),
    "eb_log_softmax_fwd": (I, [P, P, L, I, P]),
    "eb_log_softmax_bwd": (I, [P, P, P, L, I, P]),
    "eb_ctc_workspace_size": (Z, [I, I, I]),
    "eb_ctc_loss_fwd": (I, [P, L, L, I, I, I, P, L, P, P, P, I, I, I, P, P, P]),
    "eb_ctc_loss_bwd": (I, [P, L, L, P, L, L, I, I, I, P, P, I, I, I, P, P, P]),
    "eb_ctc_greedy": (I, [P, L, L, I, I, I, P, I, P, P, P, P]),
    "eb_ctc_align_workspace_size": (Z, [I, I, I]),
    "eb_ctc_align": (I, [P, L, L, I, I, I, P, L, P, P, P, I, I, P, P, P, P]),
    "eb_gemm_f32": (I, [P, L, L, P, L, L, P, L, P, I, I, I, F, F, P]),
    "eb_gemm_bf16": (I, [P, I, P, I, P, I, P, I, L, I, L, P]),
    "eb_gemm_bf16_ex": (I, [P, I, P, I, P, I, P, I, L, I, L, I, P, L, P]),
    "eb_gemm_bf16_partials": (L, [I, I, I, L, I, L, I]),
    "eb_gemm_bf16_dtanh": (I, [P, I, P, I, P, P, L, I, L, P]),
    "eb_gemm_tc_set_trace": (I, [P, I]),
    "eb_joint_dpre_reduce": (I, [P, P, P, I, I, I, I, P]),
    "eb_rnnt_simple_scratch_bytes": (Z, [I, I, I, I]),
    "eb_rnnt_simple_stats": (I, [P, P, P, P, P, I, I, I, I, I, P, P, P]),
    "eb_rnnt_simple_bwd": (I, [P, P, P, P, P, I, I, I, I, I, P, P, P, I, D, P, P, P]),
    "eb_rnnt_band_choice": (I, [P, P, I, I, I, I, P, P, P, P]),
    "eb_joint_band_hidden_fwd": (I, [P, P, P, P, P, P, I, I, I, I, I, I, P]),
    "eb_rnnt_band_loss_fwd": (I, [P, P, P, P, P, P, I, I, I, I, I, I, P, P, I, P]),
    "eb_rnnt_band_loss_bwd": (I, [P, P, I, P, P, P, P, P, I, I, I, I, I, I, P, P, I, D, P]),
    "eb_joint_band_dpre_reduce": (I, [P, P, I, P, P, P, P, P, I, I, I, I, I, P]),
    "eb_rnnt_band_lattice": (I, [P, P, P, P, I, I, I, I, P, P, I, P]),
    "eb_joint_band_logits_lse": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, I, I, I, I, P]),
    "eb_rnnt_band_loss_bwd_bf16_db": (I, [P, P, P, P, P, P, P, I, I, I, I, I, I, P, P, I, D, P, P, P]),
    "eb_lstm_scratch_bytes": (Z, [I, I]),
    "eb_lstm_seq_fwd": (I, [P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_seq_bwd": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_gru_scratch_bytes": (Z, [I, I]),
    "eb_gru_seq_fwd": (I, [P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_gru_seq_bwd": (I, [P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_gru_tc_supported": (I, [I, I]),
    "eb_gru_tc_scratch_bytes": (Z, [I, I]),
    "eb_gru_tc_fwd": (I, [P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_gru_tc_bwd": (I, [P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_tc_supported": (I, [I, I]),
    "eb_lstm_tc_scratch_bytes": (Z, [I, I]),
    "eb_lstm_tc_max_clusters": (I, [I, I]),
    "eb_lstm_tc_set_trace": (I, [P, I]),
    "eb_lstm_tc_fwd": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_tc_bwd": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_tc_bwd_chunks": (I, [P, P, P, P, P, P, P, P, P, P, P, I, P, I, I, P]),
    "eb_lstm_c4_supported": (I, [I, I]),
    "eb_lstm_c4_bwd_cluster": (I, [I]),
    "eb_lstm_c4_max_clusters": (I, [I, I]),
    "eb_lstm_c4_set_trace": (I, [P, I]),
    "eb_lstm_c4_scratch_bytes": (Z, [I, I]),
    "eb_lstm_c4_gsave_bytes": (Z, [I, I, I]),
    "eb_lstm_c4_csave_bytes": (Z, [I, I, I]),
    "eb_lstm_c4_fwd": (I, [P, P, P, P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_c4_bwd": (I, [P, P, P, P, P, P, P, P, P, P, P, I, I, I, P]),
    "eb_lstm_c4_bwd_chunks_cluster": (I, [I]),
    "eb_lstm_c4_bwd_chunks": (I, [P, P, P, P, P, P, P, P, P, P, P, I, P, I, I, P]),
    "eb_layernorm_fwd": (I, [P, P, P, P, P, P, P, P, L, I, F, P]),
    "eb_layernorm_bwd": (I, [P, P, P, P, P, P, P, P, P, L, I, P]),
    "eb_layernorm_bwd_dz": (I, [P, P, P, P, P, P, P, L, I, P]),
    "eb_layernorm_bwd_params": (I, [P, P, P, P, P, P, P, L, I, P]),
    "eb_time_reduce_fwd": (I, [P, P, P, I, I, I, P]),
    "eb_time_reduce_bwd": (I, [P, P, I, I, I, P]),
    "eb_embedding_fwd": (I, [P, I, P, P, P, I, I, I, I, I, P]),
    "eb_embedding_bwd": (I, [P, I, P, P, I, I, I, I, I, I, P]),
    "eb_joint_hidden_fwd": (I, [P, P, P, I, I, I, I, I, P]),
    "eb_joint_hidden_bwd": (I, [P, P, I, P, P, I, I, I, I, P]),
    "eb_decode_phase_size": (I, []),
    "eb_decode_run": (I, [P, I, P, I, P]),
    "eb_decode_run_ctc": (I, [P, I, P, I, P]),
    "eb_decode_run_ctc_stream": (I, [P, I, P, I, P]),
    "eb_decode_run_gru_rnnt": (I, [P, I, P, I, P]),
    "eb_decode_run_ctc_stream_beam": (I, [P, I, P, I, P]),
    "eb_colsum": (I, [P, I, P, L, I, P]),
    "eb_cast_bf16": (I, [P, P, L, P]),
    "eb_transpose_to_bf16": (I, [P, I, P, L, L, P]),
    "eb_adam_step": (I, [P, P, P, P, L, F, F, F, F, F, I, F, P]),
    "eb_adam_step_ex": (I, [P, P, P, P, L, F, F, F, F, F, I, F, P, F, I, P]),
    "eb_sumsq": (I, [P, L, P, P]),
    "eb_opt_seg_sumsq": (I, [P, P, I, P, I, P, P, P, P]),
    "eb_opt_prologue": (I, [P, F, F, I, P, P, P]),
    "eb_opt_sgd_step": (I, [P, P, P, P, P, I, OptHyper, I, P, P, P]),
    "eb_opt_sm3_step": (I, [P, P, P, P, L, P, P, I, OptHyper, I, P, P]),
    "eb_opt_adamw_step": (I, [P, P, P, P, P, P, I, OptHyper, I, P, P, P]),
    "eb_opt_novograd_step": (I, [P, P, P, P, P, P, I, P, I, OptHyper, I, P, P]),
    "eb_fe_preemph_pad": (I, [P, P, I, I, L, I, F, I, P]),
    "eb_fe_power": (I, [P, P, L, I, P]),
    "eb_fe_log_stack": (I, [P, P, I, I, I, I, I, I, I, I, P]),
    "eb_fe_mask": (I, [P, P, I, I, I, I, I, F, P]),
    "eb_fe_preemph_pad_lens": (I, [P, P, P, P, I, I, L, I, F, I, P]),
    "eb_fe_log": (I, [P, L, F, P]),
    "eb_fe_finish": (I, [P, P, P, P, I, I, I, I, I, I, I, I, I, I, P]),
    "eb_fe_deltas": (I, [P, P, I, I, I, P]),
    "eb_conv_rows_per_split": (I, [I]),
    "eb_conv1d_first_fwd": (I, [P, P, P, P, I, I, I, I, I, I, P]),
    "eb_conv1d_first_dw": (I, [P, P, P, I, L, I, I, I, I, I, I, P]),
    "eb_gn_stats": (I, [P, L, I, I, I, P, P, P, F, P]),
    "eb_gn_apply": (I, [P, L, I, I, I, P, P, P, P, P, I, I, L, L, P]),
    "eb_gn_bwd": (I, [P, L, I, I, I, P, P, P, P, L, P, P, P, P, P, L, P, P]),
    "eb_conv1d_bf16": (I, [P, L, I, I, I, P, I, I, P, P, L, L, P]),
    "eb_gemm_f32_splitk": (I, [P, L, L, P, L, L, P, I, I, I, I, P]),
    "eb_w2v_mask_fwd": (I, [P, P, P, P, L, I, P]),
    "eb_w2v_keep_rows": (I, [P, P, P, L, I, P]),
    "eb_w2v_gather": (I, [P, P, P, I, I, I, I, P]),
    "eb_w2v_scatter": (I, [P, P, P, I, I, I, I, P]),
    "eb_w2v_sq_mean": (I, [P, L, P, P]),
    "eb_w2v_scale": (I, [P, P, F, L, P, P]),
    "eb_w2v_quant_fwd": (I, [P, P, P, I, I, I, I, F, P, P, P, P, P, P, P, P]),
    "eb_w2v_quant_stats": (I, [P, P, I, I, I, P, P, P, P]),
    "eb_w2v_quant_bwd": (I, [P, P, P, P, P, I, I, I, F, P, P]),
    "eb_w2v_logits_fwd": (I, [P, P, P, I, I, I, I, F, F, P, P, P, P, P, P, P]),
    "eb_w2v_logits_bwd": (I, [P, P, P, P, P, P, P, P, P, I, I, I, I, F, F, P, P, P, P, P]),
    "eb_w2v_ce": (I, [P, I, I, I, P, P, P]),
    "eb_edit_distance_smem_bytes": (Z, [I, I, I]),
    "eb_edit_distance": (I, [P, L, P, L, P, P, I, I, P, P, I, I, P, P]),
    "eb_nbest_pack": (I, [P, P, I, I, I, P, I, P, P, I, P, P, P]),
    "eb_mwer_risk_fwd": (I, [P, P, P, I, I, P, P, P, P]),
    "eb_mwer_risk_bwd": (I, [P, P, P, I, I, P, P, P]),
    # warp-transducer compatible ABI (include/rnnt.h)
    "get_warprnnt_version": (I, []),
    "rnntGetStatusString": (C.c_char_p, [I]),
    "get_workspace_size": (I, [I, I, I, C.c_bool, C.POINTER(Z), Z]),
    "compute_rnnt_loss": (I, None),        # takes struct rnntOptions by value: bound in tests
    "compute_rnnt_loss_fp64": (I, None),
}


class LibraryMissing(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises LibraryMissing loudly if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise LibraryMissing(
                "edgedict_b200: %s not found -- build it with `python -m edgedict_b200.build` "
                "(nvcc, sm_90a).  There is no CPU / PyTorch fallback for the hot path." % LIB_PATH)
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)              # AttributeError if a declared symbol is not exported
            fn.restype = res
            if args is not None:
                fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("edgedict_b200: %s failed with status %d" % (what, rc))
