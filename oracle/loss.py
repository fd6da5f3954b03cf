"""ctypes front-ends for the loss checkers (TEST INFRASTRUCTURE).

``logits_*``   : oracle/rnnt_loss_oracle.c, GPU-entry semantics (logits in, dense grads wrt logits)
``logprobs_*`` : oracle/rnnt_loss_oracle.c, CPU-entry semantics (log-probs in, sparse grads)
``ref_cpu``    : the reference's own library (oracle/_ref/libwarprnnt_ref.so) through its C ABI,
                 warp-transducer/include/rnnt.h:104-143, options struct passed by value.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE_SO = os.path.join(_HERE, "liboracle.so")
_REF_SO = os.path.join(_HERE, "_ref", "libwarprnnt_ref.so")


def build(quiet=True):
    """Compile liboracle.so and, where the reference's warp-transducer sources are (oracle/Makefile), _ref/."""
    out = subprocess.run(["make", "-C", _HERE], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


_lib = None
_ref = None
NUM_THREADS = 0      # 0 = OpenMP default; bench.py sets this for the reference library (options.num_threads)


def _oracle():
    global _lib
    if _lib is None:
        if not os.path.exists(_ORACLE_SO):
            build()
        _lib = C.CDLL(_ORACLE_SO)
    return _lib


def have_ref():
    return os.path.exists(_REF_SO)


class RnntOptions(C.Structure):
    # warp-transducer/include/rnnt.h:43-64
    _fields_ = [("loc", C.c_int), ("num_threads", C.c_uint), ("stream", C.c_void_p),
                ("blank_label", C.c_int), ("maxT", C.c_int), ("maxU", C.c_int),
                ("batch_first", C.c_bool)]


def _refl():
    global _ref
    if _ref is None:
        _ref = C.CDLL(_REF_SO)
        _ref.get_workspace_size.argtypes = [C.c_int, C.c_int, C.c_int, C.c_bool,
                                            C.POINTER(C.c_size_t), C.c_size_t]
        _ref.compute_rnnt_loss.restype = C.c_int
        _ref.compute_rnnt_loss_fp64.restype = C.c_int
    return _ref


def _prep(acts, labels, act_lens, label_lens, dtype):
    acts = np.ascontiguousarray(acts, dtype=dtype)
    labels = np.ascontiguousarray(labels, dtype=np.int32)
    act_lens = np.ascontiguousarray(act_lens, dtype=np.int32)
    label_lens = np.ascontiguousarray(label_lens, dtype=np.int32)
    B, T, U, V = acts.shape
    assert labels.shape == (B, U - 1), (labels.shape, acts.shape)
    return acts, labels, act_lens, label_lens, B, T, U, V


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def logits(acts, labels, act_lens, label_lens, blank=0, want_grads=True, dtype=np.float32):
    """GPU-entry semantics (gpu_rnnt.h:82-215): returns (costs[B], grads wrt logits | None)."""
    acts, labels, act_lens, label_lens, B, T, U, V = _prep(acts, labels, act_lens, label_lens, dtype)
    sfx = "f32" if dtype == np.float32 else "f64"
    fn = getattr(_oracle(), "oracle_rnnt_logits_" + sfx)
    costs = np.zeros(B, dtype=dtype)
    grads = np.zeros_like(acts) if want_grads else None
    fn(_p(acts), _p(grads) if want_grads else None, _p(labels), _p(label_lens), _p(act_lens),
       C.c_int(V), C.c_int(B), C.c_int(T), C.c_int(U), C.c_int(blank), _p(costs))
    return costs, grads


def logprobs(log_probs, labels, act_lens, label_lens, blank=0, want_grads=True,
             dtype=np.float32, want_lattice=False):
    """CPU-entry semantics (cpu_rnnt.h:272-338): input is log-probs, grads wrt log-probs."""
    lp, labels, act_lens, label_lens, B, T, U, V = _prep(log_probs, labels, act_lens, label_lens, dtype)
    sfx = "f32" if dtype == np.float32 else "f64"
    fn = getattr(_oracle(), "oracle_rnnt_logprobs_" + sfx)
    costs = np.zeros(B, dtype=dtype)
    grads = np.zeros_like(lp) if want_grads else None
    al = np.zeros((B, T, U), dtype=dtype) if want_lattice else None
    be = np.zeros((B, T, U), dtype=dtype) if want_lattice else None
    fn(_p(lp), _p(grads) if want_grads else None, _p(labels), _p(label_lens), _p(act_lens),
       C.c_int(V), C.c_int(B), C.c_int(T), C.c_int(U), C.c_int(blank), _p(costs),
       _p(al) if want_lattice else None, _p(be) if want_lattice else None)
    if want_lattice:
        return costs, grads, al, be
    return costs, grads


def log_softmax(x, dtype=np.float32):
    x = np.ascontiguousarray(x, dtype=dtype)
    V = x.shape[-1]
    rows = x.size // V
    out = np.empty_like(x)
    den = np.empty(rows, dtype=dtype)
    sfx = "f32" if dtype == np.float32 else "f64"
    getattr(_oracle(), "oracle_row_log_softmax_" + sfx)(_p(x), _p(out), _p(den), C.c_long(rows), C.c_int(V))
    return out, den.reshape(x.shape[:-1])


def ref_cpu(log_probs, labels, act_lens, label_lens, blank=0, want_grads=True,
            dtype=np.float32, num_threads=0):
    """The reference's own CPU library (input = log-probs, as warprnnt_pytorch feeds it)."""
    lp, labels, act_lens, label_lens, B, T, U, V = _prep(log_probs, labels, act_lens, label_lens, dtype)
    lib = _refl()
    size = C.c_size_t(0)
    st = lib.get_workspace_size(T, U, B, False, C.byref(size), lp.itemsize)
    assert st == 0
    ws = np.zeros(size.value, dtype=np.uint8)
    costs = np.zeros(B, dtype=dtype)
    grads = np.zeros_like(lp) if want_grads else None
    opt = RnntOptions(loc=0, num_threads=num_threads or NUM_THREADS, stream=None, blank_label=blank,
                      maxT=T, maxU=U, batch_first=True)
    fn = lib.compute_rnnt_loss if dtype == np.float32 else lib.compute_rnnt_loss_fp64
    st = fn(_p(lp), _p(grads) if want_grads else None, _p(labels), _p(label_lens), _p(act_lens),
            C.c_int(V), C.c_int(B), _p(costs), _p(ws), opt)
    if st != 0:
        raise RuntimeError("reference compute_rnnt_loss status %d" % st)
    return costs, grads
