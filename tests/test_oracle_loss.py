"""Pins the loss oracle (oracle/rnnt_loss_oracle.c) against the reference's own known-answer
vectors and against what the reference's CPU library computes (tests/golden/ref_loss.npz, written by
tests/golden/make_golden.py from that library)."""
import os

import numpy as np
import pytest

from oracle import loss as ol
from tests.golden import loss_kat as K
from tests.util import GOLDEN

REF_LOSS = os.path.join(GOLDEN, "ref_loss.npz")


def test_small_kat_logits():
    costs, grads = ol.logits(K.SMALL_ACTS, K.SMALL_LABELS, [2], [2])
    assert np.allclose(costs[0], K.SMALL_COST, rtol=1e-6)
    assert np.allclose(grads, K.SMALL_GRADS_LOGITS, atol=1e-6)
    c64, g64 = ol.logits(K.SMALL_ACTS, K.SMALL_LABELS, [2], [2], dtype=np.float64)
    assert abs(c64[0] - K.SMALL_COST) < 1e-6
    assert np.allclose(g64, K.SMALL_GRADS_LOGITS, atol=2e-8)


def test_big_kat_logits():
    costs, grads = ol.logits(K.BIG_ACTS, K.BIG_LABELS, [4, 4], [2, 2], dtype=np.float64)
    assert np.allclose(costs, K.BIG_COSTS, atol=1e-9)
    assert np.allclose(grads, K.BIG_GRADS_LOGITS, rtol=1e-3, atol=1e-8)
    costs32, grads32 = ol.logits(K.BIG_ACTS, K.BIG_LABELS, [4, 4], [2, 2])
    assert np.allclose(costs32, K.BIG_COSTS, rtol=1e-6)
    assert np.allclose(grads32, K.BIG_GRADS_LOGITS, rtol=1e-3, atol=1e-6)


def test_big_kat_logprobs():
    lp, _ = ol.log_softmax(K.BIG_ACTS)
    costs, grads = ol.logprobs(lp, K.BIG_LABELS, [4, 4], [2, 2])
    assert np.allclose(costs, K.BIG_COSTS, atol=1e-4)
    assert np.allclose(grads, K.BIG_GRADS_LOGPROBS, atol=1e-4)


def test_inf_problem():
    # warp-transducer/tests/test_cpu.cpp:181-240: V=15 T=50 U=10, finite cost, no NaN
    rng = np.random.RandomState(0)
    acts = rng.uniform(0, 1, size=(1, 50, 10, 15)).astype(np.float32)
    labels = rng.randint(1, 15, size=(1, 9)).astype(np.int32)
    costs, grads = ol.logits(acts, labels, [50], [9])
    assert np.isfinite(costs).all() and np.isfinite(grads).all()


def _numeric_grad(acts, labels, tl, ul, eps=1e-4):
    g = np.zeros_like(acts)
    flat = acts.reshape(-1)
    for i in range(flat.size):
        old = flat[i]
        flat[i] = old + eps
        cp, _ = ol.logits(acts, labels, tl, ul, want_grads=False, dtype=np.float64)
        flat[i] = old - eps
        cm, _ = ol.logits(acts, labels, tl, ul, want_grads=False, dtype=np.float64)
        flat[i] = old
        g.reshape(-1)[i] = (cp.sum() - cm.sum()) / (2 * eps)
    return g


def test_numeric_gradient():
    # the check warp-transducer/tests/test_cpu.cpp:242-379 intends (its binary aborts on a
    # missing return); reduced sizes so the central differences finish in seconds
    rng = np.random.RandomState(3)
    acts = rng.uniform(0, 1, size=(2, 6, 4, 5)).astype(np.float64)
    labels = np.array([[1, 1, 3], [2, 4, 0]], dtype=np.int32)
    tl, ul = [6, 5], [3, 2]
    _, g = ol.logits(acts, labels, tl, ul, dtype=np.float64)
    num = _numeric_grad(acts.copy(), labels, tl, ul)
    assert np.allclose(g, num, atol=1e-7)


def _ref_inputs(B, T, U, V, ragged):
    """the inputs tests/golden/make_golden.py fed the reference library for ref_loss.npz"""
    rng = np.random.RandomState(B * 1000 + T)
    acts = rng.uniform(0, 1, size=(B, T, U, V)).astype(np.float32)
    labels = rng.randint(1, V, size=(B, U - 1)).astype(np.int32)
    tl = np.full(B, T, np.int32)
    ul = np.full(B, U - 1, np.int32)
    if ragged:
        tl[1:] = rng.randint(1, T + 1, size=B - 1)
        ul[1:] = rng.randint(0, U, size=B - 1)
    return acts, labels, tl, ul


@pytest.mark.parametrize("B,T,U,V,ragged", [(1, 2, 3, 5, False), (3, 17, 6, 11, True),
                                            (2, 50, 16, 20, True), (4, 10, 6, 5, True)])
def test_against_reference_library(B, T, U, V, ragged):
    acts, labels, tl, ul = _ref_inputs(B, T, U, V, ragged)
    lp, _ = ol.log_softmax(acts)
    z = np.load(REF_LOSS)
    c_ref, g_ref = z["%d_%d_%d_%d.costs" % (B, T, U, V)], z["%d_%d_%d_%d.grads" % (B, T, U, V)]
    c_o, g_o = ol.logprobs(lp, labels, tl, ul)
    assert np.allclose(c_o, c_ref, rtol=1e-6)
    # both fp32; |alpha+beta| ~ 1e2 so one ulp of the exponent argument is ~1e-5 relative
    assert np.allclose(g_o, g_ref, atol=2e-5)
    # logits-semantics oracle must agree with log-probs semantics through the softmax Jacobian
    c_l, g_l = ol.logits(acts, labels, tl, ul, dtype=np.float64)
    assert np.allclose(c_l, c_ref, rtol=1e-5)
    p = np.exp(lp.astype(np.float64))
    g_chain = g_ref - p * g_ref.sum(-1, keepdims=True)
    assert np.allclose(g_l, g_chain, atol=1e-4)


def test_reference_library_reproduces_its_own_kat():
    c = np.load(REF_LOSS)["small_kat.costs"]
    assert abs(c[0] - K.SMALL_COST) < 1e-4
    lp, _ = ol.log_softmax(K.SMALL_ACTS)                    # and the oracle's CPU-entry path agrees with the library
    c_o, _ = ol.logprobs(lp, K.SMALL_LABELS, [2], [2])
    assert np.allclose(c_o, c, rtol=1e-6)
