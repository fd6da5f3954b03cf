"""Host-side checks (no GPU) of the two restatements tests/test_gpu_features_fp64.py and the tightened feature tests
trust (tests/features_fp64.py):

* finish32 / deltas32, the float32 restatement of eb_fe_finish / eb_fe_deltas, against the fp64 oracle's CatDeltas and
  Downsample (tests/features_batch_oracle.py), including the pad_to_divisible=False drop after the deltas;
* the fp64 chain from the module's fp32 tables against the fp64 oracle on exact tables: their distance stays within
  the table terms the chain's bar adds in table mode."""
import numpy as np
import pytest
import torch

from tests import features_batch_oracle as O
from tests import features_fp64 as X
from tests.test_features_batch_host import CONFIGS, golden


@pytest.mark.parametrize("F,C,n,ptd", [(1, 3, 1, True), (2, 5, 2, True), (3, 4, 3, False), (5, 7, 2, False),
                                       (5, 7, 3, True), (23, 40, 3, False), (200, 13, 2, True), (7, 2, 3, False)])
def test_finish32_is_catdeltas_then_downsample(F, C, n, ptd):
    rng = np.random.default_rng(F * 100 + C)
    s = (rng.standard_normal((F, C)) * np.exp(rng.standard_normal((1, C)))).astype(np.float32)
    feat = s.T[None].astype(np.float64)                                 # [1, C, F], the reference's layout
    want = O.F.downsample(O.cat_deltas(feat), n, ptd)[0].T              # [T, 3 C n]
    Fs = F if ptd else F - F % n
    T = -(-F // n) if ptd else F // n
    got = X.finish32(s, F, Fs, n, T, True)
    assert got.shape == want.shape == (T, 3 * C * n)
    # three fp32 roundings per delta of |terms| <= 6 max|s| / 10, twice for d2: 1e-6 max|s| is ~40x the worst case
    assert np.abs(got - want).max() <= 1e-6 * np.abs(s).max()
    assert np.array_equal(X.finish32(s, F, Fs, n, T, False), O.F.downsample(feat, n, ptd)[0].T.astype(np.float32))
    # the dropped frames [Fs, F) still feed the deltas of the kept ones
    if Fs < F and Fs > 0:
        s2 = s.copy()
        s2[Fs:] += 1
        assert not np.array_equal(X.finish32(s2, F, Fs, n, T, True), got)
        assert np.array_equal(X.finish32(s2, F, Fs, n, T, False), X.finish32(s, F, Fs, n, T, False))


def test_deltas32_edges_and_order():
    s = np.arange(1, 6, dtype=np.float32)[:, None] ** 2                 # 1 4 9 16 25
    d = X.deltas32(s)[:, 0]
    # f = 0: (2 (9 - 1) + (4 - 1)) / 10; f = 4: (2 (25 - 9) + (25 - 16)) / 10 (replicate edges)
    assert d[0] == np.float32(19) / np.float32(10) and d[4] == np.float32(41) / np.float32(10)
    assert np.array_equal(X.deltas32(np.ones((1, 3), np.float32)), np.zeros((1, 3), np.float32))
    # the order is (2 (p2 - m2) + (p1 - m1)) / 10, not sum_k k x_k / 10: the two differ in the last bit somewhere
    rng = np.random.default_rng(3)
    s = rng.standard_normal((4000, 1)).astype(np.float32)
    i = np.arange(4000)
    g = lambda k: s[np.clip(i + k, 0, 3999)]
    other = (np.float32(-2) * g(-2) - g(-1) + g(1) + np.float32(2) * g(2)) / np.float32(10)
    assert not np.array_equal(X.deltas32(s), other)


@pytest.mark.parametrize("ft,delta,n_fft,ds,ptd", [c for c in CONFIGS if c[2] == 512 or c[0] == "mfcc"])
def test_chain_on_fp32_tables_is_within_the_table_terms_of_the_oracle(ft, delta, n_fft, ds, ptd):
    from edgedict_b200.rnnt.features import build_batch_transform
    z = golden()
    C = int(z["size"])
    _, test, _ = build_batch_transform(ft, C, n_fft=n_fft, win_length=400, hop_length=200, delta=delta, downsample=ds,
                                       pad_to_divisible=ptd, dither=0)
    basis, fbT, dct, pre = X.module_tables(test)
    x = torch.tensor(z["x"])
    kw = dict(n_fft=n_fft, hop=200, n_stack=ds, delta=delta, ptd=ptd, preemph=pre, dct=dct)
    val, bar0, ok0 = X.chain(x, z["lens"], ft, basis, fbT, **kw)
    te = X.tables_err(ft, basis, fbT, dct, n_fft, C, pre)
    _, bar, ok = X.chain(x, z["lens"], ft, basis, fbT, tables_err=te, **kw)
    want, _ = O.batch_transform(z["x"].astype(np.float64), z["lens"], ft, C, n_fft=n_fft, win_length=400,
                                hop_length=200, delta=delta, downsample=ds, pad_to_divisible=ptd)
    # the table terms alone bound the distance; 1e-12 covers the two fp64 evaluations
    X.report("%s d%d n%d ds%d p%d chain vs oracle" % (ft, delta, n_fft, ds, ptd), val, want,
             (bar - bar0).clamp_min(0) + 1e-12 * (1 + torch.from_numpy(np.abs(want))), ok & ok0)
