"""C-ABI argument validation of the GRU recurrence (eb_gru_seq_fwd / eb_gru_seq_bwd / eb_gru_scratch_bytes and the
tensor-core eb_gru_tc_fwd / eb_gru_tc_bwd / eb_gru_tc_supported / eb_gru_tc_scratch_bytes): NULL pointers, non-positive
sizes, hidden sizes outside the tensor-core kernels' range and misaligned pointers are rejected with status 2 before
any CUDA call, so these tests need no GPU."""
import pytest


@pytest.fixture(scope="module")
def L():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    return lib()


P = 1 << 20                                                   # a plausible, aligned, never dereferenced address


def fwd(L, *, xg=P, whh=P, bhn=P, h0=None, y=P, hT=P, save=P, scratch=P, B=4, T=3, H=64):
    return L.eb_gru_seq_fwd(xg, whh, bhn, h0, y, hT, save, scratch, B, T, H, None)


def bwd(L, *, dy=P, save=P, y=P, h0=None, whh=P, dhT=None, dgi=P, dgh=P, dh0=P, scratch=P, B=4, T=3, H=64):
    return L.eb_gru_seq_bwd(dy, save, y, h0, whh, dhT, dgi, dgh, dh0, scratch, B, T, H, None)


@pytest.mark.parametrize("name", ["xg", "whh", "y", "hT", "scratch"])
def test_fwd_null_pointers_are_rejected(L, name):
    assert fwd(L, **{name: None}) == 2


@pytest.mark.parametrize("name", ["dy", "save", "y", "whh", "dgi", "dgh", "dh0", "scratch"])
def test_bwd_null_pointers_are_rejected(L, name):
    assert bwd(L, **{name: None}) == 2


@pytest.mark.parametrize("call", [fwd, bwd])
def test_sizes_are_validated(L, call):
    for kw in (dict(B=0), dict(B=-1), dict(T=0), dict(T=-5), dict(H=0), dict(H=-64)):
        assert call(L, **kw) == 2, kw


@pytest.mark.parametrize("call", [fwd, bwd])
def test_misaligned_scratch_is_rejected(L, call):
    # the exchange buffer behind the barrier word is pulled with 16-byte cp.async
    for off in (4, 8, 12):
        assert call(L, scratch=P + off) == 2


def test_scratch_query_rejects_empty_shapes(L):
    assert L.eb_gru_scratch_bytes(0, 64) == 0
    assert L.eb_gru_scratch_bytes(4, 0) == 0
    assert L.eb_gru_scratch_bytes(-1, 64) == 0


def tc_fwd(L, *, xg=P, whh=P, bhn=P, h0=None, y=P, hT=P, save=P, scratch=P, B=4, T=3, H=64):
    return L.eb_gru_tc_fwd(xg, whh, bhn, h0, y, hT, save, scratch, B, T, H, None)


def tc_bwd(L, *, dy=P, save=P, y=P, h0=None, whhT=P, dhT=None, dgi=P, dgh=P, dh0=P, scratch=P, B=4, T=3, H=64):
    return L.eb_gru_tc_bwd(dy, save, y, h0, whhT, dhT, dgi, dgh, dh0, scratch, B, T, H, None)


@pytest.mark.parametrize("name", ["xg", "whh", "y", "hT", "scratch"])
def test_tc_fwd_null_pointers_are_rejected(L, name):
    assert tc_fwd(L, **{name: None}) == 2


@pytest.mark.parametrize("name", ["dy", "save", "y", "whhT", "dgi", "dgh", "dh0", "scratch"])
def test_tc_bwd_null_pointers_are_rejected(L, name):
    assert tc_bwd(L, **{name: None}) == 2


@pytest.mark.parametrize("call", [tc_fwd, tc_bwd])
def test_tc_sizes_are_validated(L, call):
    for kw in (dict(B=0), dict(B=-1), dict(T=0), dict(H=0), dict(H=32), dict(H=96), dict(H=1000), dict(H=1088),
               dict(H=2048)):
        assert call(L, **kw) == 2, kw


def test_tc_misaligned_pointers_are_rejected(L):
    # W_hh fragments are loaded as 4-byte words, the exchange buffer is pulled and published in 16 bytes
    assert tc_fwd(L, whh=P + 2) == 2 and tc_bwd(L, whhT=P + 2) == 2
    for off in (4, 8):
        assert tc_fwd(L, scratch=P + off) == 2 and tc_bwd(L, scratch=P + off) == 2


def test_tc_range_queries(L):
    for B, H in ((4, 64), (1, 1024), (40, 320)):
        assert L.eb_gru_tc_supported(B, H) == 1 and L.eb_gru_tc_scratch_bytes(B, H) > 0
    for B, H in ((0, 64), (4, 96), (4, 2048), (4, 0)):
        assert L.eb_gru_tc_supported(B, H) == 0 and L.eb_gru_tc_scratch_bytes(B, H) == 0
