"""C-ABI argument validation of eb_lstm_c4_bwd_chunks (the K-split wgmma BPTT over chunk-major buffers): the checks mirror
eb_lstm_tc_bwd_chunks and run before any CUDA call, so they need no GPU."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def L():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    return lib()


P = 1 << 20                                                   # a plausible, aligned, never dereferenced address


def call(L, *, dy=P, gates=P, cseq=P, whhT=P, dg=P, dh0=P, dc0=P, scratch=P, B=4, lens=(3, 3), n=None, H=256):
    arr = None if lens is None else (ctypes.c_int * len(lens))(*lens)
    return L.eb_lstm_c4_bwd_chunks(dy, gates, cseq, None, whhT, None, None, dg, dh0, dc0, scratch, B, arr,
                                   len(lens) if n is None else n, H, None)


@pytest.mark.parametrize("name", ["dy", "gates", "cseq", "whhT", "dg", "dh0", "dc0", "scratch"])
def test_null_pointers_are_rejected(L, name):
    assert call(L, **{name: None}) == 2


def test_chunk_list_and_shape_are_validated(L):
    assert call(L, lens=(3,) * 9) == 2                        # more than 8 chunks
    assert call(L, lens=None, n=2) == 2                       # no chunk lengths
    assert call(L, lens=(3, 0)) == 2                          # empty chunk
    assert call(L, lens=(3, -1)) == 2
    assert call(L, lens=(3, 3), n=0) == 2
    assert call(L, H=320) == 2                                # H % 256
    assert call(L, H=2048) == 2                               # H > 1024
    assert call(L, B=0) == 2
    assert call(L, gates=P + 4) == 2                          # fp32 pairs are loaded as 8-byte words


def test_cluster_query_rejects_unsupported_sizes(L):
    assert L.eb_lstm_c4_bwd_chunks_cluster(320) == 0 and L.eb_lstm_c4_bwd_chunks_cluster(2048) == 0
    assert L.eb_lstm_c4_bwd_chunks_cluster(0) == 0
