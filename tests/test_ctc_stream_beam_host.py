"""Streaming CTC beam search without a GPU: the host-side refusals of stream_engine.CTCStreamBeamEngine and
ctc.CTCStreamDecoder(beam_width=...) (all raised before any device work), the C-ABI argument checks of
eb_decode_run_ctc_stream_beam and the Python mirror of the header, and the CPU restatement of the streaming search
(tests/ctc_stream_beam_oracle.py) pinned against the offline restatement (tests/ctc_beam_oracle.py)."""
import os
import re

import numpy as np
import pytest
import torch

from tests import ctc_beam_oracle as cbo
from tests.ctc_stream_beam_oracle import CTCStreamBeamRestatement, common_prefix

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)


def _model(**over):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(0)
    return CTCEncoder(**dict(TINY, **over))


def _lm(ntok, ninp=6, nhid=10, L=2, scale=2.0, seed=3):
    """An LMModel-shaped module (encoder / rnn / decoder)."""
    torch.manual_seed(seed)
    lm = torch.nn.Module()
    lm.encoder = torch.nn.Embedding(ntok, ninp)
    lm.rnn = torch.nn.LSTM(ninp, nhid, L, batch_first=True)
    lm.decoder = torch.nn.Linear(nhid, ntok)
    with torch.no_grad():
        for p in lm.parameters():
            p.mul_(scale)
    return lm.eval()


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_engine_refusals_come_before_any_device_work():
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import CTCStreamBeamEngine as E
    cuda_before = torch.cuda.is_initialized()
    m = _model()
    with pytest.raises(TypeError, match="CTCEncoder"):
        E(torch.nn.Linear(3, 4), 1, 2, 4)
    tr = Transducer(vocab_embed_size=8, vocab_size=10, input_size=6, enc_hidden_size=8, enc_layers=2, enc_dropout=0,
                    enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0, dec_proj_size=8, joint_size=8,
                    module_type="GRU", output_loss=False)
    with pytest.raises(TypeError, match="CTCEncoder"):
        E(tr, 1, 2, 4)
    for W in (0, -1, 1025):
        with pytest.raises(ValueError, match="beam width"):
            E(m, 2, 4, W)
    big = _model()
    big.tovocab[0] = torch.nn.Linear(32, 2 ** 21, device="meta")     # W x V = 2^31: never allocated
    with pytest.raises(ValueError, match="2\\^31"):
        E(big, 1, 4, 1024)
    for blank in (-1, 40):
        with pytest.raises(ValueError, match="blank"):
            E(m, 2, 4, 4, blank=blank)
    with pytest.raises(ValueError, match="need an lm"):
        E(m, 2, 4, 4, lm_weight=0.5)
    with pytest.raises(TypeError, match="lm must"):
        E(m, 2, 4, 4, lm=torch.nn.Linear(3, 3))
    with pytest.raises(ValueError, match="lm_token_map"):
        E(m, 2, 4, 4, lm=_lm(12))                          # 12 LM tokens, 40 CTC tokens, no map
    with pytest.raises(ValueError, match="lm_bos"):
        E(m, 2, 4, 4, lm=_lm(40), lm_bos=40)
    for S, n in ((0, 2), (2, 0), (-1, 4)):
        with pytest.raises(ValueError, match="positive"):
            E(m, S, n, 4)
    for n in (1, 3, 7):
        with pytest.raises(ValueError, match="even number of frames"):
            E(m, 2, n, 4)
    with pytest.raises(ValueError, match="max_pending"):
        E(m, 2, 8, 4, max_pending=3)                       # 8 input frames give 4 output frames
    with pytest.raises(RuntimeError, match="CUDA"):        # a CPU model, every other argument valid
        E(m, 2, 8, 4, max_pending=4, lm=_lm(40), lm_weight=0.3)
    assert torch.cuda.is_initialized() == cuda_before


def test_decoder_refusals_come_before_any_device_work():
    from edgedict_b200.ctc import CTCStreamDecoder as D
    cuda_before = torch.cuda.is_initialized()
    m = _model()
    with pytest.raises(TypeError, match="CTCEncoder"):
        D(torch.nn.Linear(3, 4), None, None, device="cuda", beam_width=4)
    for bw in ("4", 4.0, True):
        with pytest.raises(TypeError, match="beam_width"):
            D(m, None, None, device="cuda", beam_width=bw)
    for bw in (0, 1025):
        with pytest.raises(ValueError, match="beam_width"):
            D(m, None, None, device="cuda", beam_width=bw)
    big = _model()
    big.tovocab[0] = torch.nn.Linear(32, 2 ** 21, device="meta")
    with pytest.raises(ValueError, match="2\\^31"):
        D(big, None, None, device="cuda", beam_width=1024)
    with pytest.raises(ValueError, match="need an lm"):
        D(m, None, None, device="cuda", beam_width=4, length_bonus=1.0)
    with pytest.raises(ValueError, match="lm_token_map"):
        D(m, None, None, device="cuda", beam_width=4, lm=_lm(12))
    with pytest.raises(ValueError, match="need beam_width"):
        D(m, None, None, device="cuda", lm=_lm(40))
    with pytest.raises(ValueError, match="even number of frames"):
        D(m, None, None, device="cuda", frames_per_chunk=3, beam_width=4)
    with pytest.raises(ValueError, match="max_pending"):
        D(m, None, None, device="cuda", frames_per_chunk=8, beam_width=4, max_pending=2)
    with pytest.raises(RuntimeError, match="CUDA"):
        D(m, None, None, device="cpu", frames_per_chunk=4, beam_width=4)
    assert torch.cuda.is_initialized() == cuda_before


# ---- C ABI and the header ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    return lib()


P = 1 << 20                                                   # a plausible, aligned, never dereferenced address


def test_run_entry_validates_its_arguments(L):
    run = L.eb_decode_run_ctc_stream_beam
    assert run(None, 3, P, 0, None) == 2
    assert run(P, 3, None, 0, None) == 2
    for nphase in (0, -1):
        assert run(P, nphase, P, 0, None) == 2


def test_phase_numbers_flag_and_layout_match_the_header(L):
    import ctypes as C
    from edgedict_b200 import stream_engine as se
    src = open(os.path.join(ROOT, "include", "edgedict_b200.h")).read()
    enum = dict((k, int(v)) for k, v in re.findall(r"EB_PH_([A-Z_]+)\s*=\s*(\d+)", src))
    for name in ("CTC_BEAM", "BEAM_COMMIT", "GATHER", "COPY", "GRU", "CTC_EMIT", "LSTM", "LINEAR"):
        assert enum[name] == getattr(se, "PH_" + name), name
    assert re.search(r"\b64 = BEAM_SELECT streams", src) and "CTC_BEAM streams with the same flag" in src
    assert se.F_STREAM == 64 and se.F_FLUSH == 128
    cu = open(os.path.join(ROOT, "edgedict_b200", "csrc", "decode.cu")).read()
    assert int(re.search(r"constexpr int CTC_SEQ_HEAD = (\d+);", cu).group(1)) == se.CTC_SEQ_HEAD == 5
    assert "int eb_decode_run_ctc_stream_beam(" in src
    assert C.sizeof(se.EbPhase) == L.eb_decode_phase_size()


# ---- the restatement ---------------------------------------------------------------------------------------------------
def _lp(T, V, seed, scale=2.5):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(T, V, generator=g, dtype=torch.float64)).log_softmax(-1).numpy()


def _chunks(T, lens):
    out, t = [], 0
    while t < T:
        n = lens[len(out) % len(lens)]
        out.append((t, min(T, t + n)))
        t += n
    return out


def _stream(y, W, lens, **kw):
    rs = CTCStreamBeamRestatement(W, **kw)
    got, per = [], []
    for a, b in _chunks(y.shape[0], lens):
        out = rs.chunk(y[a:b])
        per.append(out)
        got += out
    rest, nscore = rs.flush()
    return got + rest, nscore, per, rs


LM_SD = {k: v.detach().double() for k, v in _lm(8).state_dict().items()}


@pytest.mark.parametrize("W", [1, 3, 6])
@pytest.mark.parametrize("lens", [[1], [2], [3, 1, 4], [40]])
@pytest.mark.parametrize("lm", [None, "identity", "permuted"])
def test_restatement_over_chunks_is_the_offline_search(W, lens, lm):
    """Committed plus flushed tokens and -score equal prefix_beam_search's on the whole utterance, bitwise in fp64."""
    blank = 0 if lm != "permuted" else 3
    V, T = 8, 40
    y = _lp(T, V, seed=W * 7 + len(lens))
    kw = dict(blank=blank, max_pending=1000)
    if lm:
        kw.update(lm_sd=LM_SD, lm_weight=0.6, length_bonus=0.4,
                  lm_map=None if lm == "identity" else torch.tensor([5, 2, -1, 7, 0, 1, -1, 3]))
    got, nscore, _, rs = _stream(y, W, lens, **kw)
    okw = {k: v for k, v in kw.items() if k != "max_pending"}
    want, wscore, _, _ = cbo.prefix_beam_search(y, T, W, **okw)
    assert tuple(got) == want
    assert nscore == wscore
    assert rs.n_collapses == 0
    assert len(got) > 3


@pytest.mark.parametrize("W", [2, 5])
def test_committed_tokens_are_the_common_prefix_of_the_live_prefixes(W):
    V, T = 6, 60
    y = _lp(T, V, seed=11 + W, scale=3.0)
    rs = CTCStreamBeamRestatement(W, max_pending=1000)
    total = 0
    for a, b in _chunks(T, [2, 1, 3]):
        before = rs.committed
        out = rs.chunk(y[a:b])
        live = [h["seq"] for h in rs.hyps]
        assert rs.committed == common_prefix(live)
        assert tuple(before) + tuple(out) == rs.committed
        total += len(out)
    assert total > 5, "nothing was committed before the end"


@pytest.mark.parametrize("lm", [False, True])
def test_collapse_bounds_the_suffixes(lm):
    """A small max_pending: every live suffix stays within max_pending - n_out after each chunk end, collapses happen,
    and committed plus flushed tokens form the best prefix the restatement ends with."""
    V, T, W, n_out, P = 8, 60, 4, 2, 4
    y = _lp(T, V, seed=5, scale=1.0)                  # flat log-probs: the live prefixes keep disagreeing
    kw = dict(lm_sd=LM_SD, lm_weight=0.5, length_bonus=0.2) if lm else {}
    rs = CTCStreamBeamRestatement(W, max_pending=P, **kw)
    got = []
    for a in range(0, T, n_out):
        got += rs.chunk(y[a:a + n_out])
        assert got == list(rs.committed)
        assert max(len(h["seq"]) for h in rs.hyps) - len(rs.committed) <= P - n_out
    best = rs.hyps[int(np.argmax([float(s) for s in rs.scores()]))]["seq"]
    rest, _ = rs.flush()
    assert tuple(got + rest) == best
    assert rs.n_collapses > 0
