"""Streaming greedy CTC without a GPU: the host-side refusals of stream_engine.CTCStreamEngine and
ctc.CTCStreamDecoder (all raised before any device work), the chunking semantics pinned by the CPU restatement
(tests/ctc_stream_oracle.py) streamed over chunks against oracle/ctc.py's offline greedy decode of the concatenated
frames, bitwise in fp64, and the C-ABI argument checks of eb_decode_run_ctc_stream."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import ctc as oc
from tests.ctc_stream_oracle import CTCStreamRestatement
from tests.test_oracle_ctc import load_ctc_tiny

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = dict(vocab_size=40, input_size=24, enc_hidden_size=48, enc_layers=3, enc_dropout=0, proj_size=32)


def _model(**over):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(0)
    return CTCEncoder(**dict(TINY, **over))


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_engine_refusals_come_before_any_device_work():
    from edgedict_b200.rnnt.models import Transducer
    from edgedict_b200.stream_engine import CTCStreamEngine
    cuda_before = torch.cuda.is_initialized()
    m = _model()
    with pytest.raises(TypeError, match="CTCEncoder"):
        CTCStreamEngine(torch.nn.Linear(3, 4), 1, 2)
    tr = Transducer(vocab_embed_size=8, vocab_size=10, input_size=6, enc_hidden_size=8, enc_layers=2, enc_dropout=0,
                    enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0, dec_proj_size=8, joint_size=8,
                    module_type="GRU", output_loss=False)
    with pytest.raises(TypeError, match="CTCEncoder"):
        CTCStreamEngine(tr, 1, 2)
    for S, n in ((0, 2), (-1, 2), (2, 0), (2, -2)):
        with pytest.raises(ValueError, match="positive"):
            CTCStreamEngine(m, S, n)
    for n in (1, 3, 7):                                   # the time reduction after layer 1 pairs frames
        with pytest.raises(ValueError, match="even number of frames"):
            CTCStreamEngine(m, 2, n)
    for blank in (-1, 40):
        with pytest.raises(ValueError, match="blank"):
            CTCStreamEngine(m, 2, 2, blank=blank)
    with pytest.raises(RuntimeError, match="CUDA"):        # a CPU model, every other argument valid
        CTCStreamEngine(m, 2, 4)
    m2 = _model()
    m2.model.lstm.time_reductions = {0, 1}
    with pytest.raises(ValueError, match="even number of frames"):
        CTCStreamEngine(m2, 1, 6)                         # 6 -> 3 after layer 0, odd before layer 1's reduction
    assert torch.cuda.is_initialized() == cuda_before


def test_decoder_refusals_come_before_any_device_work():
    from edgedict_b200.ctc import CTCStreamDecoder
    cuda_before = torch.cuda.is_initialized()
    with pytest.raises(TypeError, match="CTCEncoder"):
        CTCStreamDecoder(torch.nn.Linear(3, 4), None, None, device="cpu")
    with pytest.raises(ValueError, match="even number of frames"):
        CTCStreamDecoder(_model(), None, None, device="cpu", frames_per_chunk=3)
    with pytest.raises(RuntimeError, match="CUDA"):
        CTCStreamDecoder(_model(), None, None, device="cpu", frames_per_chunk=4)
    assert torch.cuda.is_initialized() == cuda_before


# ---- chunking semantics ------------------------------------------------------------------------------------------------
def _stream(sd, xs, lens, blank=0, tr=(1,)):
    rs = CTCStreamRestatement(sd, xs.shape[0], blank, tr)
    ids, lps, t0 = [[] for _ in range(xs.shape[0])], [], 0
    for n in lens:
        out, lp, _ = rs.step(xs[:, t0:t0 + n])
        t0 += n
        lps.append(lp)
        for s, o in enumerate(out):
            ids[s] += o
    return ids, torch.cat(lps, 1), rs.score


@pytest.mark.parametrize("lens", [[2] * 7, [4, 4, 2, 4], [14], [6, 2, 6], [2, 12]])
def test_restatement_over_chunks_is_offline_greedy_fp64_fixture(lens):
    """tests/golden/ctc_tiny.npz has 15 input frames, which no even chunking reproduces: its first 14 stream."""
    z, _, sd = load_ctc_tiny()
    sd64 = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in sd.items()}
    xs = torch.as_tensor(z["xs"], dtype=torch.float64)[:, :14]
    ids, lp, score = _stream(sd64, xs, lens)
    want_lp = oc.ctc_encoder_forward(sd64, xs)
    assert torch.equal(lp, want_lp), "streamed log-probs differ from the offline forward"
    want_ids, want_nlp = oc.greedy_from_logprobs(want_lp, torch.full((xs.shape[0],), 7))
    assert [list(map(int, w)) for w in want_ids] == ids
    assert torch.allclose(score, -want_nlp, rtol=1e-12, atol=0)
    # the fixture's own first 7 log-prob frames (the reference's fp32 forward) decode to the same ids
    fix_ids, _ = oc.greedy_from_logprobs(torch.as_tensor(z["logprobs"][:, :7]), torch.full((4,), 7))
    assert [list(map(int, w)) for w in fix_ids] == ids


@pytest.mark.parametrize("blank", [0, 7])
def test_restatement_over_chunks_is_offline_greedy_fp64_random(blank):
    """A tiny CTCEncoder scaled so that many frames emit, 5 streams x 24 frames, chunkings of 2, 4 and mixed lengths."""
    m = _model()
    sd = {k: v.detach().double() * 3.0 for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(1)
    xs = torch.randn(5, 24, TINY["input_size"], generator=g, dtype=torch.float64)
    want_lp = oc.ctc_encoder_forward(sd, xs)
    want_ids, want_nlp = oc.greedy_from_logprobs(want_lp, torch.full((5,), 12), blank)
    assert sum(len(w) for w in want_ids) > 15
    am = want_lp.argmax(-1)
    assert bool(((am[:, 1:] == am[:, :-1]) & (am[:, 1:] != blank)).any()), "no repeat to collapse"
    for lens in ([2] * 12, [4] * 6, [2, 6, 4, 2, 8, 2], [24]):
        ids, lp, score = _stream(sd, xs, lens, blank)
        assert torch.equal(lp, want_lp)
        assert [list(map(int, w)) for w in want_ids] == ids, lens
        assert torch.allclose(score, -want_nlp, rtol=1e-12, atol=0)


# ---- C ABI -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    return lib()


P = 1 << 20                                                   # a plausible, aligned, never dereferenced address


def test_run_entry_validates_its_arguments(L):
    run = L.eb_decode_run_ctc_stream
    assert run(None, 3, P, 0, None) == 2
    assert run(P, 3, None, 0, None) == 2
    for nphase in (0, -1):
        assert run(P, nphase, P, 0, None) == 2


def test_phase_numbers_and_layout_match_the_header(L):
    import ctypes as C
    from edgedict_b200 import stream_engine as se
    src = open(os.path.join(ROOT, "include", "edgedict_b200.h")).read()
    enum = dict((k, int(v)) for k, v in re.findall(r"EB_PH_([A-Z_]+)\s*=\s*(\d+)", src))
    assert enum["GRU"] == se.PH_GRU == 12 and enum["CTC_EMIT"] == se.PH_CTC_EMIT == 13
    assert enum["CTC_BEAM"] == se.PH_CTC_BEAM == 11
    assert C.sizeof(se.EbPhase) == L.eb_decode_phase_size()
