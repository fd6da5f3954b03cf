"""Streaming GRU transducers without a GPU: the host-side refusals of stream_engine.GRUStreamEngine /
GRUStreamBeamEngine and of PytorchStreamDecoder on a GRU model (all raised before any device work), the C-ABI argument
checks of eb_decode_run_gru_rnnt, the chunking semantics pinned by the CPU restatement (tests/gru_stream_oracle.py)
against the reference's offline greedy decode (tests/golden/gru_rnnt_tiny.npz), and PytorchStreamDecoder built from a
flagfile with ``enc_type='GRU'``."""
import os
import types

import numpy as np
import pytest
import torch

from tests.gru_stream_oracle import GRUStreamRestatement

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SMALL = dict(vocab_embed_size=8, vocab_size=16, input_size=12, enc_hidden_size=16, enc_layers=2, enc_dropout=0,
             enc_proj_size=16, dec_hidden_size=16, dec_layers=1, dec_dropout=0, dec_proj_size=16, joint_size=16)


def load_gru_rnnt_tiny():
    z = np.load(os.path.join(GOLDEN, "gru_rnnt_tiny.npz"))
    cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith("cfg_")}
    sd = {k[3:]: torch.as_tensor(z[k]) for k in z.files if k.startswith("sd.")}
    return z, cfg, sd


def _cpu(module_type="GRU", **over):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(0)
    return Transducer(output_loss=False, module_type=module_type, **dict(SMALL, **over))


class Tok:
    vocab_size = 16

    class tokenizer:
        @staticmethod
        def id_to_token(i):
            return "<unk>" if i == 3 else "t%d</w>" % i

        @staticmethod
        def token_to_id(t):
            return 3 if t == "<unk>" else None


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_greedy_engine_refusals_come_before_any_device_work():
    """GRUStreamEngine, and StreamEngine on an LSTM encoder with the same checks in the same order."""
    from edgedict_b200.stream_engine import GRUStreamEngine, StreamEngine
    cuda_before = torch.cuda.is_initialized()
    for engine, model, other in ((GRUStreamEngine, _cpu(), "GRU"), (StreamEngine, _cpu("LSTM"), "LSTM")):
        with pytest.raises(ValueError, match=other + " encoder"):
            engine(_cpu("LSTM" if other == "GRU" else "GRU"), 1, 2)
        for S, n in ((0, 2), (-1, 2), (2, 0), (2, -2)):
            with pytest.raises(ValueError, match="positive"):
                engine(model, S, n)
        for n in (1, 3, 7):                               # the time reduction after layer 1 pairs frames
            with pytest.raises(ValueError, match="even number of frames"):
                engine(model, 2, n)
        for K in (0, 17):
            with pytest.raises(ValueError, match="max_symbols"):
                engine(model, 2, 2, max_symbols=K)
        with pytest.raises(RuntimeError, match="CUDA"):    # a CPU model, every other argument valid
            engine(model, 2, 4)
    assert torch.cuda.is_initialized() == cuda_before


@pytest.mark.parametrize("what,args,kw", [
    ("W = 0", (1, 4, 0), {}),
    ("W too large", (1, 4, 1025), {}),
    ("max_pending < n_out", (1, 8, 4), dict(max_pending=3)),
    ("max_pending < n_out * max_symbols", (1, 4, 4), dict(max_pending=3, max_symbols=2)),
    ("lm_weight without lm", (1, 4, 4), dict(lm_weight=0.5)),
    ("malformed lm state_dict", (1, 4, 4), dict(lm={"encoder.weight": torch.zeros(3, 2)})),
    ("odd chunk before a time reduction", (1, 3, 4), {}),
    ("no streams", (0, 4, 4), {}),
    ("an LSTM encoder", (1, 4, 4), dict(lstm=True)),
])
def test_beam_engine_refusals_come_before_any_device_work(what, args, kw):
    from edgedict_b200.stream_engine import GRUStreamBeamEngine
    cuda_before = torch.cuda.is_initialized()
    m = _cpu("LSTM" if kw.pop("lstm", False) else "GRU")
    with pytest.raises(ValueError, match="GRU encoder" if what == "an LSTM encoder" else None):
        GRUStreamBeamEngine(m, *args, **kw)
    assert torch.cuda.is_initialized() == cuda_before


def test_beam_engine_needs_a_cuda_model():
    from edgedict_b200.stream_engine import GRUStreamBeamEngine
    cuda_before = torch.cuda.is_initialized()
    with pytest.raises(RuntimeError, match="CUDA"):
        GRUStreamBeamEngine(_cpu(), 1, 4, 4)
    assert torch.cuda.is_initialized() == cuda_before


def test_stream_decoder_refusals_on_a_gru_model_come_before_any_device_work():
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    cuda_before = torch.cuda.is_initialized()
    for kw in (dict(), dict(beam_width=4)):
        with pytest.raises(ValueError, match="even number of frames"):
            PytorchStreamDecoder(FLAGS=None, transducer=_cpu(), transform=lambda f: f, tokenizer=Tok(), device="cpu",
                                 frames_per_chunk=3, **kw)
        with pytest.raises(RuntimeError, match="CUDA"):
            PytorchStreamDecoder(FLAGS=None, transducer=_cpu(), transform=lambda f: f, tokenizer=Tok(), device="cpu",
                                 frames_per_chunk=4, **kw)
    assert torch.cuda.is_initialized() == cuda_before


# ---- C ABI -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def L():
    from edgedict_b200 import build
    from edgedict_b200._lib import lib
    build.build()
    return lib()


P = 1 << 20                                                   # a plausible, aligned, never dereferenced address


def test_run_entry_validates_its_arguments(L):
    run = L.eb_decode_run_gru_rnnt
    assert run(None, 3, P, 0, None) == 2
    assert run(P, 3, None, 0, None) == 2
    for nphase in (0, -1):
        assert run(P, nphase, P, 0, None) == 2


# ---- chunking semantics ------------------------------------------------------------------------------------------------
MIXED = [6, 2, 4, 2, 8, 2, 6, 4, 10, 2, 4, 2, 6, 4, 2, 6, 2, 4, 6, 10, 4]       # 96 frames


@pytest.mark.parametrize("lens", [[2] * 48, [4] * 24, MIXED])
def test_restatement_over_chunks_is_the_reference_greedy_decode(lens):
    """The fixture's 96 frames streamed in even chunks with h carried: the ids of every encoder frame, blanks
    included, are the reference's offline greedy_decode ids."""
    z, _, sd = load_gru_rnnt_tiny()
    xs = torch.as_tensor(z["xs"])[None]
    assert sum(lens) == xs.shape[1]
    rs = GRUStreamRestatement(sd, 1)
    got, t0 = [], 0
    for n in lens:
        got += rs.step(xs[:, t0:t0 + n])[0].tolist()
        t0 += n
    assert got == z["greedy_ids"].tolist()
    assert rs.hit_unk == 0 and sum(k != 0 for k in got) >= 10


def test_restatement_streams_are_independent():
    """With several streams the restatement keeps them independent: each stream of a batch of 3 is its S = 1 run."""
    z, _, sd = load_gru_rnnt_tiny()
    g = torch.Generator().manual_seed(4)
    xs = torch.randn(3, 24, 12, generator=g) * 1.5
    for K in (1, 3):
        rs = GRUStreamRestatement(sd, 3, max_symbols=K)
        got = torch.cat([rs.step(xs[:, t:t + 4]) for t in range(0, 24, 4)], 1)
        for s in range(3):
            one = GRUStreamRestatement(sd, 1, max_symbols=K)
            want = torch.cat([one.step(xs[s:s + 1, t:t + 4]) for t in range(0, 24, 4)], 1)
            assert torch.equal(got[s], want[0]), (K, s)


# ---- PytorchStreamDecoder from a flagfile --------------------------------------------------------------------------------
def test_stream_decoder_builds_a_gru_transducer_from_flags(tmp_path, monkeypatch):
    """enc_type='GRU' (the reference's flag, rnnt/args.py) builds Transducer(module_type='GRU') and loads a checkpoint
    written by it; without enc_type the model is the LSTM one, as before."""
    from edgedict_b200.rnnt.models import ResLayerNormGRU, ResLayerNormLSTM
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    src = _cpu(enc_hidden_size=20)
    sd = {k: v.detach().clone() for k, v in src.state_dict().items()}
    flags = dict(name="gru_run", model_name="last.pt", bpe_size=16, feature_size=4, downsample=3, delta=False,
                 vocab_embed_size=8, enc_hidden_size=20, enc_layers=2, enc_dropout=0, enc_proj_size=16,
                 dec_hidden_size=16, dec_layers=1, dec_dropout=0, dec_proj_size=16, joint_size=16)
    os.makedirs(tmp_path / "logs" / "gru_run" / "models")
    torch.save({"model": sd}, tmp_path / "logs" / "gru_run" / "models" / "last.pt")
    monkeypatch.chdir(tmp_path)
    dec = PytorchStreamDecoder(types.SimpleNamespace(enc_type="GRU", **flags), transform=lambda f: f, tokenizer=Tok(),
                               device="cpu")
    assert isinstance(dec.encoder.lstm, ResLayerNormGRU)
    got = dec._transducer.state_dict()
    assert set(got) == set(sd)
    for k, v in sd.items():
        assert torch.equal(got[k], v), k
    # an LSTM flagfile (no enc_type) builds the LSTM model: the GRU checkpoint does not fit it
    with pytest.raises(RuntimeError):
        PytorchStreamDecoder(types.SimpleNamespace(**flags), transform=lambda f: f, tokenizer=Tok(), device="cpu")
    lstm = _cpu("LSTM", enc_hidden_size=20)
    torch.save({"model": lstm.state_dict()}, tmp_path / "logs" / "gru_run" / "models" / "last.pt")
    dec = PytorchStreamDecoder(types.SimpleNamespace(**flags), transform=lambda f: f, tokenizer=Tok(), device="cpu")
    assert isinstance(dec.encoder.lstm, ResLayerNormLSTM)
