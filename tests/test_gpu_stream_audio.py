"""Stream engines fed raw audio: the front-end phases at the head of the chunk launch write into the engine's input
bit for bit what build_batch_transform's test module gives each stream's window (every feature type, deltas,
downsampling, both pad_to_divisible settings, dither, several stream counts and grid sizes), and every engine decodes
audio to the same ids, scores and state as its twin fed those features."""
import numpy as np
import pytest
import torch

from edgedict_b200.rnnt.features import build_batch_transform

pytestmark = pytest.mark.gpu
DEV = "cuda"
E6D2_L = 1320                                  # win 320 + hop 200 * (3 * 2 - 1): youtube_live.py's window


def _audio(S, L, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(L) / 16000.0
    x = 0.05 * torch.randn(S, L, generator=g)
    for s in range(S):
        x[s] += 0.4 * torch.sin(2 * np.pi * (150.0 + 37 * s) * t) + 0.1 * torch.sin(2 * np.pi * 2500.0 * t + s)
    return x.to(DEV)


def _transform(ft, delta, ds, ptd, C=80, dither=0.0, win=320):
    return build_batch_transform(ft, C, n_fft=512, win_length=win, hop_length=200, delta=delta, downsample=ds,
                                 pad_to_divisible=ptd, dither=dither)[1].to(DEV)


def _ctc(input_size, seed=0, H=32, layers=2, proj=24, V=24, scale=1.0):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(seed)
    m = CTCEncoder(vocab_size=V, input_size=input_size, enc_hidden_size=H, enc_layers=layers, enc_dropout=0,
                   proj_size=proj).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)
    return m.to(DEV)


def _transducer(input_size, module_type="LSTM", seed=0, scale=2.0, **over):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(seed)
    cfg = dict(vocab_embed_size=16, vocab_size=32, input_size=input_size, enc_hidden_size=48, enc_layers=3,
               enc_dropout=0, enc_proj_size=40, dec_hidden_size=32, dec_layers=2, dec_dropout=0, dec_proj_size=24,
               joint_size=56)
    cfg.update(over)
    m = Transducer(output_loss=False, module_type=module_type, **cfg).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(scale)                       # random-init weights emit only blanks; scale up so symbols appear
    return m.to(DEV)


FEATURE_CASES = [  # ft, delta, ds, ptd, L, S, max_ctas
    ("logfbank", False, 3, False, E6D2_L, 64, 0),
    ("logfbank", True, 3, True, E6D2_L, 7, 3),
    ("logfbank", False, 1, True, 1200, 1, 1),   # hop divides L: the seq_len mask zeroes the last frame
    ("logfbank", True, 1, False, 1200, 7, 17),
    ("melspec", False, 3, True, E6D2_L, 7, 0),
    ("melspec", True, 1, False, 1600, 1, 3),
    ("mfcc", False, 1, False, E6D2_L, 64, 17),
    ("mfcc", True, 3, True, 2600, 7, 1),
]


@pytest.mark.parametrize("ft,delta,ds,ptd,L,S,max_ctas", FEATURE_CASES)
def test_features_bitwise_batch_transform(ft, delta, ds, ptd, L, S, max_ctas):
    from edgedict_b200.stream_engine import StreamEngine
    tr = _transform(ft, delta, ds, ptd, C=40 if ft != "logfbank" else 80)
    m = _transducer(tr.input_size, enc_time_reductions=[])       # any frame count streams
    eng = StreamEngine(m, S, None, max_ctas=max_ctas, frontend=tr, samples_per_chunk=L)
    for i in range(2):
        x = _audio(S, L, 10 * i + S)
        want, wlen = tr(x, [L] * S)
        eng.step(x)
        assert eng.xin.shape == want.shape and (wlen == want.shape[1]).all()
        assert torch.equal(eng.xin, want), (ft, float((eng.xin - want).abs().max()))


def test_e6d2_features_against_the_fp64_oracle():
    from tests import features_batch_oracle as O
    from edgedict_b200.stream_engine import StreamEngine
    tr = _transform("logfbank", False, 3, False)
    x = _audio(64, E6D2_L, 5)
    eng = StreamEngine(_transducer(240), 64, None, frontend=tr, samples_per_chunk=E6D2_L)
    eng.step(x)
    from tests import features_fp64 as X
    want, _ = O.batch_transform(x.cpu().numpy().astype(np.float64), [E6D2_L] * 64, "logfbank", 80, n_fft=512,
                                win_length=320, hop_length=200, delta=False, downsample=3, pad_to_divisible=False)
    # test_gpu_features_batch.py's bar: the chain's propagated per-element bound, in table mode
    basis, fbT, dct, pre = X.module_tables(tr)
    te = X.tables_err("logfbank", basis, fbT, dct, 512, 80, pre)
    _, bar, ok = X.chain(x, [E6D2_L] * 64, "logfbank", basis, fbT, 512, 200, 3, False, False, preemph=pre,
                         tables_err=te)
    X.report("E6D2 window vs fp64 oracle", eng.xin, want, bar, ok)


def test_dither_bitwise():
    from edgedict_b200.stream_engine import StreamEngine
    tr = _transform("logfbank", False, 3, False, dither=1e-5)
    x = _audio(7, E6D2_L, 3)
    eng = StreamEngine(_transducer(240), 7, 2, frontend=tr, samples_per_chunk=E6D2_L)
    torch.manual_seed(123)
    eng.step(x)
    torch.manual_seed(123)
    want, _ = tr(x, [E6D2_L] * 7)
    assert torch.equal(eng.xin, want)
    torch.manual_seed(124)
    eng.step(x)
    assert not torch.equal(eng.xin, want)       # fresh noise every chunk


def _engine_pair(kind, S, L, tr):
    from edgedict_b200 import stream_engine as se
    n = tr.input_size
    if kind.startswith("ctc"):
        m = _ctc(n, scale=3.0)
        cls, kw = (se.CTCStreamEngine, {}) if kind == "ctc" else (se.CTCStreamBeamEngine, dict(W=4))
    else:
        gru = "gru" in kind
        m = _transducer(n, module_type="GRU" if gru else "LSTM")
        beam = "beam" in kind
        cls = {(False, False): se.StreamEngine, (False, True): se.StreamBeamEngine,
               (True, False): se.GRUStreamEngine, (True, True): se.GRUStreamBeamEngine}[gru, beam]
        kw = dict(W=4) if beam else {}
        if kind == "k2":
            kw = dict(max_symbols=2)
        if kind == "beam_lm":
            from edgedict_b200.models import LMModel
            torch.manual_seed(7)
            lm = LMModel(32, 16, 24, 1, dropout=0.0).to(DEV).eval()
            kw = dict(W=4, lm=lm, lm_weight=0.3, length_bonus=0.1)
    a = cls(m, S, None, frontend=tr, samples_per_chunk=L, **kw)
    b = cls(m, S, a.n, **kw)
    return a, b


def _same_state(a, b):
    sa, sb = a.state(), b.state()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k].cpu(), sb[k].cpu()), k


@pytest.mark.parametrize("kind", ["greedy", "k2", "beam", "beam_lm", "gru", "gru_beam", "ctc", "ctc_beam"])
def test_tokens_bitwise_against_features_twin(kind):
    S, L, chunks = 7, E6D2_L, 22
    tr = _transform("logfbank", False, 3, False)
    a, b = _engine_pair(kind, S, L, tr)
    emitted = 0
    for i in range(chunks):
        x = _audio(S, L, 100 + i)
        ra = a.step(x)
        rb = b.step(tr(x, [L] * S)[0])
        if isinstance(ra, tuple):
            for u, v in zip(ra, rb):
                assert torch.equal(u.cpu(), v.cpu())
            emitted += int(ra[1].sum())
        else:
            assert torch.equal(ra.cpu(), rb.cpu())
            emitted += int((ra != 0).sum())
    if "beam" in kind:
        fa, fb = a.flush(), b.flush()
        for u, v in zip(fa, fb):
            assert torch.equal(u.cpu(), v.cpu())
        emitted += int(fa[1].sum())
    if kind == "ctc":
        assert torch.equal(a.score(), b.score())
    _same_state(a, b)
    assert emitted > 0, "the model emits symbols"


def test_e6d2_large_64_streams_tokens():
    from edgedict_b200.stream_engine import StreamEngine
    tr = _transform("logfbank", False, 3, False)
    m = _transducer(240, seed=10, scale=2.0, vocab_embed_size=64, vocab_size=1024, enc_hidden_size=1024, enc_layers=6,
                    enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_proj_size=640, joint_size=640)
    a = StreamEngine(m, 64, None, frontend=tr, samples_per_chunk=E6D2_L)
    b = StreamEngine(m, 64, 2)
    for i in range(20):
        x = _audio(64, E6D2_L, 300 + i)
        assert torch.equal(a.step(x).cpu(), b.step(tr(x, [E6D2_L] * 64)[0]).cpu())
    _same_state(a, b)


def test_rebuild_on_a_short_last_window_and_reset():
    from edgedict_b200.stream_engine import StreamEngine
    tr = _transform("logfbank", False, 3, False)
    m = _transducer(240)
    S = 3
    a = StreamEngine(m, S, None, frontend=tr, samples_per_chunk=E6D2_L)
    b = StreamEngine(m, S, 2)
    for i in range(6):
        x = _audio(S, E6D2_L, 40 + i)
        assert torch.equal(a.step(x).cpu(), b.step(tr(x, [E6D2_L] * S)[0]).cpu())
    L2 = 3 * 200 * 4 + 120                      # 13 frames, 12 stacked into 4 input frames
    a2 = StreamEngine(m, S, None, frontend=tr, samples_per_chunk=L2, state=a.state())
    b2 = StreamEngine(m, S, 4, state=b.state())
    x = _audio(S, L2, 77)
    assert a2.n == 4 and torch.equal(a2.step(x).cpu(), b2.step(tr(x, [L2] * S)[0]).cpu())
    _same_state(a2, b2)
    a2.reset()
    b2.reset()
    x = _audio(S, L2, 78)
    assert torch.equal(a2.step(x).cpu(), b2.step(tr(x, [L2] * S)[0]).cpu())
    _same_state(a2, b2)


class _Tok:
    class tokenizer:
        @staticmethod
        def id_to_token(i):
            return "t%d</w>" % i

        @staticmethod
        def token_to_id(t):
            return 3


@pytest.mark.parametrize("beam", [None, 4])
def test_decoders_device_front_end_text(beam):
    import types
    from edgedict_b200.ctc import CTCStreamDecoder
    from edgedict_b200.rnnt.stream import PytorchStreamDecoder
    tr = _transform("logfbank", False, 3, False)
    host = lambda w: tr(w.to(DEV), [w.shape[1]])[0].transpose(1, 2)
    flags = types.SimpleNamespace(feature_size=80, downsample=3, delta=False)
    m = _transducer(240)
    mc = _ctc(240, scale=3.0)
    kw = {} if beam is None else dict(beam_width=beam)
    pairs = [(PytorchStreamDecoder(flags, m, tr, _Tok, **kw), PytorchStreamDecoder(flags, m, host, _Tok, **kw)),
             (CTCStreamDecoder(mc, tr, _Tok, **kw), CTCStreamDecoder(mc, host, _Tok, **kw))]
    wave = _audio(1, 1200 * 14 + 120 + 1100, 9).cpu()
    for dev_dec, host_dec in pairs:
        dev_dec.reset()
        host_dec.reset()
        texts = []
        for start in range(0, wave.shape[1] - E6D2_L, 1200):
            w = wave[:, start:start + E6D2_L]
            texts.append((dev_dec.decode(w), host_dec.decode(w)))
        w = wave[:, -1100:]                     # a shorter last window rebuilds and carries the state
        texts.append((dev_dec.decode(w), host_dec.decode(w)))
        texts.append((dev_dec.flush(), host_dec.flush()))
        assert all(u == v for u, v in texts), texts
