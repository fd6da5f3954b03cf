"""Stream engines fed raw audio (a device front end from build_batch_transform): every refusal is raised on the host
before any device work (the models live on the CPU here, so a check that came after the CUDA device check would raise
RuntimeError instead), and the frame arithmetic of the E6D2 streaming window."""
import pytest
import torch

from edgedict_b200.rnnt.features import build_batch_transform


def _transducer(input_size=240, module_type="LSTM"):
    from edgedict_b200.rnnt.models import Transducer
    torch.manual_seed(0)
    return Transducer(vocab_embed_size=8, vocab_size=16, input_size=input_size, enc_hidden_size=16, enc_layers=2,
                      enc_dropout=0, enc_proj_size=12, dec_hidden_size=8, dec_layers=1, dec_dropout=0,
                      dec_proj_size=12, joint_size=10, output_loss=False, module_type=module_type).eval()


def _ctc(input_size=240):
    from edgedict_b200.rnnt.models import CTCEncoder
    torch.manual_seed(0)
    return CTCEncoder(vocab_size=16, input_size=input_size, enc_hidden_size=16, enc_layers=2, enc_dropout=0,
                      proj_size=12).eval()


def _e6d2(**kw):
    args = dict(n_fft=512, win_length=320, hop_length=200, downsample=3, pad_to_divisible=False, dither=0)
    args.update(kw)
    return build_batch_transform("logfbank", 80, **args)


def _engines():
    from edgedict_b200 import stream_engine as se
    return [(se.StreamEngine, _transducer, {}), (se.StreamBeamEngine, _transducer, dict(W=2)),
            (se.GRUStreamEngine, lambda **k: _transducer(module_type="GRU", **k), {}),
            (se.GRUStreamBeamEngine, lambda **k: _transducer(module_type="GRU", **k), dict(W=2)),
            (se.CTCStreamEngine, _ctc, {}), (se.CTCStreamBeamEngine, _ctc, dict(W=2))]


def test_e6d2_window_frame_arithmetic():
    from edgedict_b200.stream_engine import check_stream_shape, frontend_geometry
    win, hop, ds, step_n_frame = 320, 200, 3, 2
    L = win + hop * (ds * step_n_frame - 1)                     # youtube_live.py's window
    assert (L, hop * ds * step_n_frame) == (1320, 1200)
    _, test, n = _e6d2()
    g = frontend_geometry(test, L)
    assert n == 240 and g["input_size"] == 240
    assert (g["F"], g["Fs"], g["T"], g["Fc"], g["seq"]) == (7, 6, 2, 6, 7)   # 7 frames, 6 stacked by 3 into 2
    assert (g["pad"], g["R"], g["Lp"]) == (256, 10, 2000)
    assert check_stream_shape(_transducer().encoder, 64, g["T"]) == (64, 2, 1)
    # pad_to_divisible pads the 7 frames to 9: 3 input frames; deltas read every frame
    g = frontend_geometry(_e6d2(pad_to_divisible=True, delta=True)[1], L)
    assert (g["F"], g["Fs"], g["T"], g["Fc"]) == (7, 7, 3, 7)
    # the seq_len mask zeroes the last frame when hop divides L: frame L / hop is past ceil(L / hop)
    g = frontend_geometry(_e6d2(downsample=1)[1], 1200)
    assert (g["F"], g["seq"], g["T"]) == (7, 6, 7)
    # melspec and MFCC carry no mask, no pre-emphasis and no dither
    for ft in ("melspec", "mfcc"):
        g = frontend_geometry(build_batch_transform(ft, 40, n_fft=512, win_length=400, hop_length=200)[1], 1320)
        assert (g["seq"], g["preemph"], g["use_mask"], g["dither"]) == (g["F"], None, False, 0.0)


@pytest.mark.parametrize("k", range(6))
def test_refusals_before_any_device_work(k):
    cls, model, kw = _engines()[k]
    m = model()
    train, test, _ = _e6d2(T_mask=5, T_num_mask=2)
    with pytest.raises(ValueError, match="SpecAugment"):
        cls(m, 2, None, frontend=train, samples_per_chunk=1320, **kw)
    with pytest.raises(ValueError, match="n_fft // 2"):
        cls(m, 2, None, frontend=test, samples_per_chunk=256, **kw)
    with pytest.raises(ValueError, match="even"):                # 1 + 800 // 200 = 5 frames -> 1 input frame
        cls(m, 2, None, frontend=test, samples_per_chunk=800, **kw)
    with pytest.raises(ValueError, match="no model input frame"):   # 3 frames, stacked by 3 without padding: none
        cls(m, 2, None, frontend=_e6d2(downsample=4)[1], samples_per_chunk=400, **kw)
    with pytest.raises(ValueError, match="disagrees"):
        cls(m, 2, 4, frontend=test, samples_per_chunk=1320, **kw)
    with pytest.raises(ValueError, match="input width"):
        cls(model(input_size=80), 2, None, frontend=test, samples_per_chunk=1320, **kw)
    with pytest.raises(ValueError, match="needs samples_per_chunk"):
        cls(m, 2, None, frontend=test, **kw)
    with pytest.raises(ValueError, match="needs a frontend"):
        cls(m, 2, 2, samples_per_chunk=1320, **kw)
    with pytest.raises(TypeError, match="BatchTransform"):
        cls(m, 2, None, frontend=lambda x: x, samples_per_chunk=1320, **kw)
    with pytest.raises(RuntimeError, match="CUDA"):               # every check passed: the device check is last
        cls(m, 2, None, frontend=test, samples_per_chunk=1320, **kw)


class _Fake:
    """What _load needs of an engine built with a front end (no device buffers are touched on refusal)."""

    def __init__(self):
        self._fe, self.dev = {}, torch.device("cuda", 0)
        self.audio = torch.empty(2, 1320, device="meta")


@pytest.mark.parametrize("bad", [torch.zeros(2, 1320),                         # wrong device
                                 torch.zeros(2, 1320, dtype=torch.float64),    # wrong dtype
                                 torch.zeros(2, 1321), torch.zeros(1, 2, 1320), [0.0] * 1320])
def test_chunk_refusals(bad):
    from edgedict_b200.stream_engine import _ChunkEngine
    with pytest.raises(ValueError, match="fp32 audio"):
        _ChunkEngine._load(_Fake(), bad)
