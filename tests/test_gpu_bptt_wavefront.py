"""The chunked encoder backward (functional.LSTMStack._backward_wave: the BPTT in groups of time chunks, the group inputs
prepared on other streams under the layer above) against the serial schedule (functional.BPTT_WAVEFRONT = False) at
H = 1024: the output, dx and every parameter gradient are the same bits, with and without time reductions, with a ragged
last chunk, with C = 2 and the default C (groups of one, two and three chunks)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

H = 1024


def _run(net, x, w, wavefront):
    from edgedict_b200 import functional as Fn
    Fn.BPTT_WAVEFRONT = wavefront
    try:
        net.zero_grad()
        xi = x.clone().requires_grad_(True)
        y, _ = net(xi)
        (y * w[:, :y.shape[1]]).sum().backward()
        torch.cuda.synchronize()
    finally:
        Fn.BPTT_WAVEFRONT = True
    return y.detach().cpu(), xi.grad.cpu(), [p.grad.cpu().clone() for p in net.parameters()]


@pytest.mark.parametrize("B,T,L,red,chunks", [
    (32, 96, 3, (1,), 6),      # reductions, three even chunks
    (5, 100, 3, (1,), 6),      # reductions, ragged last chunk (odd length on the reduced axis)
    (32, 70, 2, (), 6),        # no reduction, ragged last chunk
    (7, 64, 3, (), 2),         # C = 2
    (32, 200, 4, (1,), 6),     # default C = 6 with reductions, ragged last chunk
])
def test_wavefront_backward_matches_serial_bitwise(B, T, L, red, chunks, monkeypatch):
    from edgedict_b200 import functional as Fn
    from edgedict_b200 import ops
    from edgedict_b200.rnnt.models import ResLayerNormLSTM
    reductions = [i in red for i in range(L)]
    monkeypatch.setattr(Fn, "WAVEFRONT_CHUNKS", chunks)
    plan = Fn.wavefront_plan(T, reductions)
    assert plan is not None and (len(plan[0]) == chunks or chunks == 6)
    torch.manual_seed(T + B)
    net = ResLayerNormLSTM(40, H, L, time_reductions=list(red)).cuda()
    for m in net.modules():
        m.precision = "bf16"
    x = torch.randn(B, T, 40).cuda()
    w = torch.randn(B, T, H).cuda()
    waves = []
    orig = Fn.LSTMStack._backward_wave
    monkeypatch.setattr(Fn.LSTMStack, "_backward_wave", staticmethod(lambda *a: (waves.append(1), orig(*a))[1]))
    y0, dx0, g0 = _run(net, x, w, False)
    assert not waves
    y1, dx1, g1 = _run(net, x, w, True)
    assert len(waves) == (1 if ops.lstm_c4_supported(B, H) and Fn._c4_bptt(H) else 0)
    assert torch.equal(y1, y0)
    assert torch.equal(dx1, dx0)
    for a, b, (name, _) in zip(g1, g0, net.named_parameters()):
        assert torch.equal(a, b), name
