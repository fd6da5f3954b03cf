"""Wav2vec pre-training without a GPU: the engine's seeded construction against the reference's weights bit for bit
(tests/golden/wav2vec_tiny.npz), the engine's span and negative draws against the reference's, the fp64 restatement of
the head (tests/wav2vec_oracle.py) against the reference, the cosine semantics, the refusals before any device work and
the argument checks of the C entries."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from tests import wav2vec_oracle as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FE = [(10, 5, 32)] + [(3, 2, 32)] * 2 + [(2, 2, 32)]
TINY = dict(frontend_params=FE, front_bias=False, input_size=32, enc_hidden_size=32, enc_layers=2, enc_dropout=0.0,
            enc_proj_size=16, num_negatives=10, latent_vars=16, mask_prob=0.3, mask_length=3)
CONFIGS = {             # tests/golden/make_golden_wav2vec.py
    "cli": dict(TINY, quantize_targets=True),
    "dflt": dict(enc_dropout=0.0),
    "qin": dict(TINY, quantize_targets=True, quantize_input=True, same_quantizer=True),
    "embed": dict(TINY, quantize_targets=True, input_size=40, final_dim=24, latent_dim=16, latent_groups=2),
    "gru": dict(TINY, quantize_targets=True, module_type="GRU"),
}


SAMPLE_WHOLE, SAMPLE_N = 512, 128          # tests/golden/make_golden_wav2vec.py


def golden():
    return np.load(os.path.join(GOLDEN, "wav2vec_tiny.npz"))


def _sha(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def audio(z):
    """The fixture's input waveforms [3, 4000], regenerated from their seed and checked against their digest."""
    x = 0.3 * torch.randn(3, 4000, generator=torch.Generator().manual_seed(2))
    assert _sha(x) == str(z["x_sha"])
    return x


def recorded_noise(z, pre):
    """The Gumbel noise of each quantizer call of a fixture step (keys pre + 'noise<i>.*'), in call order: drawn on the
    CPU from its recorded seed as F.gumbel_softmax drew it, checked against its digest, the caller's generator untouched."""
    out, i = [], 0
    while "%snoise%d.seed" % (pre, i) in z:
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(int(z["%snoise%d.seed" % (pre, i)]))
            n = -torch.empty(tuple(int(d) for d in z["%snoise%d.shape" % (pre, i)])).exponential_().log()
        assert _sha(n) == str(z["%snoise%d.sha" % (pre, i)])
        out.append(n)
        i += 1
    return out


def sample(gr):
    gr = gr.reshape(-1)
    return gr if gr.numel() <= SAMPLE_WHOLE else gr[::-(-gr.numel() // SAMPLE_N)]


def seeded(tag, z=None):
    from edgedict_b200.rnnt.wav2vec import Wav2Vec
    z = golden() if z is None else z
    torch.manual_seed(int(z[tag + ".seed"]))
    return Wav2Vec(**CONFIGS[tag])


@pytest.mark.parametrize("tag", list(CONFIGS))
def test_seeded_wav2vec_equals_the_reference_state_dict(tag):
    z = golden()
    sd = seeded(tag, z).state_dict()
    assert list(sd) == [str(k) for k in z[tag + ".keys"]]
    for k, t in sd.items():
        assert hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest() == str(z[tag + ".sha." + k]), k


@pytest.mark.parametrize("mask_type,other", [("static", 0.0), ("uniform", 1), ("normal", 2.0), ("poisson", 0.0)])
def test_mask_draw_equals_the_reference(mask_type, other):
    from edgedict_b200.rnnt.wav2vec import compute_mask_indices
    np.random.seed(7)
    m = compute_mask_indices((4, 57), None, 0.3, 4, mask_type, other, min_masks=2)
    assert np.array_equal(m, golden()["maskdraw." + mask_type])
    assert len(set(m.sum(1))) == 1


def test_negative_draw_equals_the_reference():
    from edgedict_b200.rnnt.wav2vec import sample_negative_indices
    torch.manual_seed(8)
    assert np.array_equal(sample_negative_indices(3, 9, 7).numpy(), golden()["negdraw"])


def test_step_draws_equal_the_reference():
    """With the fixture's seeds the engine's draws are the reference's: the step's spans (numpy) and negatives (torch's
    CPU generator, untouched by the Gumbel noise, which is drawn on the device)."""
    from edgedict_b200.rnnt.wav2vec import compute_mask_indices, sample_negative_indices
    z = golden()
    for tag in CONFIGS:
        seed = int(z[tag + ".seed"])
        mask = z[tag + ".mask"]
        np.random.seed(seed)
        m = seeded(tag, z)
        np.random.seed(seed)
        got = compute_mask_indices(mask.shape, None, m.mask_prob, m.mask_length, m.mask_selection, m.mask_other,
                                   min_masks=2, min_space=m.mask_min_space)
        assert np.array_equal(got, mask), tag
        torch.manual_seed(seed + 1000)
        M = int(mask[0].sum())
        assert np.array_equal(sample_negative_indices(mask.shape[0], M, m.n_negatives).numpy(), z[tag + ".neg"]), tag


def test_fixture_inputs_regenerate():
    """The audio and every Gumbel noise draw the fixture records by seed regenerate bit for bit."""
    z = golden()
    assert audio(z).shape == (3, 4000)
    for tag in CONFIGS:
        n = recorded_noise(z, tag + ".")
        assert len(n) == (0 if tag == "dflt" else 2 if tag == "qin" else 1), tag


def test_oracle_reproduces_the_reference():
    z = golden()
    m = seeded("cli", z)
    sd = {k: v.double() for k, v in m.state_dict().items()}
    q = m.quantizer
    B, M = z["cli.mask"].shape[0], int(z["cli.mask"][0].sum())
    y = torch.from_numpy(z["cli.features_masked"]).double().view(B, M, -1)
    xenc = torch.from_numpy(z["cli.enc_masked"]).double().view(B, M, -1)
    logits, loss, log = wo.head(sd, y, xenc, float(z["cli.features_pen"]), z["cli.neg"],
                                recorded_noise(z, "cli.")[0].double(), q.groups, q.curr_temp, m.logit_temp,
                                list(z["cli.weights"]))
    want = torch.from_numpy(z["cli.logits"]).double()
    fin = torch.isfinite(want)
    assert torch.equal(fin, torch.isfinite(logits))
    assert float((logits[fin] - want[fin]).abs().max()) < 1e-4
    names = [str(k) for k in z["cli.log_names"]]
    vals = dict(zip(names, z["cli.log_values"]))
    assert abs(float(loss) - float(z["cli.loss"])) < 1e-4 * abs(float(z["cli.loss"]))
    for k in ("loss_0", "loss_1", "loss_2", "prob_perplexity", "code_perplexity"):
        assert abs(float(log[k]) - vals[k]) < 1e-4 * max(1.0, abs(vals[k])), k
    assert log["correct"] == vals["correct"]


@pytest.mark.parametrize("sx,sy", [(1.0, 1.0), (1e-9, 1.0), (1e-9, 1e-5), (1.0, 1e-10)])
def test_oracle_cosine_is_torch_cosine_similarity(sx, sy):
    """Values and gradients of the restatement's cosine equal torch.cosine_similarity's, also where a norm is clamped
    at eps = 1e-8 (parallel vectors of norms 1e-9 and 1e-5 give 0.1)."""
    g = torch.Generator().manual_seed(3)
    xp = (torch.randn(1, 3, 6, generator=g, dtype=torch.float64) * sx).requires_grad_()
    yp = (torch.randn(1, 3, 6, generator=g, dtype=torch.float64) * sy).requires_grad_()
    neg = torch.tensor([[[1], [2], [0]]])
    lo = wo.contrastive_logits(xp, yp, neg, 1.0)
    cand = torch.stack([yp[0], yp[0, neg[0, :, 0]]])[:, None]
    want = torch.cosine_similarity(xp[None], cand, dim=-1)
    assert torch.allclose(lo, want, rtol=1e-12, atol=0)
    R = torch.randn(lo.shape, generator=g, dtype=torch.float64)
    ga = torch.autograd.grad((lo * R).sum(), (xp, yp))
    gb = torch.autograd.grad((want * R).sum(), (xp, yp))
    for a, b in zip(ga, gb):
        assert torch.allclose(a, b, rtol=1e-9, atol=1e-12 * float(b.abs().max()))
    e = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64)
    assert abs(float(torch.cosine_similarity(e * 1e-9, e * 1e-5, dim=-1)) - 0.1) < 1e-9
    par = wo.contrastive_logits((e * 1e-9).view(1, 1, 4).expand(1, 2, 4), torch.stack([e * 1e-5, e])[None],
                                torch.tensor([[[1], [0]]]), 1.0)
    assert abs(float(par[0, 0, 0]) - 0.1) < 1e-9


def _refuses(match, tag="cli", features_only=False, mask=True, padding_mask=None, prep=None, **over):
    from edgedict_b200.rnnt.wav2vec import Wav2Vec
    torch.manual_seed(0)
    m = Wav2Vec(**dict(CONFIGS[tag], **over))
    if prep:
        prep(m)
    with pytest.raises(ValueError, match=match):
        m(torch.zeros(2, 4000), padding_mask=padding_mask, mask=mask, features_only=features_only)


def test_refusals_raise_before_device_work():
    _refuses("padding_mask", padding_mask=torch.zeros(2, 4000, dtype=torch.bool))
    _refuses("mask_channel_prob", mask_channel_prob=0.1)
    _refuses("no_mask_overlap", no_mask_overlap=True)
    _refuses("negatives_from_everywhere", negatives_from_everywhere=True)
    _refuses("eval mode", tag="dflt", prep=lambda m: m.eval())
    _refuses("cross_sample_negatives", cross_sample_negatives=2)
    _refuses("codebook_negatives", codebook_negatives=2)
    _refuses("target_glu", target_glu=True)
    _refuses("mask=False", mask=False)
    _refuses("num_negatives", num_negatives=0)
    _refuses("mask selection", mask_selection="gamma")
    _refuses("multiples of 8", latent_vars=15, prep=lambda m: m.set_precision("bf16"))
    _refuses("multiples of 8", final_dim=20, prep=lambda m: m.set_precision("bf16"))
    _refuses("CUDA")                                          # CPU audio: no CPU path
    _refuses("CUDA", features_only=True, mask=False)


def test_criterion_refusals():
    from edgedict_b200.rnnt.wav2vec import ConstrastiveCriterion, Wav2Vec
    torch.manual_seed(0)
    m = Wav2Vec(**CONFIGS["dflt"])
    with pytest.raises(ValueError, match="infonce"):
        ConstrastiveCriterion()(m, torch.zeros(2, 4000))
    with pytest.raises(ValueError, match="loss weights"):
        ConstrastiveCriterion(infonce=True, loss_weights=[0.1, 10])(m, torch.zeros(2, 4000))


def test_set_num_updates():
    from edgedict_b200.rnnt.wav2vec import GumbelVectorQuantizer
    q = GumbelVectorQuantizer(8, 16, (2, 0.5, 0.999995), 2, False, 8, True)
    for n in (0, 1, 1000, 10 ** 6):
        q.set_num_updates(n)
        assert q.curr_temp == max(2 * 0.999995 ** n, 0.5)


def test_c_entries_check_their_arguments():
    from edgedict_b200._lib import lib
    L = lib()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert L.eb_w2v_mask_fwd(None, p, p, p, 4, 4, None) == 2
    assert L.eb_w2v_mask_fwd(p, p, p, p, 0, 4, None) == 2
    assert L.eb_w2v_keep_rows(p, None, p, 4, 4, None) == 2
    assert L.eb_w2v_gather(p, p, p, 2, 3, 4, 4, None) == 2                     # M > T
    assert L.eb_w2v_scatter(p, p, None, 2, 3, 2, 4, None) == 2
    assert L.eb_w2v_sq_mean(p, 0, p, None) == 2
    assert L.eb_w2v_scale(p, None, 1.0, 4, p, None) == 2
    assert L.eb_w2v_quant_fwd(p, p, p, 4, 2, 8, 4, 0.0, p, p, p, p, p, p, p, None) == 2   # tau <= 0 with noise
    assert L.eb_w2v_quant_fwd(p, None, p, 4, 0, 8, 4, 1.0, p, p, p, p, p, p, p, None) == 2
    assert L.eb_w2v_quant_stats(p, p, 4, 2, 8, p, None, p, None) == 2
    assert L.eb_w2v_quant_bwd(p, None, p, p, None, 4, 2, 8, 1.0, p, None) == 2         # dsoft without s
    assert L.eb_w2v_logits_fwd(p, p, p, 2, 1, 4, 3, 0.1, 1e-8, p, p, p, p, p, p, None) == 2   # M < 2
    assert L.eb_w2v_logits_fwd(p, p, p, 2, 3, 4, 3, 0.0, 1e-8, p, p, p, p, p, p, None) == 2   # temp 0
    assert L.eb_w2v_logits_bwd(p, p, p, p, p, p, p, p, p, 2, 3, 4, 0, 0.1, 1e-8, p, p, p, p, None) == 2
    assert L.eb_w2v_ce(p, 2, 3, 1, p, p, None) == 2


# ---- tests/w2v_restate.py, the per-kernel restatement of test_gpu_w2v_fp64.py, pinned to the oracle ---------------
def test_restate_lane_argmax_is_the_first_index_argmax():
    """Without NaN the kernels' lane map is torch's first-index argmax / argmin, ties across and within lanes included;
    a NaN a lane meets first sticks in that lane, a later one is skipped."""
    from tests import w2v_restate as rs
    g = torch.Generator().manual_seed(1)
    for n in (1, 2, 31, 32, 33, 70, 1100):
        v = torch.randint(-3, 4, (200, n), generator=g).float()        # many ties
        assert torch.equal(rs.lane_arg(v.numpy()), v.argmax(-1)), n
        assert torch.equal(rs.lane_arg(v.numpy(), largest=False), v.argmin(-1)), n
    v = torch.arange(70.0).repeat(3, 1)
    v[0, 0] = v[1, 37] = v[2, 69] = float("nan")
    assert rs.lane_arg(v.numpy()).tolist() == [0, 69, 68]


def test_restate_quantizer_is_the_oracle():
    """k, the perplexities (from psum = sum_r p) and d logits = quant_bwd(dsoft = dq vars^T, g_ppl) of the restatement
    equal wav2vec_oracle.quantize and its fp64 autograd."""
    from tests import w2v_restate as rs
    g = torch.Generator().manual_seed(2)
    N, G, V, vd, tau = 37, 3, 20, 5, 1.7
    tau = float(np.float32(tau))
    logits = (3 * torch.randn(N, G * V, generator=g)).double().requires_grad_()
    noise = -torch.empty(N, G * V).exponential_(generator=g).log().double()
    vars = torch.rand(G * V, vd, generator=g).double()
    q, pp, cp, k, _ = wo.quantize(logits, vars, noise, G, tau)
    R = torch.randn(N, G * vd, generator=g).double()
    ((q * R).sum() + 3.0 * pp).backward()
    pp, cp = pp.detach(), cp.detach()
    z = ((logits.detach() + noise) / tau).view(N * G, V)
    s, _ = rs.softmax(z, V)
    p, _ = rs.softmax(logits.detach().view(N * G, V), V)
    assert torch.equal(s.argmax(-1).view(N, G), k)
    k0 = logits.detach().view(N, G, V).argmax(-1)
    st = rs.quant_stats(p.view(N, G * V).sum(0), k0, N, G, V)
    assert abs(float(st["pp"]) - float(pp)) < 1e-12 * float(pp) and abs(float(st["cp"]) - float(cp)) < 1e-12 * float(cp)
    ds = torch.einsum("ngd,gvd->ngv", R.view(N, G, vd), vars.view(G, V, vd)).reshape(N, G * V)
    dl, _ = rs.quant_bwd(ds, s.view(N, -1), p.view(N, -1), st["coef"], torch.tensor([3.0], dtype=torch.float64), N, G,
                         V, tau)
    assert float((dl - logits.grad).abs().max()) < 1e-12 * float(logits.grad.abs().max())


def test_restate_cosine_logits_and_gradients_are_the_oracle():
    """normalize + logits_fwd equal contrastive_logits (the -inf included), and logits_a + logits_bwd under a dense
    upstream gradient, nonzero at the masked candidates, equal its fp64 autograd: a masked candidate passes nothing."""
    from tests import w2v_restate as rs
    g = torch.Generator().manual_seed(3)
    B, M, D, K, temp, eps = 2, 12, 9, 6, float(np.float32(0.1)), float(np.float32(1e-8))
    xp, yp = torch.randn(B, M, D, generator=g), torch.randn(B, M, D, generator=g)
    yp[0, 5] = yp[0, 3]
    xp[1, 2] *= 1e-12
    yp[1, 4] = 0.0
    neg = torch.randint(0, M, (B, M, K), generator=g)
    neg[0, 3, 0], neg[0, 5, 1], neg[1, 6, 2] = 5, 3, 6
    X, Y = xp.double().requires_grad_(), yp.double().requires_grad_()
    want = wo.contrastive_logits(X, Y, neg, temp, eps)          # the kernel's float eps
    xh, _, xn, _ = rs.normalize(xp, eps)
    yh, _, yn, _ = rs.normalize(yp, eps)
    cos, _, lo, _ = rs.logits_fwd(xh, yh, yp, neg, temp)
    assert torch.equal(lo.isinf(), want.isinf()) and int(lo.isinf().sum()) >= 3
    fin = torch.isfinite(want)
    assert float((lo[fin] - want.detach()[fin]).abs().max()) < 1e-12 / temp
    R = torch.randn(want.shape, generator=g).double() + 3.0
    (torch.where(fin, want, torch.zeros_like(want)) * R).sum().backward()
    A, _, AC, _ = rs.logits_a(R, cos, neg, lo.isinf())
    dx, _, dy, _ = rs.logits_bwd(A, AC, xh, yh, xp, yp, xn, yn, temp, eps)
    for got, ref in ((dx, X.grad), (dy, Y.grad)):
        assert float((got - ref).abs().max()) < 1e-10 * float(ref.abs().max())


def test_restate_cross_entropy_is_the_oracle():
    from tests import w2v_restate as rs
    g = torch.Generator().manual_seed(4)
    C, B, M = 33, 3, 7
    lo = 5 * torch.randn(C, B, M, generator=g)
    lo[1:4, 1, 2] = -float("inf")
    lo[:, 2, 5] = 0.25
    lo[0, 0, 3] = lo[7, 0, 3] = 40.0
    X = lo.double().requires_grad_()
    loss, correct = wo.cross_entropy(X)
    loss.backward()
    r = rs.ce(lo)
    assert abs(r["loss"] - float(loss)) < 1e-12 * float(loss) and r["correct"] == correct
    assert float((r["grad"] - X.grad).abs().max()) < 1e-12
