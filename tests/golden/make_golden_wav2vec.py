"""Generates tests/golden/wav2vec_tiny.npz with the REFERENCE's own wav2vec pre-training (only possible where its
sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_wav2vec.py

* modules: ``rnnt.wav2vec.Wav2Vec`` and ``ConstrastiveCriterion(infonce=True)`` of $EDGEDICT_REFERENCE, torch CPU fp32,
  in five configurations (CONFIGS): cli/pretrain_wav2vec.py's constructor at tiny sizes (``cli``), the constructor's
  defaults (``dflt``, with enc_dropout=0 so the step replays; dropout builds no weights), quantize_input with
  same_quantizer (``qin``), embed != input_size with final_dim and latent_dim (``embed``) and module_type='GRU' (``gru``);
* input: B = 3 waveforms of 4000 samples drawn from a seeded torch generator (``audio``; the fixture keeps their SHA-256);
* per configuration: the SHA-256 of every tensor of the seeded initial state_dict, the mask and the negatives the
  reference drew (negatives as frame indices within the utterance), the Gumbel noise of each quantizer call as the
  seed it was drawn from, its shape and its SHA-256 (``gumbel_draw``: drawn inside a forked generator, so the CPU
  generator the negatives come from is left as the engine leaves it), the logits, the loss, every logging_output value,
  and every parameter gradient through ``sample`` (whole up to SAMPLE_WHOLE elements, else about SAMPLE_N evenly
  strided elements); for ``cli`` also the oracle's inputs -- the front end's and the encoder's outputs at the masked
  frames and the features penalty -- and an eval-mode call (targets and logging values);
* the reference's compute_mask_indices under fixed numpy seeds for the four mask types, and sample_negatives' draw
  under fixed torch seeds.

The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
FE = [(10, 5, 32)] + [(3, 2, 32)] * 2 + [(2, 2, 32)]
TINY = dict(frontend_params=FE, front_bias=False, input_size=32, enc_hidden_size=32, enc_layers=2, enc_dropout=0.0,
            enc_proj_size=16, num_negatives=10, latent_vars=16, mask_prob=0.3, mask_length=3)
CONFIGS = {
    "cli": dict(kw=dict(TINY, quantize_targets=True), weights=[0.1, 10.0], seed=21),
    "dflt": dict(kw=dict(enc_dropout=0.0), weights=[10.0], seed=22),
    "qin": dict(kw=dict(TINY, quantize_targets=True, quantize_input=True, same_quantizer=True), weights=[0.1, 10.0],
                seed=23),
    "embed": dict(kw=dict(TINY, quantize_targets=True, input_size=40, final_dim=24, latent_dim=16, latent_groups=2),
                  weights=[0.1, 10.0], seed=24),
    "gru": dict(kw=dict(TINY, quantize_targets=True, module_type="GRU"), weights=[0.1, 10.0], seed=25),
}
LOG_KEYS = ["prob_perplexity", "code_perplexity", "temp"]
B, L = 3, 4000
SAMPLE_WHOLE, SAMPLE_N = 512, 128
MASK_TYPES = {"static": 0.0, "uniform": 1, "normal": 2.0, "poisson": 0.0}


def digest(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def audio():
    return 0.3 * torch.randn(B, L, generator=torch.Generator().manual_seed(2))


def gumbel_draw(seed, shape):
    """The noise F.gumbel_softmax draws on the CPU after torch.manual_seed(seed), leaving the caller's generator as it was."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        return -torch.empty(shape).exponential_().log()


def sample(gr):
    """A flattened gradient, whole up to SAMPLE_WHOLE elements, else every ceil(n / SAMPLE_N)-th element."""
    gr = gr.reshape(-1)
    return gr if gr.size <= SAMPLE_WHOLE else gr[::-(-gr.size // SAMPLE_N)]


def reference():
    if "tokenizers" not in sys.modules:
        mod = sys.modules["tokenizers"] = types.ModuleType("tokenizers")
        mod.CharBPETokenizer = object
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    import rnnt.wav2vec as w  # (the reference)
    import rnnt.data_utils as du
    return w, du


def main():
    w, du = reference()
    g = torch.Generator().manual_seed(3)
    x = audio()
    save = dict(x_sha=np.array(digest(x)), log_keys=np.array(LOG_KEYS))
    real_gumbel = w.F.gumbel_softmax
    real_mask = w.compute_mask_indices
    for tag, c in CONFIGS.items():
        torch.manual_seed(c["seed"])
        m = w.Wav2Vec(**c["kw"])
        sd = m.state_dict()
        save.update({"%s.sha.%s" % (tag, k): np.array(digest(t)) for k, t in sd.items()})
        save["%s.keys" % tag] = np.array(list(sd.keys()))
        save["%s.seed" % tag] = np.int64(c["seed"])
        save["%s.weights" % tag] = np.array(c["weights"], dtype=np.float64)
        rec = dict(noise=[], mask=[], neg=[])

        def gumbel(logits, tau=1, hard=False, _rec=rec):
            s = int(torch.randint(0, 2 ** 31, (1,), generator=g))
            noise = gumbel_draw(s, logits.shape)
            _rec["noise"].append((s, noise))
            with torch.random.fork_rng(devices=[]):
                torch.manual_seed(s)
                out = real_gumbel(logits, tau=tau, hard=hard)
            assert torch.equal(((logits + noise) / tau).softmax(-1).argmax(-1), out.argmax(-1))
            return out

        def mask_fn(*a, _rec=rec, **kw):
            out = real_mask(*a, **kw)
            _rec["mask"].append(out)
            return out

        real_sn = m.sample_negatives

        def sample_negatives(y, num, _rec=rec):
            negs, idx = real_sn(y, num)
            _rec["neg"].append((idx - torch.arange(y.shape[0])[:, None] * num).numpy())
            return negs, idx

        outs = {}
        real_fwd = m.forward

        def fwd(*a, **kw):
            r = real_fwd(*a, **kw)
            outs.update(r)
            return r

        m.sample_negatives, m.forward = sample_negatives, fwd
        if tag == "cli":
            fe_out = m.frontend(x).detach()
        w.F.gumbel_softmax, w.compute_mask_indices = gumbel, mask_fn
        try:
            crit = w.ConstrastiveCriterion(infonce=True, loss_weights=list(c["weights"]), log_keys=LOG_KEYS)
            np.random.seed(c["seed"])
            torch.manual_seed(c["seed"] + 1000)
            if tag == "cli":
                enc = []
                h = m.encoder.register_forward_hook(lambda mod, i, o: enc.append(o[0].detach().numpy()))
            loss, ss, lo = crit(m, x)
            if tag == "cli":
                h.remove()
                mk = torch.from_numpy(rec["mask"][0])
                save["cli.features_masked"] = fe_out[mk].numpy()
                save["cli.features_pen"] = np.float64(outs["features_pen"].item())
                save["cli.enc_masked"] = enc[0][mk.numpy()]
            loss.backward()
            # the engine draws the negatives from the CPU generator as it stands after the seed
            torch.manual_seed(c["seed"] + 1000)
            M = rec["neg"][0].shape[1] // m.n_negatives
            tszs = torch.arange(M).unsqueeze(-1).expand(-1, m.n_negatives).flatten()
            want = torch.randint(low=0, high=M - 1, size=(B, m.n_negatives * M))
            want[want >= tszs] += 1
            assert np.array_equal(want.numpy(), rec["neg"][0]), "the CPU generator moved before the negatives"
            save["%s.mask" % tag] = rec["mask"][0]
            save["%s.neg" % tag] = rec["neg"][0]
            for i, (s, n) in enumerate(rec["noise"]):
                save["%s.noise%d.seed" % (tag, i)] = np.int64(s)
                save["%s.noise%d.shape" % (tag, i)] = np.array(n.shape, dtype=np.int64)
                save["%s.noise%d.sha" % (tag, i)] = np.array(digest(n))
            save["%s.logits" % tag] = outs["x"].detach().numpy()
            save["%s.loss" % tag] = np.float64(loss.item())
            save["%s.log_names" % tag] = np.array(list(lo.keys()))
            save["%s.log_values" % tag] = np.array([float(v) for v in lo.values()])
            save["%s.no_grad" % tag] = np.array([k for k, p in m.named_parameters() if p.grad is None])
            for k, p in m.named_parameters():
                if p.grad is None:
                    continue
                save["%s.grad.%s" % (tag, k)] = sample(p.grad.numpy()).copy()
            if tag == "cli":
                m.eval()
                rec["mask"].clear(), rec["neg"].clear()
                outs.clear()
                np.random.seed(c["seed"] + 1)
                torch.manual_seed(c["seed"] + 2000)
                with torch.no_grad():
                    _, _, lo = crit(m, x)
                save["cli.eval.mask"] = rec["mask"][0]
                save["cli.eval.neg"] = rec["neg"][0]
                save["cli.eval.targets"] = outs["targets"].numpy()
                save["cli.eval.logits"] = outs["x"].numpy()
                save["cli.eval.log_names"] = np.array(list(lo.keys()))
                save["cli.eval.log_values"] = np.array([float(v) for v in lo.values()])
        finally:
            w.F.gumbel_softmax, w.compute_mask_indices = real_gumbel, real_mask
        print(tag, "loss", loss.item(), lo)
    for mt, other in MASK_TYPES.items():
        np.random.seed(7)
        save["maskdraw.%s" % mt] = du.compute_mask_indices((4, 57), None, 0.3, 4, mt, other, min_masks=2)
    torch.manual_seed(8)
    save["negdraw"] = sample_draw(w, 3, 9, 7)
    np.savez_compressed(os.path.join(HERE, "wav2vec_tiny.npz"), **save)


def sample_draw(w, b, num, K):
    m = types.SimpleNamespace(n_negatives=K, cross_sample_negatives=0)
    y = torch.zeros(b, num, 2)
    _, idx = w.Wav2Vec.sample_negatives(m, y, num)
    return (idx - torch.arange(b)[:, None] * num).numpy()


if __name__ == "__main__":
    main()
    print("wav2vec_tiny.npz", os.path.getsize(os.path.join(HERE, "wav2vec_tiny.npz")) // 1024, "KiB")
