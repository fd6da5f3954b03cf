"""Generates tests/golden/frontend_tiny.npz with the REFERENCE's own front end (only possible where its sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_frontend.py

* module: ``rnnt.models.FrontEnd`` of $EDGEDICT_REFERENCE, torch CPU fp32, in three configurations:
  ``train`` -- cli/train.py's ``[(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3`` with bias=True,
  ``pre``   -- the same parameters with bias=False, as cli/pretrain_wav2vec.py builds its Wav2Vec front end,
  ``dflt``  -- the constructor's defaults;
* input: B = 3 waveforms of unequal lengths, zero-padded to the longest (as seq_collate pads them);
* per configuration: the SHA-256 of every tensor of the seeded initial state_dict (its ~1 MB of weights are what
  the seed makes; the digests pin them bit for bit), the output, and every parameter gradient of sum(out * R) for a
  fixed R -- whole for tensors of up to SAMPLE_ABOVE elements, else the flattened gradient at every SAMPLE_STEP-th
  position, which keeps the fixture small.

The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import hashlib
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TRAIN = [(10, 5, 32)] + [(3, 2, 128)] * 4 + [(2, 2, 128)] * 3
DFLT = [(10, 5, 16)] + [(8, 4, 32)] + [(4, 2, 128)] * 3
CONFIGS = {"train": dict(params=TRAIN, bias=True, seed=11), "pre": dict(params=TRAIN, bias=False, seed=12),
           "dflt": dict(params=DFLT, bias=True, seed=13)}
LENS = (6400, 5130, 3877)
SAMPLE_ABOVE, SAMPLE_STEP = 4096, 31


def digest(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def FrontEnd(*args, **kw):
    """The reference's rnnt.models.FrontEnd.  rnnt.tokenizer imports the `tokenizers` package, which FrontEnd does not
    use: an empty stand-in satisfies the import."""
    if "tokenizers" not in sys.modules:
        mod = sys.modules["tokenizers"] = types.ModuleType("tokenizers")
        mod.CharBPETokenizer = object
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from rnnt.models import FrontEnd as F  # (the reference)
    return F(*args, **kw)


def main():
    g = torch.Generator().manual_seed(1)
    x = torch.zeros(len(LENS), max(LENS))
    for b, n in enumerate(LENS):
        x[b, :n] = 0.3 * torch.randn(n, generator=g)
    save = dict(x=x.numpy(), lens=np.array(LENS, dtype=np.int64))
    for tag, c in CONFIGS.items():
        torch.manual_seed(c["seed"])
        m = FrontEnd(frontend_params=c["params"], bias=c["bias"])
        save["%s.params" % tag] = np.array(c["params"], dtype=np.int64)
        save["%s.bias" % tag] = np.int64(c["bias"])
        save["%s.seed" % tag] = np.int64(c["seed"])
        sd = m.state_dict()
        save.update({"%s.sha.%s" % (tag, k): np.array(digest(t)) for k, t in sd.items()})
        save["%s.keys" % tag] = np.array(list(sd.keys()))
        out = m(x)
        R = torch.randn(out.shape, generator=torch.Generator().manual_seed(c["seed"] + 100))
        (out * R).sum().backward()
        save["%s.out" % tag], save["%s.R" % tag] = out.detach().numpy(), R.numpy()
        for k, p in m.named_parameters():
            gr = p.grad.numpy().reshape(-1)
            save["%s.grad.%s" % (tag, k)] = gr.copy() if gr.size <= SAMPLE_ABOVE else gr[::SAMPLE_STEP].copy()
        print(tag, tuple(out.shape))
    np.savez_compressed(os.path.join(HERE, "frontend_tiny.npz"), **save)


if __name__ == "__main__":
    main()
    print("frontend_tiny.npz", os.path.getsize(os.path.join(HERE, "frontend_tiny.npz")) // 1024, "KiB")
