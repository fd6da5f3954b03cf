"""Generates tests/golden/lm_tiny.npz by running the REFERENCE's language model itself (only possible where its
sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_lm.py

* language model: the top-level ``models.LMModel`` of $EDGEDICT_REFERENCE (the LM cli/train_lm.py trains), torch CPU
  fp32, eval mode.

The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def LMModel(*args, **kw):
    """The reference's top-level models.LMModel.  Importing that module pulls in its audio and text front ends
    (speechpy, unidecode, inflect, modules.tokenizers), none of which LMModel uses: empty stand-ins satisfy the
    imports."""
    for name in ("speechpy", "speechpy.processing", "unidecode", "inflect", "modules.tokenizers"):
        if name not in sys.modules:
            mod = sys.modules[name] = types.ModuleType(name)
            mod.__getattr__ = lambda attr: (lambda *a, **k: None)
    sys.modules["speechpy"].processing = sys.modules["speechpy.processing"]
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    import modules
    modules.tokenizers = sys.modules["modules.tokenizers"]
    from models import LMModel as M  # (the reference)
    return M(*args, **kw)


def lm():
    """A small LMModel (ntoken 16, 2 layers), its state_dict, a token batch that starts with <bos> = 1 as
    cli/train_lm.py's seq_collate builds it, and the reference's log-probs and final (h, c) in eval mode."""
    torch.manual_seed(77)
    m = LMModel(16, 6, 10, 2, dropout=0.5).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(4.0)                              # peaked log-probs, so that the LM decides beam ranks in tests
    toks = torch.cat([torch.ones(3, 1, dtype=torch.long), torch.randint(0, 16, (3, 6))], 1)
    with torch.no_grad():
        logp, (h, c) = m(toks, m.init_hidden(3))
    save = {"sd." + k: v.numpy() for k, v in m.state_dict().items()}
    save.update(tokens=toks.numpy().astype(np.int32), logp=logp.view(3, 7, 16).numpy(), h=h.numpy(), c=c.numpy())
    np.savez_compressed(os.path.join(HERE, "lm_tiny.npz"), **save)
    print("lm: keys", sorted(m.state_dict()))


if __name__ == "__main__":
    lm()
    print("lm_tiny.npz", os.path.getsize(os.path.join(HERE, "lm_tiny.npz")) // 1024, "KiB")
