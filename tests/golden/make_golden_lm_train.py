"""Generates tests/golden/lm_train_tiny.npz by training-step arithmetic of the REFERENCE's language model itself (only
possible where its sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_lm_train.py

* language model: the top-level ``models.LMModel`` of $EDGEDICT_REFERENCE (what cli/train_lm.py trains), torch CPU
  fp32, dropout = 0, untied (``u.``) and with tied weights (``t.``);
* batch: token sequences of unequal lengths padded as cli/train_lm.py's ``seq_collate`` pads them, so the targets hold
  0s, which its ``nn.NLLLoss(ignore_index=0)`` ignores;
* per variant: the initial state_dict under a fixed seed, the log-probs and final (h, c) of ``forward`` from
  ``init_hidden`` and from a non-zero hidden state, the loss, and the gradient of every parameter.

The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import os

import numpy as np
import torch
from torch import nn
from torch.nn.utils.rnn import pad_sequence

from make_golden_lm import LMModel

HERE = os.path.dirname(os.path.abspath(__file__))
NTOKEN, LENS = 24, (7, 5, 3, 6)
VARIANTS = {"u": dict(ninp=8, nhid=12, seed=5, tie_weights=False), "t": dict(ninp=12, nhid=12, seed=6, tie_weights=True)}


def seq_collate(batches):
    """cli/train_lm.py's seq_collate."""
    outputs = pad_sequence(batches, batch_first=True, padding_value=0)
    inputs = torch.cat([torch.ones(outputs.shape[0], 1).long(), outputs], dim=1)
    return inputs[:, :-1], outputs


def main():
    torch.manual_seed(1)
    inputs, targets = seq_collate([torch.randint(2, NTOKEN, (n,)) for n in LENS])
    save = dict(inputs=inputs.numpy(), targets=targets.numpy(), ntoken=np.int64(NTOKEN), nlayers=np.int64(2))
    for tag, v in VARIANTS.items():
        torch.manual_seed(v["seed"])
        m = LMModel(NTOKEN, v["ninp"], v["nhid"], 2, dropout=0.0, tie_weights=v["tie_weights"])
        sd = m.state_dict()
        save.update({"%s.sd.%s" % (tag, k): t.numpy().copy() for k, t in sd.items()})
        save["%s.keys" % tag] = np.array(list(sd.keys()))
        B = inputs.shape[0]
        m.train()
        logp, (h, c) = m(inputs, m.init_hidden(B))
        loss = nn.NLLLoss(ignore_index=0)(logp, targets.flatten())
        loss.backward()
        save["%s.logp" % tag], save["%s.h" % tag], save["%s.c" % tag] = logp.detach().numpy(), h.detach().numpy(), \
            c.detach().numpy()
        save["%s.loss" % tag] = np.float32(loss.item())
        for k, p in m.named_parameters():
            save["%s.grad.%s" % (tag, k)] = p.grad.numpy().copy()
        g = torch.Generator().manual_seed(v["seed"] + 100)
        h0 = 0.5 * torch.randn(2, B, v["nhid"], generator=g)
        c0 = 0.5 * torch.randn(2, B, v["nhid"], generator=g)
        with torch.no_grad():
            logp0, (h1, c1) = m(inputs, (h0, c0))
        save.update({"%s.h0" % tag: h0.numpy(), "%s.c0" % tag: c0.numpy(), "%s.logp_h0" % tag: logp0.numpy(),
                     "%s.h_h0" % tag: h1.numpy(), "%s.c_h0" % tag: c1.numpy()})
        print(tag, "loss", loss.item(), "params", [k for k, _ in m.named_parameters()])
    np.savez_compressed(os.path.join(HERE, "lm_train_tiny.npz"), **save)


if __name__ == "__main__":
    main()
    print("lm_train_tiny.npz", os.path.getsize(os.path.join(HERE, "lm_train_tiny.npz")) // 1024, "KiB")
