"""Generates tests/golden/ctc_tiny.npz by running the REFERENCE's own CTCEncoder (rnnt/models.py:272-310, torch CPU fp32):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_ctc.py

The fixture holds the state_dict, the inputs, the log-probs, and the greedy ids and scores.  Utterance 2 is a constant
input (its argmax repeats frame after frame, so the collapse of repeats matters), utterance 3 is decoded with a large
blank bias (every frame blank: an empty result), and the xlen values include one above T' (the reference truncates by
the unscaled xlen).  The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from rnnt.models import CTCEncoder  # (the reference)
    torch.manual_seed(2024)
    cfg = dict(vocab_size=12, input_size=10, enc_hidden_size=16, enc_layers=2, enc_dropout=0, proj_size=14)
    m = CTCEncoder(**cfg)
    with torch.no_grad():                # larger than the default init, so that the decode emits non-blanks
        for p in m.parameters():
            p.mul_(3.0)
    m.eval()
    xs = torch.randn(4, 15, cfg["input_size"])
    xs[2] = 0.7                          # constant input: repeated argmaxes
    xlen = torch.tensor([15, 11, 30, 6], dtype=torch.int32)
    with torch.no_grad():
        logprobs = m(xs)
        ids, nlp = m.greedy_decode(xs, xlen)
        m.tovocab[0].bias[0] += 100.0    # blank (NUL = 0) wins every frame
        blank_ids, blank_nlp = m.greedy_decode(xs, xlen)
        m.tovocab[0].bias[0] -= 100.0
    assert all(len(i) == 0 for i in blank_ids)
    assert len(ids[2]) < min(int(xlen[2]), logprobs.shape[1]), "utterance 2 should collapse repeats"
    T = logprobs.shape[1]
    save = {"cfg_" + k: np.array(v) for k, v in cfg.items()}
    save.update({"sd." + k: v.numpy() for k, v in m.state_dict().items()})
    save.update(xs=xs.numpy(), xlen=xlen.numpy(), logprobs=logprobs.numpy(),
                greedy_ids=np.stack([np.pad(i, (0, T - len(i)), constant_values=-1) for i in ids]),
                greedy_counts=np.array([len(i) for i in ids]), greedy_nlp=nlp.numpy(),
                blank_bias_nlp=blank_nlp.numpy())
    np.savez_compressed(os.path.join(HERE, "ctc_tiny.npz"), **save)
    print("ctc_tiny: T' =", T, "ids", [i.tolist() for i in ids], "nlp", nlp.numpy(), "blank-bias nlp", blank_nlp.numpy())


if __name__ == "__main__":
    main()
