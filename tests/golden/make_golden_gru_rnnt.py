"""Generates tests/golden/gru_rnnt_tiny.npz by running the REFERENCE's own GRU transducer (rnnt/models.py:182-269,
``Transducer(module_type='GRU', output_loss=False)``, torch CPU fp32):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_gru_rnnt.py

Two encoder layers with the default time reduction after layer 1, the weights scaled up so that the joint emits
symbols.  The fixture holds the config, the state_dict, one utterance of log-mel frames and the offline
``greedy_decode`` ids, one per encoder frame, blanks included.  The encoder is causal and the time reduction pairs
frames inside an even chunk, so streaming the frames in even chunks with h carried must give exactly these ids.
<unk> (3) is never the argmax, so a stream's <unk> rule never fires on the fixture.  The committed fixture is what the
tests see; nothing at test time reads the reference.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
UNK = 3


def main():
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from rnnt.models import Transducer  # (the reference)
    torch.manual_seed(2026)
    cfg = dict(vocab_embed_size=8, vocab_size=16, input_size=12, enc_hidden_size=20, enc_layers=2, enc_dropout=0,
               enc_proj_size=16, dec_hidden_size=16, dec_layers=1, dec_dropout=0, dec_proj_size=16, joint_size=24)
    m = Transducer(module_type="GRU", output_loss=False, **cfg)
    with torch.no_grad():                # larger than the default init, so that the decode emits non-blanks
        for p in m.parameters():
            p.mul_(3.0)
        m.joint.joint[2].bias[UNK] -= 10.0   # never <unk>: the stream's <unk> rule is not the reference's
        m.joint.joint[2].bias[0] += 2.0      # and about a third of the frames blank
    m.eval()
    xs = torch.randn(1, 96, cfg["input_size"])
    with torch.no_grad():
        ids, nlp = m.greedy_decode(xs, torch.tensor([xs.shape[1]]))
        h_enc, _ = m.encoder(xs)
        # the argmax over raw logits (what a stream takes) at every frame of the greedy path is never <unk>
        h_dec, (h, c) = m.decoder(xs.new_empty(1, 0))
        for t, k in enumerate(ids[0]):
            logits = m.joint(h_enc[:, t], h_dec[:, 0])
            assert int(logits.argmax(-1)) == int(k) and int(k) != UNK
            if k != 0:
                h_dec, (h, c) = m.decoder(torch.tensor([[int(k)]]), (h, c))
    ids = ids[0].astype(np.int64)
    assert len(ids) == xs.shape[1] // 2
    assert int((ids != 0).sum()) >= 10, "the fixture should emit symbols"
    save = {"cfg_" + k: np.array(v) for k, v in cfg.items()}
    save.update({"sd." + k: v.numpy() for k, v in m.state_dict().items()})
    save.update(xs=xs[0].numpy(), greedy_ids=ids, greedy_nlp=nlp.numpy())
    np.savez_compressed(os.path.join(HERE, "gru_rnnt_tiny.npz"), **save)
    print("gru_rnnt_tiny: T' =", len(ids), "non-blank", int((ids != 0).sum()), "ids", ids.tolist())


if __name__ == "__main__":
    main()
