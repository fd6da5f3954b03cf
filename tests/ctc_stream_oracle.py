"""CPU restatement of streaming greedy CTC decoding (stream_engine.CTCStreamEngine) -- TEST INFRASTRUCTURE.

Per chunk: oracle.model_torch.encoder_gru with the carried ``hiddens``, the ``tovocab`` Linear, log_softmax, then the
collapse of CTCEncoder.greedy_decode (rnnt/models.py:294-310) with the previous frame's argmax carried across chunks
(-1 after a reset, which matches no token) and the running score: the sum of the whole log-prob rows of the kept
frames.  The argmax is oracle.ctc's (``max(dim=-1)``)."""
import torch
import torch.nn.functional as F

from oracle import model_torch as mt


class CTCStreamRestatement:
    def __init__(self, sd, S, blank=0, time_reductions=(1,), dtype=torch.float64, device="cpu"):
        self.sd = {k: torch.as_tensor(v).to(device, dtype) for k, v in sd.items()}
        L = mt._n(self.sd, "model.lstm.lstms.%d.weight_ih_l0")
        H = self.sd["model.lstm.lstms.0.weight_hh_l0"].shape[1]
        self.S, self.blank, self.tr, self.dtype = S, blank, tuple(time_reductions), dtype
        self.h = torch.zeros(L, S, H, dtype=dtype, device=device)
        self.prev = torch.full((S,), -1, dtype=torch.int64)
        self.score = torch.zeros(S, dtype=torch.float64)

    @torch.no_grad()
    def step(self, chunk):
        """chunk [S, n, F] -> (list of S int64 id lists emitted in this chunk, log-probs [S, n_out, V], argmax
        [S, n_out])."""
        x, self.h = mt.encoder_gru(self.sd, torch.as_tensor(chunk).to(self.h.device, self.dtype), self.h, self.tr,
                                   pre="model.")
        lp = F.log_softmax(F.linear(x, self.sd["tovocab.0.weight"], self.sd["tovocab.0.bias"]), -1)
        _, am = lp.max(dim=-1)
        am, rows = am.cpu(), lp.sum(-1).double().cpu()
        ids = []
        for s in range(self.S):
            out = []
            for t in range(am.shape[1]):
                c = int(am[s, t])
                if c != self.blank and c != int(self.prev[s]):
                    out.append(c)
                    self.score[s] += float(rows[s, t])
                self.prev[s] = c
            ids.append(out)
        return ids, lp, am
