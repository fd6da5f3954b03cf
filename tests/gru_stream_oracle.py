"""CPU restatement of streaming greedy decoding of a GRU transducer (stream_engine.GRUStreamEngine), batched over S
independent streams, on the pieces of oracle/model_torch.py: ``encoder_gru`` with h carried from chunk to chunk, then
per encoder frame up to K rounds of joint -> argmax with the ``<unk>`` rule (logit := 0, re-argmax) -> predictor step
for the streams whose round emitted a non-blank token.  A stream's frame ends at its first blank or after K non-blank
tokens (multi_symbol_oracle.stream_decode's rule, per stream)."""
import torch

from oracle import model_torch as mt


class GRUStreamRestatement:
    def __init__(self, sd, S, unk_id=mt.UNK, blank=mt.NUL, max_symbols=1, time_reductions=(1,), fast=False):
        self.sd, self.S, self.unk, self.blank, self.K = sd, S, unk_id, blank, max_symbols
        self.tr, self.fast = time_reductions, fast
        w = sd["decoder.embed.weight"]
        L = mt._n(sd, "encoder.lstm.lstms.%d.weight_ih_l0")
        H = sd["encoder.lstm.lstms.0.weight_hh_l0"].shape[1]
        Ld = mt._n(sd, "decoder.lstm.weight_ih_l%d")
        Hd = sd["decoder.lstm.weight_hh_l0"].shape[1]
        self.enc_h = w.new_zeros(L, S, H)
        with torch.no_grad():
            self.dec_x, (self.dec_h, self.dec_c) = mt.decoder(
                sd, torch.full((S, 1), mt.BOS), (w.new_zeros(Ld, S, Hd), w.new_zeros(Ld, S, Hd)), fast=fast)
        self.hit_unk = 0                        # frames (rounds) on which the <unk> rule fired
        self.margins = []                       # top-2 logit margin of every argmax taken

    @torch.no_grad()
    def step(self, chunk):
        """chunk [S, n, F] -> ids int64 [S, n_out * K]: the K rounds of each frame in order, blank for rounds a stream
        did not take (GRUStreamEngine.step's layout)."""
        sd, K = self.sd, self.K
        enc, self.enc_h = mt.encoder_gru(sd, chunk.to(self.enc_h.dtype), self.enc_h, self.tr)
        T = enc.shape[1]
        out = torch.full((self.S, T * K), self.blank, dtype=torch.long)
        for t in range(T):
            live = torch.ones(self.S, dtype=torch.bool)
            for j in range(K):
                prob = mt.joint(sd, enc[:, t], self.dec_x[:, 0])
                pred = prob.argmax(-1)
                unk = live & (pred == self.unk)
                if unk.any():
                    self.hit_unk += int(unk.sum())
                    prob[unk, self.unk] = 0
                    pred = torch.where(unk, prob.argmax(-1), pred)
                top2 = prob[live].topk(2, -1).values
                self.margins += (top2[:, 0] - top2[:, 1]).tolist()
                out[live, t * K + j] = pred[live]
                live = live & (pred != self.blank)
                if not live.any():
                    break
                nx, (nh, nc) = mt.decoder(sd, pred[live][:, None], (self.dec_h[:, live], self.dec_c[:, live]),
                                          fast=self.fast)
                self.dec_x[live], self.dec_h[:, live], self.dec_c[:, live] = nx, nh, nc
        return out
