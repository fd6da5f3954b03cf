"""H100-native mirror of the reference's ``rnnt/models.py`` hot path.

Same class names, constructor arguments, ``forward`` signatures, return values and
``state_dict`` keys as the reference's rnnt/models.py:16-310, so ``cli/train.py``,
``cli/baseline.py``, ``cli/lightning.py`` and ``rnnt/stream.py`` can import this module
unchanged.  The torch ``nn.LSTM`` / ``nn.LayerNorm`` / ``nn.Linear`` / ``nn.Embedding`` objects
below are PARAMETER CONTAINERS ONLY (identical default initialisation and checkpoint keys); their
``forward`` is never called -- all arithmetic goes through the C-ABI of libedgedict_b200.so
(edgedict_b200/functional.py).  CUDA tensors are mandatory: there is no CPU fallback.

precision: "fp32" (default; parity mode, CUDA-core GEMMs, matches torch-CPU fp32 to ~1e-5) or
"bf16" (wgmma tensor-core GEMMs with fp32 accumulation; also selected automatically inside
``torch.autocast('cuda')``, the modern spelling of the reference's apex-O1 switch).
"""
import operator
import os

import torch
from torch import nn

from .. import functional as Fn
from .. import ops
from .tokenizer import NUL, BOS, PAD

_DEFAULT_PRECISION = os.environ.get("EDGEDICT_PRECISION", "fp32")
_PREDICTOR_STREAM = os.environ.get("EDGEDICT_PREDICTOR_STREAM", "1") != "0"
_pred_streams = {}


def _predictor_stream(device):
    s = _pred_streams.get(device)
    if s is None:
        s = _pred_streams[device] = torch.cuda.Stream(device)
    return s


def _precision(module):
    if torch.is_autocast_enabled():
        return "bf16"
    return getattr(module, "precision", _DEFAULT_PRECISION)


def _set_precision(root, precision):
    assert precision in ("fp32", "bf16")
    for m in root.modules():
        m.precision = precision
    return root


class TimeReduction(nn.Module):
    """rnnt/models.py:16-29 (only reduction_factor == 2 is used by the reference configs)."""

    def __init__(self, reduction_factor=2):
        super().__init__()
        if reduction_factor != 2:
            raise NotImplementedError("edgedict_b200 implements the reference's factor-2 reduction")
        self.reduction_factor = reduction_factor

    def forward(self, xs):
        return Fn.TimeReduce.apply(xs)


class ResLayerNormLSTM(nn.Module):
    """rnnt/models.py:32-75.  ``lstms.{i}`` / ``projs.{i}.0`` keep the reference's key layout."""

    def __init__(self, input_size, hidden_size, num_layers, dropout=0, time_reductions=[1],
                 reduction_factor=2):
        super().__init__()
        self.hidden_size = hidden_size
        self.lstms = nn.ModuleList()
        self.projs = nn.ModuleList()
        self.time_reductions = set(time_reductions)
        for i in range(num_layers):
            self.lstms.append(nn.LSTM(input_size, hidden_size, 1, batch_first=True))
            stack = [nn.LayerNorm(hidden_size)]
            if i in self.time_reductions:
                stack.append(TimeReduction(reduction_factor))
            if dropout > 0:
                stack.append(nn.Dropout(dropout))
            self.projs.append(nn.Sequential(*stack))
            input_size = hidden_size

    def _wavefront_cfg(self, xs, p):
        """(cfg, params) of the layer-wavefront schedule (functional.LSTMStack) when it applies: bf16 tensor-core
        mode, zero initial state, no active dropout, a sequence long enough to be cut into chunks."""
        if p != "bf16" or len(self.lstms) < 2 or not xs.is_cuda:
            return None
        B, T = xs.shape[0], xs.shape[1]
        if not ops.lstm_tc_supported(B, self.hidden_size):
            return None
        reductions, eps, params = [], [], []
        for cell, post in zip(self.lstms, self.projs):
            extras = list(post)[1:]
            if any(isinstance(m, nn.Dropout) and self.training and m.p > 0 for m in extras):
                return None
            reductions.append(any(isinstance(m, TimeReduction) for m in extras))
            eps.append(post[0].eps)
            params += [cell.weight_ih_l0, cell.weight_hh_l0, cell.bias_ih_l0, cell.bias_hh_l0,
                       post[0].weight, post[0].bias]
        plan = Fn.wavefront_plan(T, reductions)
        if plan is None:
            return None
        return (tuple(reductions), tuple(eps), plan), params

    def forward(self, xs, hiddens=None):
        p = _precision(self)
        if hiddens is None:
            wf = self._wavefront_cfg(xs, p)
            if wf is not None:
                out, hT, cT = Fn.LSTMStack.apply(xs, wf[0], *wf[1])
                return out, (hT, cT)
        hs, cs = (None, None) if hiddens is None else hiddens
        out_h, out_c = [], []
        for i, (cell, post) in enumerate(zip(self.lstms, self.projs)):
            h0 = None if hs is None else hs[i]
            c0 = None if cs is None else cs[i]
            y, hT, cT = Fn.LSTMLayer.apply(xs, h0, c0, cell.weight_ih_l0, cell.weight_hh_l0,
                                           cell.bias_ih_l0, cell.bias_hh_l0, p)
            ln = post[0]
            xs = Fn.LayerNormRes.apply(y, xs if i != 0 else None, ln.weight, ln.bias, ln.eps)
            for extra in list(post)[1:]:
                xs = extra(xs)
            out_h.append(hT)
            out_c.append(cT)
        return xs, (torch.stack(out_h, 0), torch.stack(out_c, 0))


class ResLayerNormGRU(nn.Module):
    """rnnt/models.py:77-116, the GRU encoder variant (`module_type='GRU'`, cli/lightning.py selects it through
    --enc_type).  Same constructor, ``state_dict`` keys (`lstms.{i}`, `projs.{i}.0`) and return value
    (xs, hs [L, B, H]) as the reference.  The ``nn.GRU`` / ``nn.LayerNorm`` objects are parameter containers only: each
    layer runs functional.GRULayer (persistent GRU recurrence: eb_gru_seq_fwd/bwd, in bf16 mode eb_gru_tc_fwd/bwd),
    LayerNorm with the residual fused (functional.LayerNormRes) and the engine's TimeReduction, layer after layer, like
    ResLayerNormLSTM's per-layer path."""

    def __init__(self, input_size, hidden_size, num_layers, dropout=0, time_reductions=[1], reduction_factor=2):
        super().__init__()
        self.hidden_size = hidden_size
        self.lstms = nn.ModuleList()
        self.projs = nn.ModuleList()
        self.time_reductions = set(time_reductions)
        for i in range(num_layers):
            self.lstms.append(nn.GRU(input_size, hidden_size, 1, batch_first=True))
            proj = [nn.LayerNorm(hidden_size)]
            if i in self.time_reductions:
                proj.append(TimeReduction(reduction_factor))
            if dropout > 0:
                proj.append(nn.Dropout(dropout))
            input_size = hidden_size
            self.projs.append(nn.Sequential(*proj))

    def forward(self, xs, hiddens=None):
        p = _precision(self)
        new_hs = []
        for i, (gru, post) in enumerate(zip(self.lstms, self.projs)):
            h0 = None if hiddens is None else hiddens[i]
            y, hT = Fn.GRULayer.apply(xs, h0, gru.weight_ih_l0, gru.weight_hh_l0, gru.bias_ih_l0, gru.bias_hh_l0, p)
            ln = post[0]
            xs = Fn.LayerNormRes.apply(y, xs if i != 0 else None, ln.weight, ln.bias, ln.eps)
            for extra in list(post)[1:]:
                xs = extra(xs)
            new_hs.append(hT)
        return xs, torch.stack(new_hs, 0)


class Encoder(nn.Module):
    """rnnt/models.py:119-136.  ``module`` defaults to the LSTM stack (the reference's default argument is the GRU
    variant, but every caller that matters passes the one it wants; Transducer passes ResLayerNormGRU for
    ``module_type='GRU'``).  Both stacks run on this library's kernels."""

    def __init__(self, input_size, hidden_size, num_layers, dropout, proj_size,
                 module=ResLayerNormLSTM, time_reductions=[1], has_proj=True):
        super().__init__()
        self.norm = nn.LayerNorm(input_size)
        self.lstm = module(input_size, hidden_size, num_layers, dropout=dropout,
                           time_reductions=time_reductions)
        self.has_proj = has_proj
        if has_proj:
            self.proj = nn.Linear(hidden_size, proj_size)

    def forward(self, xs, hiddens=None):
        xs = Fn.LayerNormRes.apply(xs, None, self.norm.weight, self.norm.bias, self.norm.eps)
        xs, hiddens = self.lstm(xs, hiddens)
        if self.has_proj:
            xs = Fn.Linear.apply(xs, self.proj.weight, self.proj.bias, _precision(self))
        return xs, hiddens


class Decoder(nn.Module):
    """Prediction network, rnnt/models.py:139-157."""

    def __init__(self, vocab_embed_size, vocab_size, hidden_size, num_layers, dropout=0,
                 proj_size=None):
        super().__init__()
        self.embed = nn.Embedding(vocab_size, vocab_embed_size, padding_idx=PAD)
        self.lstm = nn.LSTM(vocab_embed_size, hidden_size, num_layers, batch_first=True,
                            dropout=dropout)
        self.proj = nn.Linear(hidden_size, proj_size)
        self.dropout = dropout

    def forward(self, ys, hidden=None):
        p = _precision(self)
        prime = hidden is None
        xs = Fn.Embedding.apply(ys, self.embed.weight, prime, BOS, PAD)
        L = self.lstm.num_layers
        hs, cs = (None, None) if prime else hidden
        out_h, out_c = [], []
        for k in range(L):
            w = [getattr(self.lstm, n % k) for n in ("weight_ih_l%d", "weight_hh_l%d", "bias_ih_l%d", "bias_hh_l%d")]
            xs, hT, cT = Fn.LSTMLayer.apply(xs, None if hs is None else hs[k], None if cs is None else cs[k],
                                            w[0], w[1], w[2], w[3], p)
            if self.dropout > 0 and self.training and k < L - 1:
                xs = nn.functional.dropout(xs, self.dropout, True)      # nn.LSTM inter-layer dropout
            out_h.append(hT)
            out_c.append(cT)
        ys = Fn.Linear.apply(xs, self.proj.weight, self.proj.bias, p)
        return ys, (torch.stack(out_h, 0), torch.stack(out_c, 0))


class Joint(nn.Module):
    """rnnt/models.py:160-179; ``joint.0`` / ``joint.2`` key layout kept (Tanh at index 1)."""

    def __init__(self, input_size, hidden_size, vocab_size):
        super().__init__()
        self.joint = nn.Sequential(nn.Linear(input_size, hidden_size), nn.Tanh(),
                                   nn.Linear(hidden_size, vocab_size))

    def forward(self, h_enc, h_dec):
        two_d = h_enc.dim() == 2 and h_dec.dim() == 2
        if two_d:
            h_enc, h_dec = h_enc[:, None, :], h_dec[:, None, :]
        elif not (h_enc.dim() == 3 and h_dec.dim() == 3):
            raise AssertionError("Joint expects [B,T,E]/[B,U,D] or [B,E]/[B,D]")
        l0, l2 = self.joint[0], self.joint[2]
        if l0.weight.shape[1] != h_enc.shape[-1] + h_dec.shape[-1]:
            raise ValueError("joint input size mismatch")
        out = Fn.JointLogits.apply(h_enc, h_dec, l0.weight, l0.bias, l2.weight, l2.bias, _precision(self))
        return out[:, 0, 0] if two_d else out


class Transducer(nn.Module):
    """rnnt/models.py:182-269."""

    def __init__(self, vocab_embed_size, vocab_size, input_size, enc_hidden_size, enc_layers,
                 enc_dropout, enc_proj_size, dec_hidden_size, dec_layers, dec_dropout, dec_proj_size,
                 joint_size, enc_time_reductions=[1], blank=NUL, module_type='LSTM', output_loss=True,
                 fastemit_lambda=0.0, prune_range=None, simple_loss_scale=0.5, pruned_loss_scale=1.0):
        super().__init__()
        self.blank = blank
        if module_type not in ['GRU', 'LSTM']:
            raise ValueError('Unsupported module type')
        # rnnt/models.py:196-205: GRU or LSTM encoder stack, both on this engine
        self.encoder = Encoder(input_size=input_size, hidden_size=enc_hidden_size, num_layers=enc_layers,
                               dropout=enc_dropout, proj_size=enc_proj_size,
                               time_reductions=enc_time_reductions,
                               module=ResLayerNormGRU if module_type == 'GRU' else ResLayerNormLSTM)
        self.decoder = Decoder(vocab_embed_size=vocab_embed_size, vocab_size=vocab_size,
                               hidden_size=dec_hidden_size, num_layers=dec_layers, dropout=dec_dropout,
                               proj_size=dec_proj_size)
        self.joint = Joint(input_size=enc_proj_size + dec_proj_size, hidden_size=joint_size,
                           vocab_size=vocab_size)
        self.output_loss = output_loss
        if output_loss:
            from ..warprnnt_pytorch import RNNTLoss
            self.loss_fn = RNNTLoss(blank=blank)
        self.last_costs = None
        # FastEmit's lambda for the loss's backward (warprnnt_pytorch.rnnt_loss): a plain attribute, read at every
        # forward, so a trainer can ramp it between steps; not part of the state_dict.  The loss value and last_costs
        # do not depend on it.
        self.fastemit_lambda = Fn.check_fastemit_lambda(fastemit_lambda)
        # Pruned RNN-T loss (edgedict_b200/pruned.py): with an int prune_range R the model also owns the trivial
        # joiner's projections, and forward returns simple_loss_scale * mean(simple costs) + pruned_loss_scale *
        # mean(pruned costs).  The scales are plain attributes read at every forward (a trainer may ramp them);
        # prune_range=None keeps the modules, state_dict keys and code path of the full loss.
        self.prune_range = None
        if prune_range is not None:
            from ..pruned import check_prune_range
            self.prune_range = check_prune_range(prune_range)
            if self.fastemit_lambda > 0:
                raise ValueError("fastemit_lambda > 0 is not supported together with prune_range")
            self.simple_am_proj = nn.Linear(enc_proj_size, vocab_size)
            self.simple_lm_proj = nn.Linear(dec_proj_size, vocab_size)
            self.simple_loss_scale = simple_loss_scale
            self.pruned_loss_scale = pruned_loss_scale
            self.last_simple_costs = None

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def scale_length(self, logits, xlen):
        return scale_length(logits.shape[1], xlen)

    def forward(self, xs, ys, xlen, ylen):
        lam = Fn.check_fastemit_lambda(self.fastemit_lambda) if self.output_loss else 0.0
        h_enc, h_dec = self._encode(xs, ys, xlen, ylen)
        if not self.output_loss:
            return self.joint(h_enc, h_dec)
        xl = _lens_to_device(_i32(scale_length(h_enc.shape[1], xlen)), h_enc.device)
        yl = _lens_to_device(_i32(ylen), h_enc.device)
        l0, l2 = self.joint.joint[0], self.joint.joint[2]
        if self.prune_range is not None:
            return self._pruned_loss(h_enc, h_dec, _i32(ys[:, :int(ylen.max())]), xl, yl, lam)
        loss, costs = Fn.JointLoss.apply(h_enc, h_dec, l0.weight, l0.bias, l2.weight, l2.bias,
                                         _i32(ys[:, :int(ylen.max())]), xl, yl, self.blank, _precision(self), lam)
        self.last_costs = costs
        return loss

    def _pruned_loss(self, h_enc, h_dec, labels, xl, yl, lam):
        """The simple loss on the trivial joiner, the bands it picks, and the joint + loss on the bands only."""
        if lam > 0:
            raise ValueError("fastemit_lambda > 0 is not supported together with prune_range")
        p = _precision(self)
        B, T = h_enc.shape[:2]
        U = h_dec.shape[1]
        if T > 12288 or U > 1024:
            raise ValueError("the pruned loss needs T' <= 12288 encoder frames and U + 1 <= 1024, got %d and %d" % (T, U))
        am = Fn.Linear.apply(h_enc, self.simple_am_proj.weight, self.simple_am_proj.bias, p)
        lm = Fn.Linear.apply(h_dec, self.simple_lm_proj.weight, self.simple_lm_proj.bias, p)
        simple_costs, ws = Fn.SimpleLoss.apply(am, lm, labels, xl, yl, self.blank)
        self.last_simple_costs = simple_costs.detach()
        loss = float(self.simple_loss_scale) * simple_costs.mean()
        self.last_costs = None
        if float(self.pruned_loss_scale) != 0.0:
            s_begin, nopath = ops.rnnt_band_choice(xl, yl, B, T, U, self.prune_range, ws)
            l0, l2 = self.joint.joint[0], self.joint.joint[2]
            pl, costs = Fn.PrunedJointLoss.apply(h_enc, h_dec, l0.weight, l0.bias, l2.weight, l2.bias, s_begin, nopath,
                                                 self.prune_range, labels, xl, yl, self.blank, p)
            self.last_costs = costs
            loss = loss + float(self.pruned_loss_scale) * pl[0]
        return loss.reshape(1)

    def _encode(self, xs, ys, xlen, ylen):
        """The encoder and the prediction network of forward / align on xs[:, :max xlen] and ys[:, :max ylen]."""
        xs = xs[:, :int(xlen.max())].contiguous()
        ys = ys[:, :int(ylen.max())].contiguous()
        if xs.is_cuda and _PREDICTOR_STREAM:
            # The prediction network (2 x 129 recurrent steps) is independent of the encoder until the joint: it runs on
            # a side stream under the encoder's recurrence (its kernels use 32 of the 132 SMs at H_d = 256); autograd
            # replays each node's backward on the stream of its forward, so the backward passes overlap the same way.
            main = torch.cuda.current_stream(xs.device)
            side = _predictor_stream(xs.device)
            side.wait_stream(main)
            ys.record_stream(side)
            with torch.cuda.stream(side):
                h_dec, _ = self.decoder(ys)
            h_enc, _ = self.encoder(xs)
            main.wait_stream(side)
            h_dec.record_stream(main)
        else:
            h_enc, _ = self.encoder(xs)
            h_dec, _ = self.decoder(ys)
        return h_enc, h_dec

    @torch.no_grad()
    def align(self, xs, ys, xlen, ylen):
        """Forced alignment of the transcripts ys to the audio xs: the best (Viterbi) path through the RNN-T lattice,
        which gives the encoder frame at which each label is emitted.  Takes ``forward``'s arguments and runs the
        encoder, the predictor and the joint as ``forward`` does, following ``set_precision`` / autocast: bf16 mode
        takes the softmax statistics from the logits GEMM, fp32 mode runs the fp32 logits GEMM and the loss's
        statistics pass.  Utterance b covers scale_length(xlen)[b] encoder frames, as in the loss.

        Returns (list of B int64 arrays: the frame of each of the ylen[b] labels, non-decreasing; list of B arrays of
        their log-probs at those frames; -score [B] on the device, the negated log-prob of the best path, which is at
        least the loss's cost).  On an exact tie a cell takes the blank step (include/edgedict_b200.h, eb_rnnt_viterbi).

        Frames are encoder-output frames, after the time reductions.  Frame f starts at
        f * 2**len(reductions) * downsample * hop / sample_rate seconds of audio (the feature front end's hop and
        sample rate, its frame stacking / downsampling factor, and one factor 2 per time reduction of the encoder).
        The logits are freed on return."""
        h_enc, h_dec = self._encode(xs, ys, xlen, ylen)
        xl = _lens_to_device(_i32(scale_length(h_enc.shape[1], xlen)), h_enc.device)
        yl = _lens_to_device(_i32(ylen), h_enc.device)
        l0, l2 = self.joint.joint[0], self.joint.joint[2]
        frames, logp, score = Fn.joint_align(h_enc, h_dec, l0.weight, l0.bias, l2.weight, l2.bias,
                                             _i32(ys[:, :int(ylen.max())]), xl, yl, self.blank, _precision(self))
        frames, logp = frames.cpu().numpy(), logp.cpu().numpy()
        n = [int(k) for k in ylen]
        return ([frames[b, :n[b]].astype("int64") for b in range(len(n))], [logp[b, :n[b]] for b in range(len(n))],
                -score)

    @torch.no_grad()
    def greedy_decode(self, xs, xlen, max_symbols=1):
        """rnnt/models.py:243-269: at most one symbol per encoder frame; returns (list of id arrays
        incl. blanks, truncated by the UNSCALED xlen as the reference does, -sum log p).  The T'
        per-frame iterations run device-side in one persistent kernel (stream_engine.GreedyEngine).

        ``max_symbols`` = K (1 to 16) lets a frame emit up to K symbols, as the RNN-T lattice allows: the frame repeats
        joint -> argmax -> predictor step until a blank or K non-blank tokens.  Each array then holds K entries per
        frame (blank for rounds not taken) for the first xlen frames, and log p sums every round taken.  K = 1 is the
        reference's decode, bit for bit."""
        from ..stream_engine import GreedyEngine, check_max_symbols, param_fingerprint
        K = check_max_symbols(max_symbols)
        h_enc, _ = self.encoder(xs)
        B, T = h_enc.shape[0], h_enc.shape[1]
        # the phase program bakes raw weight pointers: re-homed parameters (FlatAdam, .to(), .float()) rebuild it
        key = (B, T, K, h_enc.device, param_fingerprint(self))
        cache = self.__dict__.setdefault("_greedy_engines", {})
        eng = cache.get(key)
        if eng is None:
            cache.clear()                                  # one resident program is enough
            eng = cache[key] = GreedyEngine(self, B, T, blank=self.blank, max_symbols=K)
        ids, logp = eng.run(h_enc)
        ids = ids.cpu().numpy()
        out = [ids[i, :int(n) * K].astype("int64") for i, n in enumerate(xlen)]
        return out, -logp.clone()


    @torch.no_grad()
    def beam_search(self, xs, xlen=None, W=4, merge=True, *, lm=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
                    lm_token_map=None, max_symbols=1, nbest=None, context=None, ngram=None, ngram_weight=0.0):
        """SURVEY 8(f) N4: beam decode.  The reference has no beam search in rnnt/ (north_star mentions one); its
        legacy v0 stack holds a batch-1 Graves-style search (models.py:121-202, with no-op `sorted(...)` calls and a
        removed `volatile=` API).  This is a time-synchronous beam under the SAME emission constraint as
        `greedy_decode` (at most one symbol per encoder frame, rnnt/models.py:243-269): per frame every hypothesis is
        scored against the whole vocabulary, the W best continuations survive (ties to the lowest hypothesis, then
        token index; hypotheses that reach the same token sequence are merged by log-add when `merge`), and only the
        survivors that emitted a non-blank take a predictor step.  W = 1 reproduces `greedy_decode` token for token.
        xs [B,T,F] -> (list of non-blank id lists, -log p [B]).  Utterance b decodes min(T', scale_length(xlen)[b])
        encoder frames (all T' when xlen is None).

        All utterances are searched together on the device after the encoder, in one persistent kernel launch
        (stream_engine.BeamEngine); each utterance's result does not depend on the rest of the batch.  The joint and
        the log-softmax run in fp32-accurate arithmetic (3xTF32 products, fp32 log-softmax) whatever `set_precision`
        or autocast says, as in `greedy_decode`; only the encoder follows the precision setting.

        Shallow fusion of a language model: `lm` is the reference's `LMModel` (models.py:224-261; an nn.Embedding
        `encoder`, a batch_first one-direction nn.LSTM `rnn` without proj_size, an nn.Linear `decoder` over the same
        tokens) or its state_dict (what cli/train_lm.py saves).  Per frame the candidate (slot q, token k) is ranked by
        (a + f) + logp[q], with a the acoustic log-softmax value and, for k != blank,
        f = lm_weight * log_softmax(LM logits of slot q)[map(k)] + length_bonus, or f = length_bonus when
        map(k) = -1 (a token the LM does not score); f = 0 for blank.  `map` is the identity (the LM's tokens must be
        the transducer's) or `lm_token_map`, an integer tensor [V] with values in [-1, ntoken).  Each hypothesis' LM
        state starts from zeros with one step on `lm_bos` (<bos> = 1 in cli/train_lm.py's seq_collate) and steps on
        map(k) only when the hypothesis emits a non-blank k with map(k) >= 0; there is no end-of-sentence term.  The LM
        runs as in eval mode (no dropout), in the same fp32-accurate arithmetic as the predictor.  Ranking, merging
        (log-add of the fused values) and the final pick are as without LM, and the returned -log p is the negated
        fused score of the best hypothesis.  With lm_weight = length_bonus = 0 the result is bitwise that of lm=None.

        Several symbols per frame: ``max_symbols`` = K (1 to 16, as in `greedy_decode`) runs rounds j = 0 .. K-1 in
        every frame.  Every hypothesis is open at round 0.  An open hypothesis q offers every token k at the value above:
        blank closes it, a non-blank k extends its sequence and keeps it open unless j = K-1 (the frame has then emitted
        K symbols, greedy's rule).  A closed hypothesis offers one candidate, its "stay", of value logp[q] with nothing
        added, ranked at flat index q*V + blank.  Each round keeps the W best candidates (ties as above); hypotheses
        merge only when both their sequences and their closedness are equal.  A survivor that took a non-blank token
        steps its predictor (and LM); the others keep their parent's state.  An utterance's frame ends after round K-1
        or as soon as none of its hypotheses is open.  K = 1 is the search above, bit for bit, and W = 1 gives the
        non-blank tokens of `greedy_decode(max_symbols=K)`.

        N-best lists: ``nbest`` = N (an integer in [1, W]) returns, instead of the pair above, a list of B lists of
        `stream_engine.Hypothesis(tokens, frames, nlogp)`, best first: the live hypotheses at the end of the search,
        ranked by log p descending (lowest slot on ties, the rule the best-only call picks by), min(N, live) of them.
        nlogp is the negated log p (the fused score with an LM), and entry 0 of each list is bitwise the best-only
        call's ids and -log p, for every W, K, `merge` and LM setting.  ``frames`` gives each token's encoder output
        frame (after the time reductions): the frame in which the search's own path took it.  The tokens of one frame
        appear in round order, at most K per frame, so frames are non-decreasing (strictly increasing for K = 1).
        With `merge` the frames are those of the back-pointer chain the history recorded for the surviving
        candidate, and nlogp is the merged score.  An utterance of 0 frames gives one empty hypothesis with nlogp 0.
        For the E6D2 front end, frame f starts at f * 2**len(reductions) * downsample * hop / sample_rate seconds of
        audio, as in `align`.  Still one device-to-host copy; `nbest` is part of the engine cache key.

        Contextual biasing: ``context`` is an `edgedict_b200.context.ContextGraph` over this model's V tokens (a
        ValueError otherwise, before any device work).  A candidate that appends a non-blank k to a hypothesis in
        automaton state s adds the graph's increment delta(s, k) to its fusion term: f = f_LM + delta (f = delta
        without an LM), value (a + f) + logp[q] as above; blank and a closed hypothesis' stay add nothing and keep the
        state.  During the search a value therefore holds the banked phrase bonus plus the pending bonus P(s) of the
        partial match; the final ranking, the returned -log p and every N-best nlogp use value - P(s), so a partly
        matched phrase earns nothing.  The state is a function of the token sequence, so merging stays exact.  An empty
        graph (or None) gives the search without context bit for bit; the graph's fingerprint is part of the engine
        cache key.

        N-gram shallow fusion: ``ngram`` is an `edgedict_b200.ngram.NgramLM` over this model's V tokens and blank (a
        ValueError otherwise, before the encoder runs) and ``ngram_weight`` = w a finite real.  Each hypothesis carries
        the model's state h (the start state first).  A candidate that appends a non-blank k adds w g(h, k) right after
        the LM term: f = f0 + w g, f0 the LM term or, without an LM, ``length_bonus`` (legal with an ngram alone), then
        + delta with context; value (a + f) + logp[q].  Blank and a closed hypothesis' stay keep the state and add
        nothing.  The final ranking, the returned -log p and every N-best nlogp use (value + w e(h)) - P(s), e(h) the
        model's end-of-sentence term (absent without </s> in the model).  The state is a function of the token sequence,
        so merging stays exact.  ngram=None builds the search without it; the model's fingerprint, w and the length
        bonus are part of the engine cache key."""
        from ..context import check_context, context_cache_key
        from ..ngram import check_ngram, check_ngram_weight, ngram_cache_key
        from ..stream_engine import (BeamEngine, BEAM_MAX_W, check_lm_args, check_max_symbols, check_nbest,
                                     lm_cache_key, nbest_lists, param_fingerprint)
        K = check_max_symbols(max_symbols)
        W = operator.index(W)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width W must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        N = 0 if nbest is None else check_nbest(nbest, W)
        model = check_ngram(ngram, self.joint.joint[2].weight.shape[0], self.blank)
        ng_w = check_ngram_weight(model, ngram_weight)
        fusion = check_lm_args(lm, self.joint.joint[2].weight.shape[0], lm_weight, length_bonus, lm_bos, lm_token_map,
                               ngram=model is not None)
        lm_key = lm_cache_key(fusion)
        graph = check_context(context, self.joint.joint[2].weight.shape[0], self.blank)
        h_enc, _ = self.encoder(xs)
        B, T = h_enc.shape[0], h_enc.shape[1]
        if xlen is None:
            frames = torch.full((B,), T, dtype=torch.int32)
        else:
            frames = scale_length(T, xlen).clamp(max=T).to(torch.int32)
        frames = _lens_to_device(frames.cpu(), h_enc.device)
        # the phase program bakes raw weight pointers: re-homed parameters (FlatAdam, .to(), .float()) rebuild it
        key = (B, T, W, bool(merge), K, N, h_enc.device, param_fingerprint(self), lm_key, context_cache_key(graph),
               ngram_cache_key(model, ng_w, length_bonus))
        cache = self.__dict__.setdefault("_beam_engines", {})
        eng = cache.get(key)
        if eng is None:
            cache.clear()                                  # one resident program is enough
            eng = cache[key] = BeamEngine(self, B, T, W, merge=bool(merge), blank=self.blank, lm=lm,
                                          lm_weight=lm_weight, length_bonus=length_bonus, lm_bos=lm_bos,
                                          lm_token_map=lm_token_map, max_symbols=K, nbest=N, context=graph,
                                          ngram=model, ngram_weight=ng_w)
        if N:
            return nbest_lists(eng.run(h_enc, frames), B, N, eng.ids.shape[-1])
        ids, nlogp = eng.run(h_enc, frames)
        ids = ids.cpu().numpy()
        return [[int(k) for k in row if k >= 0] for row in ids], nlogp.clone()

    def mwer_loss(self, xs, ys, xlen, ylen, W=4, nbest=None, ce_weight=0.01, max_symbols=1, word_table=None):
        """Minimum word error rate loss (Prabhavalkar et al., ICASSP 2018; Weng et al., Interspeech 2019 for RNN-T):
        the expected number of errors over the N-best list of each utterance, plus ``ce_weight`` times the RNN-T loss
        of the reference.  Takes ``forward``'s arguments and returns [1] like it.

        The encoder runs as in ``forward``; the beam search (``beam_search(W, merge=True, max_symbols,
        nbest=N)``, N = ``nbest`` or W) runs on its detached output and gives N distinct hypotheses per utterance
        (fewer when fewer are live).  Each hypothesis' errors E_i are its edit distance to ys, in tokens, or in words with
        ``word_table`` (mwer.word_table); its cost c_i = -log P(y_i | x) is the RNN-T loss of the hypothesis as a
        label sequence, through the predictor and the full joint on the same encoder output.  With P_i = softmax of
        -c_i over the utterance's hypotheses, the loss is mean_b sum_i P_i (E_i - mean E) + ce_weight * mean_b c_ref,
        and gradients reach the encoder, the predictor and the joint through every cost (the search takes none).
        fastemit_lambda > 0 raises ValueError, and the pruned loss's trivial joiner (``prune_range``) is not used.

        ``self.last_mwer`` keeps, on the device, costs [B, N+1] (the reference last), errors [B, N], posteriors [B, N]
        (0 past the count) and count [B].  One device-to-host copy of the label row lengths per call."""
        from .. import mwer
        from ..stream_engine import BeamEngine, BEAM_MAX_W, check_max_symbols, check_nbest, param_fingerprint
        K = check_max_symbols(max_symbols)
        W = operator.index(W)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width W must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        N = W if nbest is None else check_nbest(nbest, W)
        ce = mwer.check_ce_weight(ce_weight)
        table = mwer.check_word_table(word_table, self.joint.joint[2].weight.shape[0])
        if Fn.check_fastemit_lambda(self.fastemit_lambda) > 0:
            raise ValueError("mwer_loss does not take FastEmit (fastemit_lambda > 0): its rows are weighted by signed "
                             "risks, which FastEmit does not regularise")
        p = _precision(self)
        h_enc, _ = self.encoder(xs[:, :int(xlen.max())].contiguous())
        B, T, dev = h_enc.shape[0], h_enc.shape[1], h_enc.device
        xl = _lens_to_device(_i32(scale_length(T, xlen)), dev)
        key = (B, T, W, K, N, dev, param_fingerprint(self))
        cache = self.__dict__.setdefault("_mwer_engines", {})
        eng = cache.get(key)
        if eng is None:
            cache.clear()                                  # one resident program is enough
            eng = cache[key] = BeamEngine(self, B, T, W, merge=True, blank=self.blank, max_symbols=K, nbest=N)
        with torch.no_grad():
            buf = eng.run(h_enc.detach(), xl)
        ylen = torch.as_tensor(ylen).reshape(-1).cpu().to(torch.int64)
        refs = _i32(ys[:, :int(ylen.max())])
        labels, lens, _, valid, errors, count = mwer.nbest_rows(buf, B, N, eng.ids.shape[-1], refs, ylen, table,
                                                                self.joint.joint[2].weight.shape[0])
        rows = torch.arange(B, device=dev).repeat_interleave(N + 1)
        h_dec, _ = self.decoder(labels)
        l0, l2 = self.joint.joint[0], self.joint.joint[2]
        costs = Fn.JointCosts.apply(h_enc.index_select(0, rows), h_dec, l0.weight, l0.bias, l2.weight, l2.bias, labels,
                                    xl.index_select(0, rows), lens, self.blank, p).view(B, N + 1)
        return _mwer_result(self, costs, errors, valid, count, ce)


class CTCEncoder(nn.Module):
    """rnnt/models.py:272-310: the GRU encoder stack (``model.*``) and a ``Linear(proj_size, vocab_size)`` + LogSoftmax
    head (``tovocab.0.*``), same constructor and ``state_dict`` keys as the reference.  ``Encoder`` gets
    ``module=ResLayerNormGRU`` explicitly: that is the reference's default argument, which our ``Encoder`` does not share.
    Train it with ``edgedict_b200.ctc.CTCLoss`` on ``forward(xs).transpose(0, 1)``.

    Follows ``set_precision``: in bf16 mode the encoder and the projection GEMM run bf16; the log-softmax is fp32 in both
    modes (csrc/ctc.cu)."""

    def __init__(self, vocab_size, input_size, enc_hidden_size, enc_layers, enc_dropout, proj_size, blank=NUL):
        super().__init__()
        self.blank = blank
        self.model = Encoder(input_size=input_size, hidden_size=enc_hidden_size, num_layers=enc_layers,
                             dropout=enc_dropout, proj_size=proj_size, module=ResLayerNormGRU)
        self.tovocab = nn.Sequential(nn.Linear(proj_size, vocab_size), nn.LogSoftmax(dim=-1))

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def forward(self, xs):
        """xs [B, T, F] -> log-probs [B, T', V] (fp32)."""
        xs, _ = self.model(xs)
        lin = self.tovocab[0]
        return Fn.LogSoftmax.apply(Fn.Linear.apply(xs, lin.weight, lin.bias, _precision(self)))

    @torch.no_grad()
    def greedy_decode(self, xs, xlen):
        """rnnt/models.py:294-310 -> (list of int64 id arrays, -score [B] on the device).  Per frame the argmax (NaN first,
        ties to the lowest id); frames repeating the previous frame's argmax and blanks are dropped, after truncation to
        the first xlen frames -- the xlen as passed, not scaled to T' (the reference's behaviour).  The score keeps the
        reference's quirk: it sums the WHOLE log-prob rows of the kept frames, not the chosen ids' log-probs.  One kernel
        (eb_ctc_greedy) and one device-to-host copy."""
        lp = self.forward(xs)
        B, T = lp.shape[0], lp.shape[1]
        xl = torch.as_tensor(xlen).reshape(-1).to(torch.int64).clamp(0, T).to(torch.int32)
        if xl.numel() != B:
            raise ValueError("xlen must have one entry per utterance (%d), got %d" % (B, xl.numel()))
        out = ops.ctc_greedy(lp, _lens_to_device(xl.cpu(), lp.device), self.blank)
        host = out.cpu().numpy()
        ids, counts = host[:B * T].reshape(B, T), host[B * T:B * T + B]
        return [ids[i, :int(counts[i])].astype("int64") for i in range(B)], out[B * T + B:].view(torch.float32).clone()

    @torch.no_grad()
    def beam_search(self, xs, xlen=None, W=4, *, lm=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1, lm_token_map=None,
                    nbest=None, context=None, ngram=None, ngram_weight=0.0):
        """CTC prefix beam search (Hannun et al., 2014) after ``forward`` (which follows ``set_precision``), optionally
        with shallow fusion of the reference's LSTM language model.  xs [B, T, F] -> (list of B int64 id arrays, -score
        [B] on the device).  Utterance b decodes min(T', scale_length(xlen)[b]) log-prob frames (all T' when xlen is
        None): xlen is in input frames and is scaled to T' as in ``Transducer.beam_search``.  This is deliberately not
        ``greedy_decode``'s behaviour, which truncates to the unscaled xlen as the reference does.

        A hypothesis is a prefix l (non-blank ids) with pb = log P(l, the path so far ends in blank), pnb = log P(l, it
        ends in a non-blank) and a fusion term f; it starts as l = (), pb = 0, pnb = -inf, f = 0.  With (+) the log-add
        m + log1p(exp(-|a - b|)), m = max(a, b) (-inf when m is), frame t of log-probs y, for each live prefix l with
        last token e:
          * stay: pb' = (pb (+) pnb) + y[blank], pnb' = pnb + y[e] (-inf for l = ()), f' = f;
          * extension by a non-blank c to l + c: pb' = -inf, pnb' = (c == e ? pb : pb (+) pnb) + y[c], and
            f' = f + lm_weight * log_softmax(LM logits of l)[map(c)] + length_bonus (f + length_bonus when
            map(c) = -1; f' = f without an LM);
          * when l + c is the prefix of another live hypothesis l2, the extension is no candidate of its own: its pnb'
            is log-added into l2's stay pnb' (after l2's repeat term), and l2 keeps its f and LM state;
          * candidates are ranked by (pb' (+) pnb') + f' descending, ties to the lowest flat index q*V + k (a stay at
            k = blank, q the slot); the min(W, candidates) best survive, -inf candidates included.
        The result is the best live hypothesis by (pb (+) pnb) + f (lowest slot on ties) and -score is its negated
        value.  An utterance of length 0 gives an empty prefix and score 0.  The LM (as in ``Transducer.beam_search``:
        primed on lm_bos, stepped on map(c) when a hypothesis extends by a c the LM scores, no end-of-sentence term)
        runs in fp32-accurate arithmetic whatever the precision setting.  lm_weight = length_bonus = 0 gives the
        result of lm=None bit for bit.  NaN log-probs are outside the contract: the search still ends and stays in
        bounds, but which hypotheses a NaN keeps is unspecified.  See ``edgedict_b200.ctc.beam_search`` (this search on
        log-probs you already have) for the arguments, for ``nbest``, which returns N-best lists with the log-prob
        frame of each token, for ``context``, contextual biasing toward a phrase list, and for ``ngram`` /
        ``ngram_weight``, shallow fusion of a token n-gram model."""
        from .. import ctc
        from ..context import check_context
        from ..ngram import check_ngram, check_ngram_weight
        from ..stream_engine import BEAM_MAX_W, check_lm_args, check_nbest
        W = operator.index(W)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width W must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        if nbest is not None:
            check_nbest(nbest, W)
        model = check_ngram(ngram, self.tovocab[0].weight.shape[0], self.blank)
        check_ngram_weight(model, ngram_weight)
        check_context(context, self.tovocab[0].weight.shape[0], self.blank)
        check_lm_args(lm, self.tovocab[0].weight.shape[0], lm_weight, length_bonus, lm_bos, lm_token_map,
                      ngram=model is not None)
        lp = self.forward(xs)
        B, T = lp.shape[0], lp.shape[1]
        frames = torch.full((B,), T, dtype=torch.int64) if xlen is None else _ctc_frames(T, xlen, B)
        return ctc.beam_search(lp, frames, W, self.blank, lm=lm, lm_weight=lm_weight, length_bonus=length_bonus,
                               lm_bos=lm_bos, lm_token_map=lm_token_map, nbest=nbest, context=context, ngram=ngram,
                               ngram_weight=ngram_weight)

    @torch.no_grad()
    def align(self, xs, ys, xlen, ylen):
        """Forced alignment of the transcripts ys (padded [B, S] or concatenated, ylen labels each) to the audio xs:
        ``forward`` (which follows ``set_precision``), then ``edgedict_b200.ctc.forced_align`` over
        min(T', scale_length(xlen)[b]) log-prob frames, xlen scaled to T' as in ``beam_search``.  Returns
        (alignments [B, T'] in ys' dtype, per-frame log-probs [B, T'] fp32) on the device; see ``forced_align``."""
        from .. import ctc
        lp = self.forward(xs)
        return ctc.forced_align(lp, ys, _ctc_frames(lp.shape[1], xlen, lp.shape[0]), ylen, self.blank)

    def mwer_loss(self, xs, ys, xlen, ylen, W=4, nbest=None, ce_weight=0.01, max_symbols=1, word_table=None):
        """``Transducer.mwer_loss`` for CTC: ``forward`` gives the log-probs, the prefix beam search
        (``beam_search(W, nbest=N)``, N = ``nbest`` or W, over min(T', scale_length(xlen)) frames) runs on them
        detached, and each hypothesis' cost is its CTC loss (``ctc.ctc_loss(reduction='none')``) on the same log-probs
        and frames; the loss is mean_b sum_i P_i (E_i - mean E) + ce_weight * mean_b (CTC loss of ys).  CTC takes one
        label per frame: ``max_symbols`` must be 1.  ``self.last_mwer`` as in ``Transducer.mwer_loss``; one
        device-to-host copy of the label row lengths per call."""
        from .. import ctc, mwer
        from ..stream_engine import BEAM_MAX_W, CTCBeamEngine, check_max_symbols, check_nbest
        if check_max_symbols(max_symbols) != 1:
            raise ValueError("CTC emits at most one label per frame: max_symbols must be 1, got %d" % max_symbols)
        W = operator.index(W)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width W must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        N = W if nbest is None else check_nbest(nbest, W)
        ce = mwer.check_ce_weight(ce_weight)
        V = self.tovocab[0].weight.shape[0]
        table = mwer.check_word_table(word_table, V)
        lp = self.forward(xs)
        B, T, dev = lp.shape[0], lp.shape[1], lp.device
        frames = _ctc_frames(T, xlen, B)
        key = (B, T, V, W, N, dev)
        cache = self.__dict__.setdefault("_mwer_engines", {})
        eng = cache.get(key)
        if eng is None:
            cache.clear()                                  # one resident program is enough
            eng = cache[key] = CTCBeamEngine(B, T, V, W, self.blank, device=dev, nbest=N)
        with torch.no_grad():
            buf = eng.run(lp.detach(), _lens_to_device(frames.to(torch.int32), dev))
        ylen = torch.as_tensor(ylen).reshape(-1).cpu().to(torch.int64)
        refs = _i32(ys[:, :int(ylen.max())])
        labels, _, lens_h, valid, errors, count = mwer.nbest_rows(buf, B, N, T, refs, ylen, table, V)
        rows = torch.arange(B, device=dev).repeat_interleave(N + 1)
        costs = ctc.ctc_loss(lp.index_select(0, rows).transpose(0, 1), labels, frames.repeat_interleave(N + 1), lens_h,
                             blank=self.blank, reduction="none").view(B, N + 1)
        return _mwer_result(self, costs, errors, valid, count, ce)


def _mwer_result(model, costs, errors, valid, count, ce_weight):
    """The MWER loss [1] of costs [B, N+1] (the reference's last) and model.last_mwer."""
    B, N = errors.shape
    risk, post = Fn.ExpectedRisk.apply(costs[:, :N], errors, valid)
    model.last_mwer = dict(costs=costs.detach(), errors=errors, posteriors=post, count=count)
    return (risk + ce_weight * costs[:, N].sum() / B).reshape(1)


def _ctc_frames(T, xlen, B):
    """CTCEncoder's log-prob frames per utterance: xlen (input frames, host) scaled to T' and clamped to [0, T]."""
    xl = torch.as_tensor(xlen).reshape(-1).cpu()
    if xl.numel() != B:
        raise ValueError("xlen must have one entry per utterance (%d), got %d" % (B, xl.numel()))
    frames = torch.zeros(B, dtype=torch.int64)                    # scale_length divides by the longest xlen
    if int(xl.max()) > 0:
        frames = scale_length(T, xl).clamp(0, T).to(torch.int64)
    return frames


def _i32(t):
    return t.to(torch.int32).contiguous()


def _lens_to_device(t, device):
    """Host length vector -> device without stalling the host: a copy from PAGEABLE memory synchronises the stream first
    (the host then sits behind the whole encoder forward, 0.2 - 0.4 ms of idle GPU per step in the kernel timeline); a pinned
    staging tensor + non_blocking copy does not (the caching host allocator keeps the block until the copy has run)."""
    if t.device == device or device.type != "cuda":
        return t.to(device)
    staged = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
    staged.copy_(t)
    return staged.to(device, non_blocking=True)


def scale_length(T_out, xlen):
    """Transducer.scale_length (rnnt/models.py:223-226) on the host lengths."""
    scale = (xlen.max().float() / T_out).ceil()
    return (xlen / scale).ceil().int()


def CausalConv1d(in_channels, out_channels, kernel_size, dilation=1, **kwargs):
    """rnnt/models.py:313-317: nn.Conv1d padded by (kernel_size - 1) * dilation, kaiming-normal weight."""
    pad = (kernel_size - 1) * dilation
    conv = nn.Conv1d(in_channels, out_channels, kernel_size, padding=pad, dilation=dilation, **kwargs)
    nn.init.kaiming_normal_(conv.weight)
    return conv


def _conv_spec(conv):
    k, s, d = conv.kernel_size[0], conv.stride[0], conv.dilation[0]
    if d != 1:
        raise ValueError("edgedict_b200's front end implements dilation 1 only (FrontEnd always passes 1)")
    if k == 1:
        raise ValueError("kernel_size 1: the reference's trim x[:, :, :-0] returns an empty tensor")
    return k, s


def _check_wave(x, what):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise ValueError("%s needs a CUDA tensor (there is no CPU path)" % what)
    if x.dtype != torch.float32:
        raise ValueError("%s needs float32 input, got %s" % (what, x.dtype))


def _check_lengths(T, specs):
    for k, s in specs:
        T = Fn.conv_out_len(T, k, s)
        if T < 1:
            raise ValueError("the front end's input is too short: a conv layer (k=%d, s=%d) has no output frame" % (k, s))
    return T


def _check_bf16_channels(chans):
    if any(c % 16 for c in chans):
        raise ValueError("bf16 mode needs the channel count of every conv block to be a multiple of 16 (got %s); use "
                         "set_precision('fp32')" % (list(chans),))


class DilatedConvBlock(nn.Module):
    """rnnt/models.py:319-334: conv(GroupNorm(1, C_in)(GELU(x))) and the trim; x [B, C_in, T] -> [B, C_out, T_out]."""

    def __init__(self, in_channels, out_channels, kernel_size, dilation=1, group_norm_size=1, **kwargs):
        super().__init__()
        pad = (kernel_size - 1) * dilation
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size, padding=pad, dilation=dilation, **kwargs)
        nn.init.kaiming_normal_(self.conv.weight)
        self.gn = nn.GroupNorm(group_norm_size, in_channels)
        self.act = nn.GELU()

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def _spec(self):
        if self.gn.num_groups != 1 or self.conv.groups != 1 or not isinstance(self.act, nn.GELU) or \
                self.act.approximate != "none":
            raise ValueError("edgedict_b200 implements DilatedConvBlock with GroupNorm(1, C), groups=1 and exact GELU")
        k, s = _conv_spec(self.conv)
        return (k, s, self.conv.in_channels, self.conv.out_channels, self.conv.bias is not None, float(self.gn.eps))

    def _params(self):
        c = self.conv
        return [c.weight] + ([c.bias] if c.bias is not None else []) + [self.gn.weight, self.gn.bias]

    def forward(self, x):
        _check_wave(x, "DilatedConvBlock")
        spec = self._spec()
        _check_lengths(x.shape[-1], [spec[:2]])
        p = _precision(self)
        if p == "bf16":
            _check_bf16_channels(spec[2:4])
        y = Fn.FrontEndStack.apply(x.transpose(1, 2).contiguous(), (None, (spec,), None), p, *self._params())
        return y.transpose(1, 2)


class FrontEnd(nn.Module):
    """rnnt/models.py:336-365: the learned front end on raw audio.  x [B, L] or [B, 1, L] fp32 -> [B, T, C_last]
    (the reference's return value), every step through the C-ABI: causal strided convs (bf16 mode: TMA + wgmma),
    GELU + GroupNorm(1, C) with statistics over the whole padded batch row, LayerNorm(C_last)."""

    def __init__(self, frontend_params=[(10, 5, 16)] + [(8, 4, 32)] + [(4, 2, 128)] * 3, bias=True):
        super().__init__()
        kernel_sizes = [p[0] for p in frontend_params]
        strides = [p[1] for p in frontend_params]
        channels = [p[2] for p in frontend_params]
        assert len(kernel_sizes) == len(strides)
        self.conv1 = CausalConv1d(1, channels[0], kernel_size=kernel_sizes[0], dilation=1, stride=strides[0], bias=bias)
        self.encode = nn.Sequential(*[
            DilatedConvBlock(channels[idx - 1], channels[idx], kernel_size=kernel_sizes[idx], dilation=1,
                             stride=strides[idx], group_norm_size=1, bias=bias)
            for idx in range(1, len(strides))
        ])
        self.layer_norm = nn.LayerNorm(frontend_params[-1][-1])

    def set_precision(self, precision):
        return _set_precision(self, precision)

    def output_length(self, L):
        """Frames of the output for L input samples (16 s at 16 kHz: 399 with cli/train.py's parameters)."""
        specs = [_conv_spec(self.conv1)] + [blk._spec()[:2] for blk in self.encode]
        return _check_lengths(L, specs)

    def forward(self, x):
        if isinstance(x, torch.Tensor) and x.dim() == 3:
            if x.shape[1] != 1:
                raise ValueError("FrontEnd takes [B, L] or [B, 1, L] audio, got %s" % (tuple(x.shape),))
            x = x[:, 0]
        _check_wave(x, "FrontEnd")
        if x.dim() != 2:
            raise ValueError("FrontEnd takes [B, L] or [B, 1, L] audio, got %s" % (tuple(x.shape),))
        c1 = self.conv1
        if c1.in_channels != 1:
            raise ValueError("FrontEnd's first conv takes one channel")
        k0, s0 = _conv_spec(c1)
        blocks = tuple(blk._spec() for blk in self.encode)
        self.output_length(x.shape[1])
        p = _precision(self)
        if p == "bf16":
            _check_bf16_channels([c1.out_channels] + [b[3] for b in blocks])
        params = [c1.weight] + ([c1.bias] if c1.bias is not None else [])
        for blk in self.encode:
            params += blk._params()
        params += [self.layer_norm.weight, self.layer_norm.bias]
        if self.layer_norm.normalized_shape != (blocks[-1][3] if blocks else c1.out_channels,) or \
                not self.layer_norm.elementwise_affine:
            raise ValueError("FrontEnd's layer_norm must be an affine LayerNorm over the last conv's channels")
        spec = ((k0, s0, c1.out_channels, c1.bias is not None), blocks, float(self.layer_norm.eps))
        return Fn.FrontEndStack.apply(x.contiguous(), spec, p, *params)


def frontend_lengths(xlen, T):
    """cli/train.py:236-238's frame lengths of FrontEnd's output: floor(xlen / (max(xlen) / T)), T = the output's time
    axis (dimension 1 of FrontEnd's [B, T, C] output)."""
    max_length = xlen.max()
    return torch.floor(xlen.float() / (max_length.item() / T)).int()


def convert_lightning2normal(checkpoint):
    """rnnt/models.py:368-380: unwrap a Lightning checkpoint; when its keys carry the ``model.``
    prefix, drop it and re-wrap as {'model': state_dict}."""
    if 'state_dict' not in checkpoint:
        return checkpoint
    sd = checkpoint['state_dict']
    if 'model.' in next(iter(sd.keys())):
        return {'model': {k.replace('model.', ''): v for k, v in sd.items()}}
    return sd
