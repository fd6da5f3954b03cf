"""Host side of the persistent streaming-decode kernel (csrc/decode.cu).

``StreamEngine(transducer, n_streams, frames_per_chunk)`` owns the per-stream recurrent state on
the device and a *phase program* (array of ``EbPhase``) built once; ``step(chunk)`` copies the
chunk's log-mel frames into a fixed input buffer and launches ONE cooperative kernel that runs the
stateful encoder, then for every encoder output frame joint -> argmax (with the ``<unk>`` rule) ->
masked predictor step, for all streams at once.  Semantics per stream are exactly those of
PytorchStreamDecoder.reset/decode (reference rnnt/stream.py:78-120): at most one symbol per
encoder frame, argmax over raw logits, predictor advanced only on non-blank.  With ``max_symbols`` = K > 1 a frame
repeats joint -> argmax -> predictor step until a blank or K symbols (GreedyEngine likewise).
"""
import collections
import ctypes as C
import functools
import math
import numbers
import operator

import torch

from . import ops
from ._lib import lib, check
from .context import check_context
from .ngram import check_ngram, check_ngram_weight
from .rnnt.tokenizer import NUL, BOS, UNK

PH_LN, PH_PAIR, PH_LSTM, PH_LINEAR, PH_ARGMAX, PH_COPY, PH_BEAM_SELECT, PH_GATHER, PH_BEAM_FINAL, PH_BEAM_COMMIT, \
    PH_SKIP, PH_CTC_BEAM, PH_GRU, PH_CTC_EMIT, PH_FE_FRAME, PH_FE_GEMM, PH_FE_POWER, PH_FE_LOG, PH_FE_FINISH = range(19)
F_TANH, F_EMBED, F_MASKED, F_LOGP, F_MERGE, F_LM, F_STREAM, F_FLUSH, F_CONT, F_ROUNDS, F_FRONTEND, F_CONTEXT, \
    F_NGRAM = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096
BEAM_MAX_W = 1024                                     # EB_BEAM_MAX_W
CTC_SEQ_HEAD = 5                                      # CTC_BEAM's token rows: {len, hash lo / hi, parent hash lo / hi}
MAX_SYMBOLS = 16                                      # bounds the program: about (5 + L_dec) * K phases per frame


class EbPhase(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("type", "S", "K1", "K2", "N", "flags", "ldx1", "ldx2", "ldw1", "ldw2",
                                         "ldy", "aux", "aux2", "hist_ld", "hist_col", "x1_div")] + \
               [(n, C.c_void_p) for n in ("x1", "x2", "w1", "w2", "b1", "b2", "y", "y2", "c", "tok_in", "tok_out",
                                          "hist", "seq_in", "seq_out", "src", "fuse", "tok_map", "tok_out2", "ctx")]


class EbNgram(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("unigram", "bo", "suffix", "depth", "first", "count", "tok", "prob", "next",
                                          "end", "state0", "state1", "row")] + [("weight", C.c_float), ("pad_", C.c_int32)]


def _ptr(t, off=0):
    return None if t is None else t.data_ptr() + off * t.element_size()


def lstm_layers(lstm):
    """[(weight_ih, weight_hh, bias_ih, bias_hh)] of every layer of an nn.LSTM."""
    return [tuple(getattr(lstm, n % k) for n in ("weight_ih_l%d", "weight_hh_l%d", "bias_ih_l%d", "bias_hh_l%d"))
            for k in range(lstm.num_layers)]


def predictor_phases(prog, embed, layers, proj_w, proj_b, S, h, c, htmp, x, tok, rest, masked):
    """Append one step of an embedding -> LSTM stack -> Linear network for S rows to the phase list ``prog``: the
    embedding row (of table ``embed``) of ``tok`` through every LSTM layer (``layers`` as from lstm_layers; h, c, htmp
    [Ld, S, Hd]; with ``masked``, rows whose token is ``rest`` keep their state), then the output Linear into x [S, D].
    The transducer's predictor rests on blank, a fused language model on -1."""
    Ld, Hd = len(layers), layers[0][1].shape[1]
    Em, D = embed.shape[1], proj_w.shape[0]
    fl = F_EMBED | (F_MASKED if masked else 0)
    for k, w in enumerate(layers):
        prog.append(EbPhase(type=PH_LSTM, S=S, N=Hd, K1=Em if k == 0 else Hd, K2=Hd,
                            flags=fl if k == 0 else (fl & F_MASKED),
                            x1=_ptr(embed) if k == 0 else _ptr(htmp[k - 1]), ldx1=Em if k == 0 else Hd,
                            x2=_ptr(h[k]), ldx2=Hd, w1=_ptr(w[0]), ldw1=w[0].shape[1], w2=_ptr(w[1]), ldw2=Hd,
                            b1=_ptr(w[2]), b2=_ptr(w[3]), c=_ptr(c[k]), y=_ptr(htmp[k]), ldy=Hd, tok_in=_ptr(tok),
                            aux=rest))
    prog.append(EbPhase(type=PH_COPY, S=Ld * S, N=Hd, x1=_ptr(htmp), y=_ptr(h)))
    prog.append(EbPhase(type=PH_LINEAR, S=S, N=D, K1=Hd, x1=_ptr(h[Ld - 1]), ldx1=Hd, w1=_ptr(proj_w),
                        ldw1=Hd, b1=_ptr(proj_b), y=_ptr(x), ldy=D))


def _dec_phases(prog, dec, S, h, c, htmp, x, tok, blank, masked):
    predictor_phases(prog, dec.embed.weight, lstm_layers(dec.lstm), dec.proj.weight, dec.proj.bias, S, h, c, htmp, x,
                     tok, blank, masked)


def check_max_symbols(max_symbols):
    """The per-frame symbol cap K of greedy decoding, an integer in [1, MAX_SYMBOLS].  Raises TypeError / ValueError;
    touches no device."""
    if isinstance(max_symbols, bool) or not isinstance(max_symbols, numbers.Integral):
        raise TypeError("max_symbols must be an integer, got %r" % (max_symbols,))
    K = int(max_symbols)
    if not 1 <= K <= MAX_SYMBOLS:
        raise ValueError("max_symbols must be in [1, %d], got %d" % (MAX_SYMBOLS, K))
    return K


Hypothesis = collections.namedtuple("Hypothesis", ["tokens", "frames", "nlogp"])
Hypothesis.__doc__ = """One entry of an N-best list (``beam_search(nbest=N)``): the non-blank token ids (int64 ndarray),
the encoder output frame each of them entered the hypothesis at (int32 ndarray, same length) and nlogp, the negated
score the best-only call returns for its one hypothesis."""


def check_nbest(nbest, W):
    """The list length N of an N-best beam search of width W, an integer in [1, W].  Raises TypeError / ValueError;
    touches no device."""
    if isinstance(nbest, bool) or not isinstance(nbest, numbers.Integral):
        raise TypeError("nbest must be an integer, got %r" % (nbest,))
    N = int(nbest)
    if not 1 <= N <= W:
        raise ValueError("nbest must be in [1, W = %d], got %d" % (W, N))
    return N


def _engine_nbest(nbest, W):
    """An engine's nbest: 0 (the best hypothesis alone, the program as without N-best) or check_nbest's N."""
    if isinstance(nbest, numbers.Integral) and not isinstance(nbest, bool) and nbest == 0:
        return 0
    return check_nbest(nbest, W)


def final_outputs(e, B, N, L):
    """Allocate on engine ``e`` what BEAM_FINAL writes for B utterances, ids rows of length L.  N = 0 (the best
    hypothesis alone): e.ids int32 [B, L] and e.nlogp [B].  N >= 1: one int32 buffer ``e.nbest_out`` (one copy to the
    host), ids | frames [B, N, L] | -log p (fp32 bits) [B, N] | count [B], with the views e.ids, e.nbest_frames,
    e.nlogp and e.nbest_count."""
    e.nbest = N
    if not N:
        e.ids = torch.zeros(B, L, dtype=torch.int32, device=e.dev)
        e.nlogp = torch.zeros(B, dtype=torch.float32, device=e.dev)
        e.nbest_out = e.nbest_frames = e.nbest_count = None
        return
    n = B * N * L
    e.nbest_out = torch.zeros(2 * n + B * N + B, dtype=torch.int32, device=e.dev)
    e.ids, e.nbest_frames = e.nbest_out[:n].view(B, N, L), e.nbest_out[n:2 * n].view(B, N, L)
    e.nlogp = e.nbest_out[2 * n:2 * n + B * N].view(torch.float32).view(B, N)
    e.nbest_count = e.nbest_out[2 * n + B * N:]


def final_phase(e, W, y, K, ctx=None):
    """The BEAM_FINAL phase of engine ``e`` (final_outputs done, e.hist from beam_history) over the slot values y, K
    history columns per frame.  With e.nbest = 0 the N-best fields stay zero / NULL: the best-only phase.  ``ctx``
    (context_program's fields and the parity that holds the final context states) ranks by y - pending[state]."""
    B, L = e.ids.shape[0], e.ids.shape[-1]
    ph = EbPhase(type=PH_BEAM_FINAL, S=B, aux=W, aux2=e.blank, y=_ptr(y), hist=_ptr(e.hist),
                 hist_ld=e.hist_live.shape[1], tok_out=_ptr(e.ids), ldy=L, y2=_ptr(e.nlogp), K1=e.nbest,
                 ldw2=K if e.nbest else 0, seq_out=_ptr(e.nbest_frames), tok_out2=_ptr(e.nbest_count))
    if ctx is not None:
        fields, parity = ctx
        ph.flags, ph.ctx, ph.hist_col = fields["flags"], fields["ctx"], parity
    return ph


def context_program(e, graph, state, ng=None):
    """Contextual biasing on beam engine ``e`` (its ``dev`` set) with the ContextGraph ``graph`` (check_context done)
    and the per-slot automaton states ``state`` (two int32 [R] parities on the device): uploads the tables and the
    EbContext descriptor {next, delta, pending, state[0], state[1], ng} and returns the fields a BEAM_SELECT / CTC_BEAM /
    BEAM_FINAL phase reads it through.  e._ctx keeps the buffers alive.  ``ng`` (ngram_program's descriptor) rides in
    the same descriptor and adds flag F_NGRAM; graph = None then leaves the context fields NULL and F_CONTEXT unset."""
    ptrs, tabs, flags = [0] * 5, None, 0
    if graph is not None:
        tabs = graph.to(e.dev)
        nV = graph.n_states * graph.vocab_size
        base = tabs.data_ptr()
        ptrs = [base, base + 4 * nV, base + 8 * nV, state[0].data_ptr(), state[1].data_ptr()]
        flags |= F_CONTEXT
    if ng is not None:
        flags |= F_NGRAM
    desc = torch.tensor(ptrs + [ng or 0], dtype=torch.int64).to(e.dev)
    e._ctx = (tabs, desc, state)
    return dict(flags=flags, ctx=desc.data_ptr())


def ngram_program(e, model, state, weight, length_bonus, R, V):
    """N-gram fusion on beam engine ``e`` (its ``dev`` and ``lm`` set) with the NgramLM ``model`` (check_ngram done),
    the per-slot n-gram states ``state`` (two int32 [R] parities on the device) and ``weight``: uploads the tables,
    allocates the row workspace e.ng_row [R, V] and the EbNgram descriptor, and returns its device address (for
    context_program) and the phase fields it needs besides: without an LM, ``fuse`` = {0, length_bonus}."""
    buf, offs = model.to(e.dev)
    base = buf.data_ptr()
    tabs = [base + 4 * o for o in offs] + ([] if model.has_end else [None])
    e.ng_row = torch.zeros(R, V, dtype=torch.float32, device=e.dev)
    d = EbNgram(*tabs, state[0].data_ptr(), state[1].data_ptr(), e.ng_row.data_ptr(), weight, 0)
    desc = torch.frombuffer(bytearray(bytes(d)), dtype=torch.uint8).to(e.dev)
    e.ng_start = model.start
    fields = {}
    if not e.lm:
        e.ng_fuse = torch.tensor([0.0, length_bonus], dtype=torch.float32, device=e.dev)
        fields["fuse"] = _ptr(e.ng_fuse)
    e._ng = (buf, desc, state)
    return desc.data_ptr(), fields


def fusion_fields(e, sel, graph, cstate, model, nstate, weight, length_bonus, R, V):
    """Add contextual biasing (graph) and n-gram fusion (model) to the BEAM_SELECT / CTC_BEAM fields ``sel`` of engine
    ``e``; returns what final_phase needs (None without either)."""
    if graph is None and model is None:
        return None
    ng, extra = ngram_program(e, model, nstate, weight, length_bonus, R, V) if model is not None else (None, {})
    cf = context_program(e, graph, cstate, ng)
    sel.update(flags=sel["flags"] | cf["flags"], ctx=cf["ctx"], **extra)
    return cf


def nbest_lists(buf, B, N, L):
    """An engine's N-best output ``buf`` (nbest_buffer's layout, on the device) -> B lists of Hypothesis, best first,
    each of length min(N, live slots).  One device-to-host copy."""
    host = buf.cpu().numpy()
    n = B * N * L
    ids, frames = host[:n].reshape(B, N, L), host[n:2 * n].reshape(B, N, L)
    nlogp = host[2 * n:2 * n + B * N].view("float32").reshape(B, N)
    count = host[2 * n + B * N:]
    out = []
    for b in range(B):
        hyps = []
        for r in range(int(count[b])):
            keep = ids[b, r] >= 0
            hyps.append(Hypothesis(ids[b, r][keep].astype("int64"), frames[b, r][keep].astype("int32"),
                                   float(nlogp[b, r])))
        out.append(hyps)
    return out


def greedy_frame(prog, K, S, tok, blank, round_phases):
    """Append one encoder frame of greedy decoding with at most K symbols for S rows.  ``round_phases(j)`` appends round
    j: the joint, an ARGMAX into ``tok`` (with F_CONT for j >= 1: rows whose frame already ended stay blank) and the
    predictor step masked on blank.  Each round j >= 1 opens with a SKIP to the end of the frame, taken when every row's
    round j-1 token was blank.  With K = 1 this is round 0 alone, the one-symbol program."""
    skips = []
    for j in range(K):
        if j:
            skips.append(len(prog))
            prog.append(EbPhase(type=PH_SKIP, S=S, aux2=blank, tok_in=_ptr(tok)))
        round_phases(j)
    for i in skips:
        prog[i].aux = len(prog) - i - 1


def joint_phases(prog, joint, S, x_enc, ldx_enc, dec_x, hidden, logits, x1_div=0):
    """Append the joint for S rows: hidden [S, J] = tanh(W1 [encoder frame | dec_x] + b1), then logits [S, V] =
    W2 hidden + b2, ``joint`` being (W1, b1, W2, b2).  The encoder frame of row r is at x_enc, row stride ldx_enc; with
    x1_div = W the W rows of a beam's utterance share row r // W."""
    w1, b1, w2, b2 = joint
    J, V, D = w1.shape[0], w2.shape[0], dec_x.shape[1]
    E = w1.shape[1] - D
    prog.append(EbPhase(type=PH_LINEAR, S=S, N=J, flags=F_TANH, K1=E, x1=x_enc, ldx1=ldx_enc, x1_div=x1_div,
                        w1=_ptr(w1), ldw1=E + D, K2=D, x2=_ptr(dec_x), ldx2=D, w2=_ptr(w1, E), ldw2=E + D, b1=_ptr(b1),
                        y=_ptr(hidden), ldy=J))
    prog.append(EbPhase(type=PH_LINEAR, S=S, N=V, K1=J, x1=_ptr(hidden), ldx1=J, w1=_ptr(w2), ldw1=J, b1=_ptr(b2),
                        y=_ptr(logits), ldy=V))


def greedy_round(prog, e, dec, h_enc, k, j, flags, unk, logp=None):
    """Append round j of encoder frame k of greedy decoding on engine ``e`` (GreedyEngine, StreamEngine): the joint of
    frame k of h_enc [rows, T', E] with the predictor output e.dec_x, an ARGMAX of the logits into e.tok and history
    column k * K + j (``flags``, F_CONT added for j >= 1; ``unk`` the token re-argmaxed when it wins, -1 for none; the
    log p of every row added into ``logp`` with F_LOGP), then the predictor step masked on blank."""
    S, T, E = h_enc.shape
    V = e.logits.shape[1]
    joint_phases(prog, e._joint, S, _ptr(h_enc, k * E), T * E, e.dec_x, e.hidden, e.logits)
    prog.append(EbPhase(type=PH_ARGMAX, S=S, N=V, flags=flags | (F_CONT if j else 0), x1=_ptr(e.logits), ldx1=V,
                        aux=e.blank, aux2=unk, tok_out=_ptr(e.tok), hist=_ptr(e.hist), hist_ld=e.hist.shape[1],
                        hist_col=k * e.max_symbols + j, y=_ptr(logp)))
    _dec_phases(prog, dec, S, e.dec_h, e.dec_c, e.dec_htmp, e.dec_x, e.tok, e.blank, masked=True)


def beam_state(e, R, Ld, Hd, D, LS, context=False, ngram=False):
    """Allocate on engine ``e`` (its ``dev`` set) the per-slot state of a beam search over R rows, for each parity p
    in one flat buffer ``e._home[p]``: the predictor state e._st[p] [2 Ld, R, Hd] (h of every layer, then c; views
    e.dec_h[p] / e.dec_c[p]), its output e.dec_x[p] [R, D], the token sequences e.seqs[p] int32 [R, LS], with an LM
    (``e.lm``, lm_fusion done) its state e._lst[p] [2 Ll, R, Hl] (e.lm_h[p] / e.lm_c[p]) and with ``context`` the
    context automaton states e.ctx_state[p] int32 [R] (else None), with ``ngram`` the n-gram states e.ng_state[p] int32
    [R] (else None).  One COPY of e._home[1] into e._home[0] moves all of it, which a round of a multi-symbol frame
    needs (beam_frame)."""
    Ll, _, Hl = e.lm_htmp.shape if e.lm else (0, 0, 0)
    sizes = [2 * Ld * R * Hd, R * D, R * LS, 2 * Ll * R * Hl, R if context else 0, R if ngram else 0]
    offs = [0]
    for n in sizes:
        offs.append(offs[-1] + -(-n // 64) * 64)           # 256-byte aligned segments
    assert offs[-1] < 2 ** 31
    e._home = torch.zeros(2, offs[-1], dtype=torch.float32, device=e.dev)
    seg = lambda p, i: e._home[p, offs[i]:offs[i] + sizes[i]]
    e._st = [seg(p, 0).view(2 * Ld, R, Hd) for p in (0, 1)]
    e.dec_h, e.dec_c = [s[:Ld] for s in e._st], [s[Ld:] for s in e._st]
    e.dec_x = [seg(p, 1).view(R, D) for p in (0, 1)]
    e.seqs = [seg(p, 2).view(torch.int32).view(R, LS) for p in (0, 1)]
    e._lst = [seg(p, 3).view(2 * Ll, R, Hl) for p in (0, 1)] if Ll else None
    if Ll:
        e.lm_h, e.lm_c = [s[:Ll] for s in e._lst], [s[Ll:] for s in e._lst]
    e.ctx_state = [seg(p, 4).view(torch.int32) for p in (0, 1)] if context else None
    e.ng_state = [seg(p, 5).view(torch.int32) for p in (0, 1)] if ngram else None


def beam_history(e, B, T, W):
    """Allocate on engine ``e`` the beam history of B utterances over T columns, which BEAM_SELECT / CTC_BEAM write
    and BEAM_FINAL / BEAM_COMMIT read: one int32 buffer ``e.hist``, parent | token | log p | live, with the views
    e.hist_parent / e.hist_token [B, T, W], e.hist_logp (fp32) [B, T, W] and e.hist_live [B, T]."""
    n = B * T * W
    e.hist = torch.zeros(3 * n + B * T, dtype=torch.int32, device=e.dev)
    e.hist_parent, e.hist_token = e.hist[:n].view(B, T, W), e.hist[n:2 * n].view(B, T, W)
    e.hist_logp = e.hist[2 * n:3 * n].view(torch.float32).view(B, T, W)
    e.hist_live = e.hist[3 * n:].view(B, T)


def beam_reset(e):
    """Start a new utterance in every beam of engine ``e`` (BeamEngine, StreamBeamEngine): one live slot of log p 0
    (the others -inf) with the empty sequence and the zero predictor state primed with <bos>, and with an LM the zero
    LM state primed with lm_bos."""
    e._st[0].zero_()
    e.seqs[0].zero_()
    if e.ctx_state is not None:
        e.ctx_state[0].zero_()                                  # every slot at the automaton's root
    if e.ng_state is not None:
        e.ng_state[0].fill_(e.ng_start)                         # every slot at the n-gram start state
    e.logp.fill_(float("-inf"))
    e.logp.view(-1, e.W)[:, 0] = 0.0
    e.tok.fill_(BOS)
    if e.lm:
        e._lst[0].zero_()
        e.lm_tok.fill_(e.lm_bos)


def beam_frame(prog, e, dec, t, x_enc, ldx_enc, sel, lm_step):
    """Append encoder frame t of the beam search, the same for BeamEngine and StreamBeamEngine (engine ``e``): up to
    K = e.max_symbols rounds of joint hidden (the encoder frame at x_enc, row stride ldx_enc, shared by an utterance's W
    rows) and logits, BEAM_SELECT (``sel``: its fields common to every round), GATHER of the parents' predictor (and
    LM) state, and the masked steps of the predictor ``dec`` and, with an LM, of the LM (``lm_step`` from lm_fusion).

    K = 1 is the one-symbol frame: the state alternates between the buffers by frame parity.  For K > 1 the number of
    rounds a frame runs is known only on the device (SKIP, greedy_frame), so the state ends every round in buffer 0:
    GATHER writes buffer 1 and one COPY moves it back."""
    K, R = e.max_symbols, e.R
    D = e.dec_x[0].shape[1]

    def round_phases(j):
        p, q = (t & 1, 1 - (t & 1)) if K == 1 else (0, 1)
        joint_phases(prog, e._joint, R, x_enc, ldx_enc, e.dec_x[p], e.hidden, e.logits, x1_div=e.W)
        ph = EbPhase(hist_col=t * K + j, seq_in=_ptr(e.seqs[p]), seq_out=_ptr(e.seqs[q]), **sel)
        if K > 1:
            ph.flags |= F_ROUNDS
            ph.ldw2 = K
        prog.append(ph)
        Ld, Hd = e._st[0].shape[0] // 2, e._st[0].shape[2]
        prog.append(EbPhase(type=PH_GATHER, S=R, N=Hd, aux=2 * Ld, x1=_ptr(e._st[p]), y=_ptr(e._st[q]), K2=D,
                            x2=_ptr(e.dec_x[p]), y2=_ptr(e.dec_x[q]), src=_ptr(e.src)))
        if e._lst is not None:
            prog.append(EbPhase(type=PH_GATHER, S=R, N=e._lst[0].shape[2], aux=e._lst[0].shape[0],
                                x1=_ptr(e._lst[p]), y=_ptr(e._lst[q]), src=_ptr(e.src)))
        if K > 1:
            prog.append(EbPhase(type=PH_COPY, S=1, N=e._home.shape[1], x1=_ptr(e._home[1]), y=_ptr(e._home[0])))
            q = 0
        _dec_phases(prog, dec, R, e.dec_h[q], e.dec_c[q], e.dec_htmp, e.dec_x[q], e.tok, e.blank, masked=True)
        if lm_step is not None:
            lm_step(prog, e.lm_h[q], e.lm_c[q], masked=True)

    greedy_frame(prog, K, R, e.tok, e.blank, round_phases)


def lm_state_dict(lm):
    """The fusion LM's weights as {key: tensor} in the layout of the reference's LMModel state_dict
    (``encoder.weight``, ``rnn.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}``, ``decoder.{weight,bias}``), from the
    module or from such a state_dict.  Raises TypeError / ValueError for anything else; touches no device."""
    import torch.nn as nn
    if isinstance(lm, nn.Module):
        enc, rnn, dec = (getattr(lm, n, None) for n in ("encoder", "rnn", "decoder"))
        if not (isinstance(enc, nn.Embedding) and isinstance(rnn, nn.LSTM) and isinstance(dec, nn.Linear)):
            raise TypeError("lm must have encoder = nn.Embedding, rnn = nn.LSTM and decoder = nn.Linear (LMModel)")
        if not rnn.batch_first or rnn.bidirectional or rnn.proj_size or not rnn.bias or dec.bias is None:
            raise ValueError("lm.rnn must be a batch_first, one-direction LSTM with biases and no proj_size, and "
                             "lm.decoder a Linear with bias")
        sd = {"encoder.weight": enc.weight, "decoder.weight": dec.weight, "decoder.bias": dec.bias}
        for k, w in enumerate(lstm_layers(rnn)):
            for n, t in zip(("weight_ih", "weight_hh", "bias_ih", "bias_hh"), w):
                sd["rnn.%s_l%d" % (n, k)] = t
    elif isinstance(lm, dict):
        sd = dict(lm)
    else:
        raise TypeError("lm must be an LMModel-like nn.Module or its state_dict, got %s" % type(lm).__name__)
    L = 0
    while "rnn.weight_ih_l%d" % L in sd:
        L += 1
    want = ["encoder.weight", "decoder.weight", "decoder.bias"] + \
        ["rnn.%s_l%d" % (n, k) for k in range(L) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    if L == 0 or set(sd) != set(want):
        raise ValueError("lm state_dict keys must be exactly %s, got %s" % (want if L else "encoder.weight, "
                         "rnn.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}, decoder.{weight,bias}", sorted(sd)))
    for k, t in sd.items():
        if not isinstance(t, torch.Tensor) or not t.is_floating_point():
            raise TypeError("lm weight %s must be a floating-point tensor" % k)
    sd = {k: t.detach() for k, t in sd.items()}
    ntok, ninp = sd["encoder.weight"].shape if sd["encoder.weight"].dim() == 2 else (0, 0)
    H = sd["rnn.weight_hh_l0"].shape[-1]
    shapes = {"encoder.weight": (ntok, ninp), "decoder.weight": (ntok, H), "decoder.bias": (ntok,)}
    for k in range(L):
        shapes.update({"rnn.weight_ih_l%d" % k: (4 * H, ninp if k == 0 else H), "rnn.weight_hh_l%d" % k: (4 * H, H),
                       "rnn.bias_ih_l%d" % k: (4 * H,), "rnn.bias_hh_l%d" % k: (4 * H,)})
    for k, s in shapes.items():
        if tuple(sd[k].shape) != s or 0 in s:
            raise ValueError("lm weight %s has shape %s, the layout needs %s" % (k, tuple(sd[k].shape), s))
    return sd


def _finite(name, v):
    if isinstance(v, bool) or not isinstance(v, numbers.Real):
        raise TypeError("%s must be a real number, got %r" % (name, v))
    v = float(v)
    if not math.isfinite(v):
        raise ValueError("%s must be finite, got %r" % (name, v))
    return v


def check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map, ngram=False):
    """Validate the shallow-fusion arguments of a beam search over a vocabulary of V tokens.  Returns
    (lm state_dict, lm_weight, length_bonus, lm_bos, token map int64 [V] on the host) or None without ``lm``.
    ``ngram``: an n-gram model is fused too, so length_bonus is legal without ``lm``.  Raises TypeError /
    ValueError; touches no device."""
    if lm is None:
        if lm_weight != 0.0 or (length_bonus != 0.0 and not ngram) or lm_token_map is not None:
            raise ValueError("lm_weight, length_bonus and lm_token_map need an lm")
        if ngram:
            _finite("length_bonus", length_bonus)
        return None
    sd = lm_state_dict(lm)
    ntok = sd["encoder.weight"].shape[0]
    vals = [_finite(name, v) for name, v in (("lm_weight", lm_weight), ("length_bonus", length_bonus))]
    lm_bos = operator.index(lm_bos)
    if not 0 <= lm_bos < ntok:
        raise ValueError("lm_bos must be in [0, %d), got %d" % (ntok, lm_bos))
    if lm_token_map is None:
        if ntok != V:
            raise ValueError("the LM has %d tokens and the transducer %d: pass lm_token_map" % (ntok, V))
        tmap = torch.arange(V)
    else:
        if not isinstance(lm_token_map, torch.Tensor) or lm_token_map.is_floating_point() or \
                lm_token_map.is_complex() or lm_token_map.dtype == torch.bool:
            raise TypeError("lm_token_map must be an integer tensor [%d]" % V)
        if tuple(lm_token_map.shape) != (V,):
            raise ValueError("lm_token_map must have shape [%d], got %s" % (V, tuple(lm_token_map.shape)))
        tmap = lm_token_map.detach().to("cpu", torch.int64)
        if bool(((tmap < -1) | (tmap >= ntok)).any()):
            raise ValueError("lm_token_map values must be in [-1, %d)" % ntok)
    return sd, vals[0], vals[1], lm_bos, tmap


def lm_fusion(e, fusion, R):
    """Shallow fusion on beam engine ``e`` (its ``dev`` and ``_keep`` set) over R rows, from check_lm_args' result:
    keeps the LM weights in e._keep (read in place when they already are fp32 on e.dev, so tied weights stay tied),
    allocates the LM scratch e.lm_htmp [Ll, R, Hl], e.lm_logits [R, ntok] and e.lm_tok, the token map e.lm_map and
    e.lm_fuse = (lm_weight, length_bonus), and sets e.lm_bos.  Returns the fields a BEAM_SELECT / CTC_BEAM phase reads
    the LM through (besides flag F_LM) and ``step(prog, h, c, masked)``, which appends one LM step on state h, c
    [Ll, R, Hl] (predictor_phases resting on -1)."""
    lsd, lw, lb, e.lm_bos, tmap = fusion
    lsd = {k: v.to(e.dev, torch.float32).contiguous() for k, v in lsd.items()}
    e._keep += list(lsd.values())
    Ll = (len(lsd) - 3) // 4
    layers = [tuple(lsd["rnn.%s_l%d" % (n, k)] for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
              for k in range(Ll)]
    Hl, ntok = layers[0][1].shape[1], lsd["encoder.weight"].shape[0]
    z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=e.dev)
    e.lm_htmp, e.lm_logits, e.lm_tok = z(Ll, R, Hl), z(R, ntok), z(R, dtype=torch.int32)
    e.lm_map = tmap.to(e.dev, torch.int32)
    e.lm_fuse = torch.tensor([lw, lb], dtype=torch.float32, device=e.dev)

    def step(prog, h, c, masked):
        predictor_phases(prog, lsd["encoder.weight"], layers, lsd["decoder.weight"], lsd["decoder.bias"], R, h, c,
                         e.lm_htmp, e.lm_logits, e.lm_tok, -1, masked)
    return dict(x2=_ptr(e.lm_logits), ldx2=ntok, K2=ntok, fuse=_ptr(e.lm_fuse), tok_map=_ptr(e.lm_map),
                tok_out2=_ptr(e.lm_tok)), step


def param_fingerprint(module):
    """Identity of the parameter storage a phase program was built over: the programs bake raw device pointers, so a
    re-homed parameter (FlatAdam bucket, .to(), .float(), p.data = ...) must trigger a rebuild."""
    return tuple(p.data_ptr() for p in module.parameters())


def _odd_chunk():
    return ValueError("streaming chunks must hold an even number of frames before each time reduction "
                      "(cli/export_onnx.py:20-21 asserts the same)")


def stream_frames_out(enc, n):
    """Encoder output frames of a streaming chunk of n input frames; ValueError when a time reduction meets an odd
    count.  Touches no device."""
    for i in range(len(enc.lstm.lstms)):
        if i in enc.lstm.time_reductions:
            if n % 2:
                raise _odd_chunk()
            n //= 2
    return n


def check_stream_shape(enc, n_streams, frames_per_chunk):
    """(S, n, encoder output frames per chunk) of a streaming engine; ValueError for S < 1, n < 1, an odd count before
    a time reduction or a chunk that gives no output frame.  Touches no device."""
    S, n = operator.index(n_streams), operator.index(frames_per_chunk)
    if S < 1 or n < 1:
        raise ValueError("n_streams and frames_per_chunk must be positive, got %d and %d" % (S, n))
    T = stream_frames_out(enc, n)
    if T < 1:
        raise ValueError("a chunk of %d frames gives no encoder output frame" % n)
    return S, n, T


def frontend_geometry(frontend, samples_per_chunk):
    """What a stream engine's device front end computes per window of L = ``samples_per_chunk`` samples: the operands
    and flags of the feature module of ``frontend`` (build_batch_transform's test module, a BatchTransform) and the
    window's frame arithmetic, as ops.fe_batch lays it out for one utterance of L samples: F = 1 + L // hop frames,
    Fs of them kept by Downsample (all with pad_to_divisible, else F - F % n_stack), T = ceil(Fs / n_stack) model input
    frames, the seq_len mask from frame ``seq`` on (logfbank; F for melspec and MFCC), ``Fc`` frames computed (Fs, or F
    when the deltas read up to frame F - 1), the reflect padding ``pad`` = n_fft // 2 and the padded row of ``Lp`` = R
    hop samples.  Raises TypeError / ValueError for a module that is not a BatchTransform, a train module that carries
    SpecAugment masks or L <= n_fft // 2; touches no device."""
    from .rnnt.features import BatchTransform, FilterbankFeatures, MelSpectrogram, MFCC
    if not isinstance(frontend, BatchTransform):
        raise TypeError("frontend must be a BatchTransform (build_batch_transform's test module), got %s"
                        % type(frontend).__name__)
    if (frontend.T_mask > 0 and frontend.T_num_mask > 0) or (frontend.F_mask > 0 and frontend.F_num_mask > 0):
        raise ValueError("frontend carries SpecAugment masks: stream with build_batch_transform's test module, as the "
                         "reference streams its test transform")
    f = frontend.features
    g = dict(dct=None, preemph=None, take_log=False, use_mask=False, dither=0.0)
    if isinstance(f, FilterbankFeatures):
        g.update(basis=f.dft_basis, fbT=f.fb_t, n_fft=f.n_fft, hop=f.hop_length, preemph=f.preemph, take_log=f.log,
                 use_mask=True, dither=float(f.dither))
    else:
        ms = f.MelSpectrogram if isinstance(f, MFCC) else f
        if not isinstance(ms, MelSpectrogram):
            raise TypeError("frontend.features must be FilterbankFeatures, MelSpectrogram or MFCC, got %s"
                            % type(f).__name__)
        g.update(basis=ms.spectrogram.dft_basis, fbT=ms.mel_scale.fb, n_fft=ms.n_fft, hop=ms.hop_length)
        if isinstance(f, MFCC):
            g["dct"] = f.dct_mat
    L = operator.index(samples_per_chunk)
    n_fft, hop, n_stack = g["n_fft"], g["hop"], frontend.downsample
    pad = n_fft // 2
    if L <= pad:
        raise ValueError("samples_per_chunk must exceed n_fft // 2 = %d (reflect padding), got %d" % (pad, L))
    F = 1 + L // hop
    Fs = F if frontend.pad_to_divisible else F - F % n_stack
    _, (T,) = ops.fe_lengths([L], hop, n_stack, frontend.pad_to_divisible)
    R = -(-(L + 2 * pad) // hop)
    g.update(L=L, pad=pad, R=R, Lp=R * hop, F=F, Fs=Fs, T=T, seq=-(-L // hop) if g["use_mask"] else F,
             Fc=F if frontend.delta else Fs, n_stack=n_stack, delta=frontend.delta, input_size=frontend.input_size)
    return g


def frontend_phases(engine, g, S):
    """The front-end program of engine ``engine`` (whose ``dev`` and ``xin`` [S, T, input_size] are set) for S streams
    of windows with frontend_geometry ``g``: FE_FRAME (dither, pre-emphasis, reflect padding), the direct-DFT FE_GEMM
    over the Fc computed frames of each stream (the strided frames of the padded row), FE_POWER, the mel FE_GEMM, for
    MFCC FE_LOG and the DCT FE_GEMM, and FE_FINISH into xin.  Allocates its buffers on ``engine``: ``audio`` [S, L],
    ``noise`` [S, L] (with dither, else None) and the intermediates; keeps the module's tables on the device in
    engine._keep.  Returns the phase list."""
    dev, L, Lp, Fc = engine.dev, g["L"], g["Lp"], g["Fc"]
    z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=dev)
    on_dev = lambda t: None if t is None else t.detach().to(dev, torch.float32).contiguous()
    basis, fbT, dct = on_dev(g["basis"]), on_dev(g["fbT"]), on_dev(g["dct"])
    nb2, n_mels = basis.shape[1], fbT.shape[1]
    M = S * Fc
    engine.audio = z(S, L)
    engine.noise = z(S, L) if g["dither"] > 0 else None
    pre = g["preemph"]
    engine._fe_consts = torch.tensor([g["dither"], float(pre or 0.0)], dtype=torch.float32, device=dev)
    xp, spec, power, feat = z(S * Lp + g["n_fft"]), z(M, nb2), z(M, nb2 // 2), z(M, n_mels)
    engine._fe_bufs = [xp, spec, power, feat]
    engine._keep += [t for t in (basis, fbT, dct) if t is not None]
    gemm = lambda x1, aux, ldx1, ldx2, K, w, y: EbPhase(type=PH_FE_GEMM, S=M, N=w.shape[1], K1=K, aux=aux, ldx1=ldx1,
                                                        ldx2=ldx2, x1=_ptr(x1), w1=_ptr(w), ldw1=w.shape[1], y=_ptr(y),
                                                        ldy=w.shape[1])
    fe = [EbPhase(type=PH_FE_FRAME, S=S, N=L, K1=g["pad"], ldy=Lp, x1=_ptr(engine.audio), x2=_ptr(engine.noise),
                  fuse=_ptr(engine._fe_consts), flags=int(pre is not None), y=_ptr(xp)),
          gemm(xp, Fc, Lp, g["hop"], g["n_fft"], basis, spec),
          EbPhase(type=PH_FE_POWER, S=M, N=nb2 // 2, x1=_ptr(spec), y=_ptr(power)),
          gemm(power, M, 0, nb2 // 2, nb2 // 2, fbT, feat)]
    if dct is not None:
        cep = z(M, dct.shape[1])
        engine._fe_bufs.append(cep)
        fe += [EbPhase(type=PH_FE_LOG, S=M, N=n_mels, x1=_ptr(feat), y=_ptr(feat)),
               gemm(feat, M, 0, n_mels, n_mels, dct, cep)]
        feat = cep
    C, T = feat.shape[1], g["T"]
    fe.append(EbPhase(type=PH_FE_FINISH, S=S, K1=Fc, N=C, aux=g["n_stack"], aux2=T, hist_ld=g["F"], hist_col=g["Fs"],
                      x1_div=g["seq"], flags=int(g["take_log"]) | (2 if g["delta"] else 0), x1=_ptr(feat),
                      y=_ptr(engine.xin), ldy=engine.xin.shape[1] * engine.xin.shape[2]))
    assert tuple(engine.xin.shape) == (S, T, C * (3 if g["delta"] else 1) * g["n_stack"])
    return fe


def encoder_phases(prog, engine, enc, S, n):
    """Append the stateful streaming encoder for S streams and chunks of n log-mel frames to the phase list ``prog``:
    LayerNorm of the input, then per layer n LSTM cell steps from the carried (h, c), the residual LayerNorm and the
    time reduction, then the projection.  Allocates on ``engine`` (whose ``dev`` is set) the chunk input ``xin``
    [S, n, F], the carried state ``enc_h`` / ``enc_c`` [L, S, H] (with ``enc_htmp``, the last step's h, which the
    chunk program's last phase copies into enc_h: _ChunkEngine._finish) and the output ``enc_out`` [S, n_out, E]; sets
    ``engine.n_out``.  A GRU encoder (ResLayerNormGRU) gets GRU cell steps instead, and its carried state is ``enc_h``
    alone (``enc_c`` is None); its programs run through eb_decode_run_ctc_stream (CTC) or eb_decode_run_gru_rnnt
    (transducer)."""
    from .rnnt.models import ResLayerNormGRU
    gru = isinstance(enc.lstm, ResLayerNormGRU)
    lstms = list(enc.lstm.lstms)
    L = len(lstms)
    H = enc.lstm.hidden_size
    F = enc.norm.weight.shape[0]
    reductions = enc.lstm.time_reductions
    z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=engine.dev)
    engine.xin, engine.a0 = z(S, n, F), z(S, n, F)
    engine.enc_h, engine.enc_c, engine.enc_htmp = z(L, S, H), None if gru else z(L, S, H), z(L, S, H)
    prog.append(EbPhase(type=PH_LN, S=S * n, N=F, x1=_ptr(engine.xin), ldx1=F, w1=_ptr(enc.norm.weight),
                        b1=_ptr(enc.norm.bias), y=_ptr(engine.a0), ldy=F))
    X, I, ni = engine.a0, F, n
    engine._bufs = []
    for i, (cell, post) in enumerate(zip(lstms, enc.lstm.projs)):
        yL, zL = z(S, ni, H), z(S, ni, H)
        engine._bufs += [yL, zL]
        for t in range(ni):
            prog.append(EbPhase(type=PH_GRU if gru else PH_LSTM, S=S, N=H, K1=I, K2=H, x1=_ptr(X, t * I), ldx1=ni * I,
                                x2=_ptr(engine.enc_h[i]) if t == 0 else _ptr(yL, (t - 1) * H),
                                ldx2=H if t == 0 else ni * H, w1=_ptr(cell.weight_ih_l0), ldw1=I,
                                w2=_ptr(cell.weight_hh_l0), ldw2=H, b1=_ptr(cell.bias_ih_l0), b2=_ptr(cell.bias_hh_l0),
                                c=None if gru else _ptr(engine.enc_c[i]), y=_ptr(yL, t * H), ldy=ni * H,
                                y2=_ptr(engine.enc_htmp[i]) if t == ni - 1 else None))
        ln = post[0]
        prog.append(EbPhase(type=PH_LN, S=S * ni, N=H, x1=_ptr(yL), ldx1=H, x2=_ptr(X) if i > 0 else None, ldx2=H,
                            w1=_ptr(ln.weight), b1=_ptr(ln.bias), y=_ptr(zL), ldy=H))
        X, I = zL, H
        if i in reductions:
            if ni % 2:
                raise _odd_chunk()
            zr = z(S, ni // 2, H)
            engine._bufs.append(zr)
            prog.append(EbPhase(type=PH_PAIR, S=S, N=H, aux=ni, x1=_ptr(zL), y=_ptr(zr)))
            X, ni = zr, ni // 2
    engine.n_out = ni
    E = enc.proj.weight.shape[0] if enc.has_proj else H
    if enc.has_proj:
        engine.enc_out = z(S, ni, E)
        prog.append(EbPhase(type=PH_LINEAR, S=S * ni, N=E, K1=H, x1=_ptr(X), ldx1=H, w1=_ptr(enc.proj.weight),
                            ldw1=H, b1=_ptr(enc.proj.bias), y=_ptr(engine.enc_out), ldy=E))
    else:
        engine.enc_out = X
    return E


def _upload(prog, dev):
    """The phase list ``prog`` as the device bytes a decode kernel entry reads."""
    assert C.sizeof(EbPhase) == lib().eb_decode_phase_size(), "EbPhase layout mismatch"
    arr = (EbPhase * len(prog))(*prog)
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev)


def _launch(entry, prog, nphase, bar, max_ctas):
    """Run the first nphase phases of the uploaded program ``prog`` through the decode kernel entry ``entry`` on the
    current stream; ``bar`` is the engine's grid barrier, which the entry zeroes at every launch."""
    check(getattr(lib(), entry)(prog.data_ptr(), nphase, bar.data_ptr(), max_ctas,
                                torch.cuda.current_stream().cuda_stream), entry)


class _ChunkEngine:
    """What the streaming engines (StreamEngine, StreamBeamEngine, CTCStreamEngine) share: the host-side checks in a
    fixed order (the encoder kind, check_stream_shape, then the CUDA device), the stateful encoder at the head of the
    chunk program and the COPY that closes it, the launches, and ``state()`` / ``load_state()`` over
    ``_state_views()``.

    Every engine takes ``frontend`` (build_batch_transform's test module) with ``samples_per_chunk`` = L: ``step`` then
    takes fp32 audio [S, L] on the device, one window per stream, and the chunk program opens with the feature
    transform (frontend_phases, in the same launch), which writes into ``xin`` bit for bit what ``frontend(audio, [L] *
    S)[0]`` gives.  frames_per_chunk then follows from L (None, or the same count).  No front-end state is carried
    between chunks: each window is transformed on its own, as the reference streams overlapping windows."""
    GRU = False          # the encoder kind: ResLayerNormGRU cells, carrying enc_h alone, or ResLayerNormLSTM cells
    HOST_STATE = ()      # keys of state() kept on the host, outside _state_views

    @functools.cached_property
    def RUN(self):
        """The decode kernel entry every program of the engine runs through (an instance may set another)."""
        return "eb_decode_run_gru_rnnt" if self.GRU else "eb_decode_run"

    def _check_shape(self, enc, n_streams, frames_per_chunk, frontend=None, samples_per_chunk=None):
        """check_stream_shape's (S, n, encoder output frames per chunk), after refusing an encoder of the other kind
        with ValueError.  With a ``frontend`` (see frontend_geometry) the chunk is L = ``samples_per_chunk`` samples of
        audio per stream, n follows from L, and a ``frames_per_chunk`` given as well must agree with it; the window
        must give at least one model input frame, and the module's input_size must be the encoder's input width.
        Sets ``_fe`` (the geometry, or None).  Touches no device."""
        from .rnnt.models import ResLayerNormGRU, ResLayerNormLSTM
        if not isinstance(enc.lstm, ResLayerNormGRU if self.GRU else ResLayerNormLSTM):
            # the encoder phases are cells of one kind: LSTM (4H-row weights) or GRU (3H rows)
            who, kind, got = type(self).__name__, "a GRU" if self.GRU else "an LSTM", type(enc.lstm).__name__
            raise ValueError("%s streams %s encoder only, got %s" % (who, kind, got))
        self._fe = None
        if frontend is None:
            if samples_per_chunk is not None:
                raise ValueError("samples_per_chunk needs a frontend")
            return check_stream_shape(enc, n_streams, frames_per_chunk)
        if samples_per_chunk is None:
            raise ValueError("a frontend needs samples_per_chunk, the audio samples of a chunk per stream")
        g = frontend_geometry(frontend, samples_per_chunk)
        if g["T"] < 1:
            raise ValueError("a window of %d samples gives %d frames, no model input frame after stacking by %d"
                             % (g["L"], g["F"], g["n_stack"]))
        if frames_per_chunk is not None and operator.index(frames_per_chunk) != g["T"]:
            raise ValueError("frames_per_chunk (%d) disagrees with the %d model input frames a window of %d samples "
                             "gives" % (operator.index(frames_per_chunk), g["T"], g["L"]))
        F = enc.norm.weight.shape[0]
        if g["input_size"] != F:
            raise ValueError("frontend.input_size (%d) differs from the encoder's input width (%d)"
                             % (g["input_size"], F))
        self._fe = g
        return check_stream_shape(enc, n_streams, g["T"])

    def _build_encoder(self, prog, model, enc, S, n, T):
        """After every other check, the CUDA device check; then encoder_phases into ``prog`` (T output frames per
        chunk).  The program reads ``model``'s weights in place: they are kept, and ``fingerprint`` tells when they
        move.  Returns the encoder output width E."""
        self.dev = enc.norm.weight.device
        if self.dev.type != "cuda":
            raise RuntimeError("%s needs the model on a CUDA device" % type(self).__name__)
        self._keep = [p.detach() for p in model.parameters()]
        self.fingerprint = param_fingerprint(model)
        self._bar = torch.zeros(64, dtype=torch.int32, device=self.dev)
        E = encoder_phases(prog, self, enc, S, n)
        assert self.n_out == T
        if self._fe is not None:                             # the front end opens the chunk program
            fe = frontend_phases(self, self._fe, S)
            self._fe_prog = _upload(fe, self.dev)
            prog.insert(0, EbPhase(type=PH_GATHER, flags=F_FRONTEND, x1=_ptr(self._fe_prog), K1=len(fe),
                                   tok_out=_ptr(self._bar, 1)))
        return E

    def _finish(self, prog, state):
        """Close the chunk program ``prog`` with the COPY of the encoder's last h into the carried enc_h and upload it;
        then start every stream from ``state`` (a rebuilt program continues the utterance, rnnt/stream.py:97-98), or
        from ``reset()`` without one."""
        L, S, H = self.enc_h.shape
        prog.append(EbPhase(type=PH_COPY, S=L * S, N=H, x1=_ptr(self.enc_htmp), y=_ptr(self.enc_h)))
        self._chunk, self.n_chunk_phases = _upload(prog, self.dev), len(prog)
        if state is None:
            self.reset()
        else:
            self.load_state(state)

    def _run(self, prog, nphase):
        _launch(self.RUN, prog, nphase, self._bar, self.max_ctas)

    def _load(self, chunk):
        """Put a chunk where the chunk program reads it: log-mel frames [S, n, F] (device or pinned host) into xin, or
        with a front end fp32 audio [S, L] on the engine's device into ``audio`` and, with dither, N(0, 1) noise from
        the current generator into ``noise`` (what the module's randn_like(x) draws).  ValueError for a chunk of the
        wrong shape, dtype or device, before any device work."""
        if self._fe is None:
            self.xin.copy_(chunk, non_blocking=True)
            return
        if not isinstance(chunk, torch.Tensor) or chunk.dtype != torch.float32 or chunk.device != self.dev or \
                tuple(chunk.shape) != tuple(self.audio.shape):
            raise ValueError("with a front end a chunk is fp32 audio %s on %s, got %s" % (
                list(self.audio.shape), self.dev, "%s %s on %s" % (chunk.dtype, list(chunk.shape), chunk.device)
                if isinstance(chunk, torch.Tensor) else type(chunk).__name__))
        self.audio.copy_(chunk)
        if self.noise is not None:
            torch.randn(self.noise.shape, device=self.dev, out=self.noise)

    def _fetch(self, width):
        """Copy ``_out`` (ids [S, width] | counts [S] | any further values) to the pinned ``_host``: the chunk's only
        device-to-host copy.  -> (ids [S, width], counts [S], the further values) on the host."""
        S = self.S
        self._host.copy_(self._out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        rest = self._host[S * width:].clone()
        return self._host[:S * width].view(S, width).clone(), rest[:S], rest[S:]

    def _state_views(self):
        v = dict(enc_h=self.enc_h)
        if self.enc_c is not None:                           # a GRU encoder carries h alone
            v["enc_c"] = self.enc_c
        return v

    def state(self):
        """The recurrent state of every stream (what PytorchStreamDecoder carries between chunks, rnnt/stream.py:78-91),
        as a dict of device tensors."""
        return {k: t.clone() for k, t in self._state_views().items()}

    @torch.no_grad()
    def load_state(self, st):
        """Continue from ``state()`` of an engine of the same kind over the same model and n_streams, with any chunk
        length or re-homed weights."""
        views = self._state_views()
        if set(st) != set(views) | set(self.HOST_STATE):
            raise ValueError("state keys %s do not match this engine's %s (an LSTM encoder carries enc_h and enc_c, a "
                             "GRU encoder enc_h alone; a beam needs the same LM use)"
                             % (sorted(st), sorted(set(views) | set(self.HOST_STATE))))
        for k, t in views.items():
            if tuple(st[k].shape) != tuple(t.shape):
                raise ValueError("state %s has shape %s, this engine needs %s (same model and n_streams, and for a "
                                 "beam the same W and max_pending)" % (k, tuple(st[k].shape), tuple(t.shape)))
            t.copy_(st[k])


class _CommitEngine(_ChunkEngine):
    """What the streaming beams (StreamBeamEngine, CTCStreamBeamEngine) share beyond _ChunkEngine: the chunk end that
    commits each stream's common prefix with BEAM_COMMIT (``_chunk_end``, which each engine appends for its own state),
    the flush and re-bound programs built from it, and the host bookkeeping of committed tokens: ``step`` / ``flush``
    return them, ``state()`` carries those not yet returned, and ``load_state`` re-bounds the carried beam.  The beam
    rests in the parity-0 buffers between launches; ``logp`` [S*W] is the value BEAM_COMMIT collapses by.

    With contextual biasing (``_context``) each slot's phrase-automaton state ``ctx_state`` (two parities) rides along:
    the chunk end copies it beside the rest of the beam, BEAM_COMMIT collapses by logp - pending[state] and moves it
    with its slot, ``flush`` reports that value, and ``state()`` carries it with the graph's fingerprint."""
    UNRETURNED = ("unreturned_ids", "unreturned_counts")
    HOST_STATE = UNRETURNED
    _graph = _cf = None          # the ContextGraph and context_program's fields, with contextual biasing

    def _context(self, graph, sel):
        """Contextual biasing with the checked ContextGraph ``graph`` (None: none), the slot states ``ctx_state`` already
        allocated: uploads the tables and adds the flag and descriptor to the search phase's fields ``sel``.  The chunk
        end's BEAM_COMMIT then reads them too (_commit_phase), and state() gains the key ``context``."""
        if graph is None:
            return
        self._graph, self._cf = graph, context_program(self, graph, self.ctx_state)
        self._pending = torch.from_numpy(graph.pending).to(self.dev)
        sel.update(flags=sel["flags"] | F_CONTEXT, ctx=self._cf["ctx"])
        self.HOST_STATE = self.UNRETURNED + ("context",)

    def _chunk_end(self, pr, in_parity0, flush):
        """Append the chunk end to ``pr``: commit (and collapse) from parity 1 into parity 0, the state found in parity 0
        (``in_parity0``) copied over first; ``flush`` collapses unconditionally."""
        raise NotImplementedError

    def _commit_buffers(self):
        """The chunk end's output, committed ids [S, max_pending] | counts [S] | collapsed [S], and its host copy."""
        S, P = self.S, self.max_pending
        self._out = torch.zeros(S * P + 2 * S, dtype=torch.int32, device=self.dev)
        self._host = torch.zeros(self._out.shape, dtype=torch.int32).pin_memory()
        self.n_collapses = 0

    def _commit_phase(self, flush, n_add, **kw):
        """BEAM_COMMIT of every stream from parity 1 into parity 0, for chunks that add up to ``n_add`` tokens to a
        hypothesis; ``kw`` adds the row head (K2) and the last-token buffer (y2) of CTC rows."""
        S, P = self.S, self.max_pending
        if self._cf is not None:                 # the automaton states: parity 1 in, parity 0 out
            kw.update(ctx=self._cf["ctx"])
        return EbPhase(type=PH_BEAM_COMMIT, S=S, N=P, aux=self.W, aux2=P - n_add, K1=self.seqs[0].shape[1],
                       flags=(F_FLUSH if flush else 0) | (F_CONTEXT if self._cf is not None else 0), y=_ptr(self.logp),
                       hist=_ptr(self.hist), hist_ld=self.hist_live.shape[1], seq_in=_ptr(self.seqs[1]),
                       seq_out=_ptr(self.seqs[0]), tok_out=_ptr(self._out), tok_out2=_ptr(self._out, S * P),
                       src=_ptr(self.src), **kw)

    def _commit_programs(self, prog, in_parity0):
        """Close the chunk program ``prog`` with the chunk end (the frames left the state in parity 0 when
        ``in_parity0``) and build the flush and the re-bound programs, which find the state in parity 0."""
        self._chunk_end(prog, in_parity0, flush=False)
        flush, rebound = [], []
        self._chunk_end(flush, True, flush=True)
        self._chunk_end(rebound, True, flush=False)   # a loaded beam under this engine's bound
        self._flush, self._rebound = _upload(flush, self.dev), _upload(rebound, self.dev)
        self.n_flush_phases, self.n_rebound_phases = len(flush), len(rebound)

    def _reset_commits(self):
        """One live slot per stream (the caller starts its state) and nothing committed but not returned."""
        self.hist_live[:, -1] = 1
        self._unreturned = (torch.zeros(self.S, 0, dtype=torch.int32), torch.zeros(self.S, dtype=torch.int32))

    def state(self):
        """Every stream's encoder state and beam, as a dict of tensors, with the committed tokens not yet returned by
        ``step`` (host ids [S, K] and counts [S])."""
        st = super().state()
        st["unreturned_ids"], st["unreturned_counts"] = (t.clone() for t in self._unreturned)
        if self._graph is not None:
            st["context"] = self._graph.fingerprint
        return st

    def _check_context_state(self, st):
        """ValueError, before any device work, for a state carried with another context graph, with or without
        contextual biasing where this engine differs, or with a live slot's automaton state outside [0, n_states)."""
        mine, theirs = (self._graph.fingerprint if self._graph is not None else None), st.get("context")
        if (mine is None) != (theirs is None):
            raise ValueError("the state was carried %s contextual biasing and this engine decodes %s it; build the "
                             "engine with the same context" % (("with", "without") if mine is None else
                                                               ("without", "with")))
        if mine is None:
            return
        if theirs != mine:
            raise ValueError("the state was carried with another context graph (fingerprint %s, this engine's %s): "
                             "build a new engine and reset() to change the phrases" % (theirs, mine))
        cs, live = st.get("ctx_state"), st.get("live")
        if not isinstance(cs, torch.Tensor) or not isinstance(live, torch.Tensor) or \
                tuple(cs.shape) != (self.R,) or tuple(live.shape) != (self.S,):
            return                                       # the key and shape checks of load_state refuse it
        cs = cs.to("cpu", torch.int64).view(self.S, self.W)
        used = torch.arange(self.W)[None, :] < live.to("cpu", torch.int64)[:, None]
        bad = used & ((cs < 0) | (cs >= self._graph.n_states))
        if bool(bad.any()):
            s, j = (int(v) for v in bad.nonzero()[0])
            raise ValueError("state ctx_state: live slot %d of stream %d holds automaton state %d, outside [0, %d)"
                             % (j, s, int(cs[s, j]), self._graph.n_states))

    @torch.no_grad()
    def load_state(self, st):
        """Continue from ``state()`` of an engine of the same kind over the same model, LM, n_streams, W and max_pending,
        with any chunk length.  The previous engine bounded every stored suffix by max_pending minus ITS n_out; when
        this engine's chunks yield more encoder frames, that bound is too loose, so the chunk-end commit and collapse
        rule runs once here with this engine's bound.  The tokens it commits are returned by the next ``step``.  With
        contextual biasing the state must come from an engine with the same graph (its fingerprint), and every live
        slot's automaton state must lie in [0, n_states); ValueError otherwise, before any device work."""
        self._check_context_state(st)
        super().load_state(st)
        self._unreturned = tuple(st[k].to("cpu", torch.int32) for k in self.UNRETURNED)
        self._run(self._rebound, self.n_rebound_phases)
        ids, counts, collapsed = self._fetch(self.max_pending)
        self.n_collapses += int(collapsed.sum())
        self._add_unreturned(ids, counts)

    def _add_unreturned(self, ids, counts):
        """Append committed tokens (ids [S, K], counts [S]) to those not yet returned."""
        uids, ucounts = self._unreturned
        n = ucounts + counts
        out = torch.zeros(self.S, int(n.max()), dtype=torch.int32)
        for s in range(self.S):
            a, b = int(ucounts[s]), int(counts[s])
            out[s, :a] = uids[s, :a]
            out[s, a:a + b] = ids[s, :b]
        self._unreturned = (out, n)

    def _take(self, ids, counts):
        """The tokens just committed, after any committed earlier and not yet returned."""
        if int(self._unreturned[1].max()) > 0:
            self._add_unreturned(ids, counts)
            ids, counts = self._unreturned
            self._unreturned = (ids[:, :0].clone(), torch.zeros_like(counts))
        return ids, counts

    @torch.no_grad()
    def step(self, chunk):
        """chunk [S, n, F] log-mel frames (device or pinned host), or with a front end fp32 audio [S, L] on the device,
        -> (committed ids int32 [S, K], counts int32 [S]) on
        the host: row s holds in its first counts[s] entries the tokens stream s committed in this chunk.  K is
        max_pending, or more on the first step after load_state had to commit carried tokens (they come first).
        ``n_collapses`` counts the forced collapses so far."""
        self._load(chunk)
        self._run(self._chunk, self.n_chunk_phases)
        ids, counts, collapsed = self._fetch(self.max_pending)
        self.n_collapses += int(collapsed.sum())
        return self._take(ids, counts)

    @torch.no_grad()
    def flush(self):
        """Collapse every stream's beam to its best hypothesis and commit all of that hypothesis' remaining tokens;
        decoding continues from it.  -> (ids int32 [S, K], counts int32 [S] as from ``step``, -log p [S] of the best
        hypothesis, the negated fused score with an LM), on the host.  With contextual biasing the score is
        -(value - pending[state]) in fp32, what BEAM_FINAL reports: a phrase only partly matched earns nothing."""
        self._run(self._flush, self.n_flush_phases)
        ids, counts, _ = self._fetch(self.max_pending)
        ids, counts = self._take(ids, counts)
        y = self.logp.view(self.S, self.W)[:, 0]
        if self._graph is not None:
            y = y - self._pending[self.ctx_state[0].view(self.S, self.W)[:, 0].long()]
        return ids, counts, -y.cpu()


class StreamEngine(_ChunkEngine):
    STATE = ("enc_h", "enc_c", "dec_h", "dec_c", "dec_x", "tok")   # the carried state (enc_c: None for a GRU encoder)

    def __init__(self, transducer, n_streams, frames_per_chunk, unk_id=UNK, blank=NUL, max_ctas=0, state=None,
                 max_symbols=1, frontend=None, samples_per_chunk=None):
        """``max_symbols`` = K: per output frame up to K rounds of joint -> argmax (with the <unk> rule) -> masked
        predictor step; a stream's frame ends at its first blank or after K non-blank tokens.  ``step`` then returns
        [S, n_out * K]: K entries per frame, blank for the rounds a stream did not take."""
        K = check_max_symbols(max_symbols)
        enc, dec, joint = transducer.encoder, transducer.decoder, transducer.joint.joint
        S, n, T = self._check_shape(enc, n_streams, frames_per_chunk, frontend, samples_per_chunk)
        self.S, self.n, self.blank, self.unk, self.max_ctas, self.max_symbols = S, n, blank, unk_id, max_ctas, K
        prog = []
        E = self._build_encoder(prog, transducer, enc, S, n, T)
        # ---- predictor + joint state
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=self.dev)
        Ld, Hd = dec.lstm.num_layers, dec.lstm.hidden_size
        D = dec.proj.weight.shape[0]
        J, V = joint[0].weight.shape[0], joint[2].weight.shape[0]
        assert joint[0].weight.shape[1] == E + D
        self.dec_h, self.dec_c, self.dec_htmp = z(Ld, S, Hd), z(Ld, S, Hd), z(Ld, S, Hd)
        self.dec_x, self.hidden, self.logits = z(S, D), z(S, J), z(S, V)
        self.tok = torch.zeros(S, dtype=torch.int32, device=self.dev)
        self.hist = torch.zeros(S, T * K, dtype=torch.int32, device=self.dev)
        self._joint = (joint[0].weight, joint[0].bias, joint[2].weight, joint[2].bias)
        for k in range(T):
            greedy_frame(prog, K, S, self.tok, blank,
                         lambda j: greedy_round(prog, self, dec, self.enc_out, k, j, 0, unk_id))
        prime = []
        _dec_phases(prime, dec, S, self.dec_h, self.dec_c, self.dec_htmp, self.dec_x, self.tok, blank,
                    masked=False)                  # priming program: tok = BOS from a zero state
        self._prime, self.n_prime_phases = _upload(prime, self.dev), len(prime)
        self._finish(prog, state)

    def _state_views(self):
        return {k: getattr(self, k) for k in self.STATE if getattr(self, k) is not None}

    @torch.no_grad()
    def reset(self):
        """PytorchStreamDecoder.reset (rnnt/stream.py:78-91) for every stream."""
        for t in (self.enc_h, self.enc_c, self.dec_h, self.dec_c):
            if t is not None:
                t.zero_()
        self.tok.fill_(BOS)
        self._run(self._prime, self.n_prime_phases)

    @torch.no_grad()
    def step(self, chunk):
        """chunk [S, n, F] log-mel frames (device or pinned host), or with a front end fp32 audio [S, L] on the device,
        -> int32 [S, n_out * max_symbols] token ids, the
        max_symbols rounds of each frame in order (blank = 0 means 'no symbol in this round')."""
        self._load(chunk)
        if self.max_symbols > 1:
            self.hist.fill_(self.blank)             # the columns of rounds skipped for every stream are not written
        self._run(self._chunk, self.n_chunk_phases)
        return self.hist


class GreedyEngine:
    """Device-side batched greedy decode (reference Transducer.greedy_decode, rnnt/models.py:243-269):
    the T' per-frame iterations (joint -> log_softmax/argmax -> predictor step for every row -> keep
    the new state only where the prediction is non-blank) run inside ONE cooperative kernel launch as
    a phase program over the encoder output, instead of T' Python iterations of ~10 launches each."""

    def __init__(self, transducer, batch, t_out, blank=NUL, max_ctas=0, max_symbols=1):
        """``max_symbols`` = K: per encoder frame up to K rounds of joint -> argmax -> masked predictor step; a row's
        frame ends at its first blank or after K non-blank tokens (the predictor has then stepped on the K-th).  log p
        accumulates over every round taken; ``hist`` is [B, T' * K], frame-major, blank for rounds not taken."""
        K = check_max_symbols(max_symbols)
        dec, joint = transducer.decoder, transducer.joint.joint
        self.dev = dec.embed.weight.device
        if self.dev.type != "cuda":
            raise RuntimeError("GreedyEngine needs the model on a CUDA device")
        f32 = torch.float32
        B, T = batch, t_out
        self.B, self.T, self.blank, self.max_ctas, self.max_symbols = B, T, blank, max_ctas, K
        z = lambda *shape: torch.zeros(*shape, dtype=f32, device=self.dev)
        Ld, Hd = dec.lstm.num_layers, dec.lstm.hidden_size
        D = dec.proj.weight.shape[0]
        J, V = joint[0].weight.shape[0], joint[2].weight.shape[0]
        E = joint[0].weight.shape[1] - D
        self.h_enc = z(B, T, E)
        self.dec_h, self.dec_c, self.dec_htmp = z(Ld, B, Hd), z(Ld, B, Hd), z(Ld, B, Hd)
        self.dec_x, self.hidden, self.logits = z(B, D), z(B, J), z(B, V)
        self.tok = torch.zeros(B, dtype=torch.int32, device=self.dev)
        self.hist = torch.zeros(B, T * K, dtype=torch.int32, device=self.dev)
        self.logp = z(B)
        self._keep = [p.detach() for p in transducer.parameters()]
        self._joint = (joint[0].weight, joint[0].bias, joint[2].weight, joint[2].bias)
        prog = []
        _dec_phases(prog, dec, B, self.dec_h, self.dec_c, self.dec_htmp, self.dec_x, self.tok, blank,
                    masked=False)                   # prime with BOS from the zero state
        for k in range(T):
            greedy_frame(prog, K, B, self.tok, blank,
                         lambda j: greedy_round(prog, self, dec, self.h_enc, k, j, F_LOGP, -1, self.logp))
        self.nphase = len(prog)
        self._prog = _upload(prog, self.dev)
        self._bar = torch.zeros(64, dtype=torch.int32, device=self.dev)

    @torch.no_grad()
    def run(self, h_enc):
        """h_enc [B, T', E] -> (ids int32 [B, T' * max_symbols] incl. blanks, sum of log p [B])."""
        self.h_enc.copy_(h_enc)
        for t in (self.dec_h, self.dec_c, self.logp):
            t.zero_()
        if self.max_symbols > 1:
            self.hist.fill_(self.blank)             # the columns of rounds skipped for every row are not written
        self.tok.fill_(BOS)
        _launch("eb_decode_run", self._prog, self.nphase, self._bar, self.max_ctas)
        return self.hist, self.logp


class BeamEngine:
    """Device-side batched beam search (Transducer.beam_search): the time-synchronous beam under greedy_decode's
    emission rule (at most one symbol per encoder frame, or K with ``max_symbols`` = K: see beam_frame and
    Transducer.beam_search) for B utterances of W slots each, in ONE cooperative kernel launch.  Row r = b*W + j
    holds slot j of utterance b.  Per frame: joint hidden (the encoder frame shared by the utterance's W rows) and logits for every row, BEAM_SELECT (log-softmax, exact top-W of the live slots' candidates,
    ties to the lowest flat index slot*V + token, merge of equal token sequences by log-add when ``merge``), GATHER of
    the parents' predictor state, and the masked predictor step for the survivors that emitted a non-blank.  The
    predictor state alternates between two buffers by frame parity (a permutation cannot be gathered in place; with
    K > 1 every round gathers into buffer 1 and copies back to buffer 0).
    BEAM_FINAL picks the best live slot of each utterance and walks its back-pointers.

    ``hist_parent`` / ``hist_token`` / ``hist_logp`` [B, T', W] and ``hist_live`` [B, T'] keep the beam of every
    frame (slots below the live count are live; frames at or past an utterance's length repeat its last beam).

    With ``lm`` (the reference's LMModel or its state_dict, see check_lm_args) the LM is fused into the candidate
    values (shallow fusion, decode.cu flag 32): each slot carries an LM state ``lm_h`` / ``lm_c`` (two parities, like
    the predictor's), primed with ``lm_bos`` and stepped with ``lm_token_map[k]`` only when the slot emitted a
    non-blank token k the LM scores; after the predictor step, the LM's output Linear recomputes ``lm_logits`` for all
    rows (a row that did not step gets its parent's logits bit for bit, rows being independent).

    With ``context`` (a ContextGraph over the transducer's V tokens, edgedict_b200.context) each slot carries its
    phrase-automaton state (``ctx_state``, two parities beside the token sequences) and BEAM_SELECT adds the
    automaton's increment to every non-blank candidate's fusion term (decode.cu flag 2048); BEAM_FINAL ranks by the
    value minus the pending bonus of the slot's state.  An empty graph builds the program without context.

    With ``ngram`` (an NgramLM over the transducer's V tokens, edgedict_b200.ngram) each slot carries its n-gram state
    (``ng_state``, two parities beside the token sequences, every slot at the model's start state after ``run``'s
    reset); BEAM_SELECT builds each slot's row of g(state, .) in ``ng_row`` and adds ngram_weight * g right after the LM
    term (decode.cu flag 4096), and BEAM_FINAL adds ngram_weight * e(state).  Transducer.beam_search states the rule."""

    def __init__(self, transducer, batch, t_out, W, merge=True, blank=NUL, max_ctas=0, lm=None, lm_weight=0.0,
                 length_bonus=0.0, lm_bos=1, lm_token_map=None, max_symbols=1, nbest=0, context=None, ngram=None,
                 ngram_weight=0.0):
        """``max_symbols`` = K: up to K rounds per encoder frame (Transducer.beam_search states the rule).  The history
        then has one column per round, [B, T' * K, W] (column t*K + j; a round a row did not take holds parent = slot,
        token = blank and live count 0, except the last column, which holds the final live count), and ``ids`` is
        [B, T' * K].  ``nbest`` = N in [1, W]: BEAM_FINAL writes the N best hypotheses with their frames into
        ``nbest_out`` (final_outputs' layout, L = max(T' * K, 1)); 0 builds the best-only program."""
        K = check_max_symbols(max_symbols)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width must be in [1, %d], got %r" % (BEAM_MAX_W, W))
        N = _engine_nbest(nbest, W)
        model = check_ngram(ngram, transducer.joint.joint[2].weight.shape[0], blank)
        ng_w = check_ngram_weight(model, ngram_weight)
        fusion = check_lm_args(lm, transducer.joint.joint[2].weight.shape[0], lm_weight, length_bonus, lm_bos,
                               lm_token_map, ngram=model is not None)
        graph = check_context(context, transducer.joint.joint[2].weight.shape[0], blank)
        dec, joint = transducer.decoder, transducer.joint.joint
        self.dev = dec.embed.weight.device
        if self.dev.type != "cuda":
            raise RuntimeError("BeamEngine needs the model on a CUDA device")
        f32, i32 = torch.float32, torch.int32
        B, T, R = batch, t_out, batch * W
        TK = T * K                                             # history columns: one per round
        self.B, self.T, self.W, self.R, self.merge, self.blank, self.max_ctas, self.max_symbols = \
            B, T, W, R, merge, blank, max_ctas, K
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=self.dev)
        Ld, Hd = dec.lstm.num_layers, dec.lstm.hidden_size
        D = dec.proj.weight.shape[0]
        J, V = joint[0].weight.shape[0], joint[2].weight.shape[0]
        E = joint[0].weight.shape[1] - D
        self.h_enc, self.frames = z(B, T, E), z(B, dtype=i32)
        self._keep = [p.detach() for p in transducer.parameters()]
        self.lm = fusion is not None
        lm_sel, lm_step = lm_fusion(self, fusion, R) if self.lm else ({}, None)
        # per parity: predictor state, its output, {len, hash lo, hash hi, tokens} per row and the LM state
        beam_state(self, R, Ld, Hd, D, TK + 3, context=graph is not None, ngram=model is not None)
        self.dec_htmp, self.hidden, self.logits = z(Ld, R, Hd), z(R, J), z(R, V)
        self.tok, self.src, self.logp = z(R, dtype=i32), z(R, dtype=i32), z(R)
        beam_history(self, B, TK, W)
        self._slots = torch.arange(W, dtype=i32, device=self.dev)
        final_outputs(self, B, N, max(TK, 1))
        self._joint = (joint[0].weight, joint[0].bias, joint[2].weight, joint[2].bias)
        prog = []
        _dec_phases(prog, dec, R, self.dec_h[0], self.dec_c[0], self.dec_htmp, self.dec_x[0], self.tok, blank,
                    masked=False)                         # prime every row with BOS from the zero state
        if self.lm:
            lm_step(prog, self.lm_h[0], self.lm_c[0], masked=False)    # prime every row with lm_bos from zeros
        sel = dict(type=PH_BEAM_SELECT, S=B, N=V, aux=W, aux2=blank,
                   flags=(F_MERGE if merge else 0) | (F_LM if self.lm else 0), x1=_ptr(self.logits), ldx1=V,
                   y=_ptr(self.logp), tok_in=_ptr(self.frames), tok_out=_ptr(self.tok), src=_ptr(self.src),
                   hist=_ptr(self.hist), hist_ld=TK, **lm_sel)
        cf = fusion_fields(self, sel, graph, self.ctx_state, model, self.ng_state, ng_w, length_bonus, R, V)
        ctx = None if cf is None else (cf, T & 1 if K == 1 else 0)   # where the last frame left the states (beam_frame)
        for t in range(T):
            beam_frame(prog, self, dec, t, _ptr(self.h_enc, t * E), T * E, sel, lm_step)
        prog.append(final_phase(self, W, self.logp, K, ctx))
        self.nphase = len(prog)
        self._prog = _upload(prog, self.dev)
        self._bar = torch.zeros(64, dtype=torch.int32, device=self.dev)

    @torch.no_grad()
    def run(self, h_enc, frames):
        """h_enc [B, T', E], frames int32 [B] on the device (encoder frames each utterance decodes, <= T') ->
        (ids int32 [B, max(T', 1)]: the best hypothesis' non-blank tokens right-aligned, -1 before them;
        -log p [B] of that hypothesis, the negated fused score with an LM).  With ``nbest`` it returns ``nbest_out``
        (nbest_lists reads it), rank 0 of which holds those same values."""
        self.h_enc.copy_(h_enc)
        self.frames.copy_(frames)
        beam_reset(self)
        if self.max_symbols > 1 and self.T > 0:  # what a round a row does not take leaves: parent = slot, token = blank
            self.hist_parent.copy_(self._slots.expand_as(self.hist_parent))
            self.hist_token.fill_(self.blank)
            self.hist_live.zero_()
            self.hist_live[:, -1] = 1                           # the live count every round reads and writes
        _launch("eb_decode_run", self._prog, self.nphase, self._bar, self.max_ctas)
        return self.nbest_out if self.nbest else (self.ids, self.nlogp)


class StreamBeamEngine(_CommitEngine):
    """Streaming beam search: S streams of W hypotheses each, carried from one chunk to the next, one persistent kernel
    launch per chunk.  The chunk program runs StreamEngine's stateful encoder, then per encoder output frame exactly
    BeamEngine's frame (joint, BEAM_SELECT, GATHER, masked predictor and LM steps, with or without LM fusion), so how
    the audio is cut into chunks does not change which hypotheses survive.  Row r = s*W + slot.

    After the chunk's last frame BEAM_COMMIT commits each stream's longest common prefix of its live hypotheses' token
    sequences: no later frame can change it, so it is final and ``step`` returns it while audio is still arriving.
    Each slot stores only its uncommitted suffix, at most ``max_pending`` tokens.  If after the commit a live suffix
    holds more than ``max_pending - n_out`` tokens (a chunk adds at most n_out), the beam collapses: the best live
    slot (highest log p, lowest slot on ties) commits its whole suffix and becomes slot 0, the only live slot, with its
    log p, predictor state and LM state.  ``flush()`` is that collapse done unconditionally.

    The beam state (slot log p, token sequences, live counts, predictor and LM states) lives in the parity-0 buffers
    between launches, whatever the parity of n_out: the chunk-end phases read the other parity (copied there first
    when n_out is even, since GATHER is not in-place safe) and write parity 0.  ``state()`` / ``load_state()`` carry
    it to an engine rebuilt for another chunk length or re-homed weights.  The carried beam was bounded for the old
    n_out; load_state runs the chunk-end rule once with the new bound (a longer chunk may need a collapse) and the
    tokens that commits come first in the next ``step``'s output.

    The reference's ``<unk>`` rule (re-argmax when the argmax is ``<unk>``) is a device of the greedy loop; the beam,
    like Transducer.beam_search, does not apply it.

    With ``context`` (a ContextGraph over the transducer's V tokens, edgedict_b200.context) every slot carries its
    phrase-automaton state from chunk to chunk, as BeamEngine's slots do from frame to frame: BEAM_SELECT adds the
    automaton's increment, a collapse picks the live slot of highest log p - pending[state] (BEAM_FINAL's ranking), and
    ``flush`` returns -(log p - pending[state]).  A phrase may straddle chunks and commits, so the committed ids plus
    ``flush`` are BeamEngine(context=...)'s best hypothesis on the concatenated encoder output, its -log p bit for bit,
    when no forced collapse happens.  ``state()`` carries the states and the graph's fingerprint; ``load_state``
    refuses a state of another graph, or of an engine that differs in using context.  An empty graph builds the program
    without context."""

    def __init__(self, transducer, n_streams, frames_per_chunk, W, merge=True, lm=None, lm_weight=0.0,
                 length_bonus=0.0, lm_bos=1, lm_token_map=None, max_pending=64, state=None, blank=NUL, max_ctas=0,
                 max_symbols=1, frontend=None, samples_per_chunk=None, context=None):
        K = check_max_symbols(max_symbols)
        W = operator.index(W)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width must be in [1, %d], got %r" % (BEAM_MAX_W, W))
        V = transducer.joint.joint[2].weight.shape[0]
        fusion = check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map)
        graph = check_context(context, V, blank)
        enc, dec, joint = transducer.encoder, transducer.decoder, transducer.joint.joint
        S, n, T = self._check_shape(enc, n_streams, frames_per_chunk, frontend, samples_per_chunk)
        P = operator.index(max_pending)
        if P < T * K:
            raise ValueError("max_pending (%d) must be at least the encoder frames per chunk times max_symbols (%d x %d):"
                             " a chunk can add that many tokens to a hypothesis" % (P, T, K))
        f32, i32 = torch.float32, torch.int32
        R, LS, TK = S * W, P + 3, T * K
        self.S, self.n, self.W, self.R, self.merge, self.blank, self.max_ctas, self.max_pending, self.max_symbols = \
            S, n, W, R, merge, blank, max_ctas, P, K
        prog = []
        E = self._build_encoder(prog, transducer, enc, S, n, T)
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=self.dev)
        Ld, Hd = dec.lstm.num_layers, dec.lstm.hidden_size
        D = dec.proj.weight.shape[0]
        J = joint[0].weight.shape[0]
        self.lm = fusion is not None
        lm_sel, lm_step = lm_fusion(self, fusion, R) if self.lm else ({}, None)
        # per parity: predictor state, its output, {suffix length, hash lo, hash hi, tokens since the last commit} per
        # row and the LM state
        beam_state(self, R, Ld, Hd, D, LS, context=graph is not None)
        self.dec_htmp, self.hidden, self.logits = z(Ld, R, Hd), z(R, J), z(R, V)
        self.tok, self.src, self.logp = z(R, dtype=i32), z(R, dtype=i32), z(R)
        self.frames = torch.full((S,), T, dtype=i32, device=self.dev)      # a stream never freezes
        beam_history(self, S, TK, W)                          # hist_live's last column: the live count between launches
        self._commit_buffers()
        self._joint = (joint[0].weight, joint[0].bias, joint[2].weight, joint[2].bias)
        prime = []
        _dec_phases(prime, dec, R, self.dec_h[0], self.dec_c[0], self.dec_htmp, self.dec_x[0], self.tok, blank,
                    masked=False)
        if self.lm:
            self._lm_logits_tmp = z(R, self.lm_logits.shape[1])           # the chunk end gathers the LM logits
            lm_step(prime, self.lm_h[0], self.lm_c[0], masked=False)
        sel = dict(type=PH_BEAM_SELECT, S=S, N=V, aux=W, aux2=blank,
                   flags=F_STREAM | (F_MERGE if merge else 0) | (F_LM if self.lm else 0), K1=LS, x1=_ptr(self.logits),
                   ldx1=V, y=_ptr(self.logp), tok_in=_ptr(self.frames), tok_out=_ptr(self.tok), src=_ptr(self.src),
                   hist=_ptr(self.hist), hist_ld=TK, **lm_sel)
        self._context(graph, sel)
        for t in range(T):
            beam_frame(prog, self, dec, t, _ptr(self.enc_out, t * E), T * E, sel, lm_step)
        self._prime, self.n_prime_phases = _upload(prime, self.dev), len(prime)
        self._commit_programs(prog, K > 1 or T % 2 == 0)     # where the frames left the state
        self._finish(prog, state)

    def _chunk_end(self, pr, in_parity0, flush):
        st, R = self._st, self.R
        Ld, Hd, D, LS = st[0].shape[0] // 2, st[0].shape[2], self.dec_x[0].shape[1], self.seqs[0].shape[1]
        if in_parity0:
            pr.append(EbPhase(type=PH_COPY, S=2 * Ld * R, N=Hd, x1=_ptr(st[0]), y=_ptr(st[1])))
            pr.append(EbPhase(type=PH_COPY, S=R, N=D, x1=_ptr(self.dec_x[0]), y=_ptr(self.dec_x[1])))
            pr.append(EbPhase(type=PH_COPY, S=R, N=LS, x1=_ptr(self.seqs[0]), y=_ptr(self.seqs[1])))
            if self.lm:
                pr.append(EbPhase(type=PH_COPY, S=self._lst[0].shape[0] * R, N=self._lst[0].shape[2],
                                  x1=_ptr(self._lst[0]), y=_ptr(self._lst[1])))
            if self.ctx_state is not None:
                pr.append(EbPhase(type=PH_COPY, S=1, N=R, x1=_ptr(self.ctx_state[0]), y=_ptr(self.ctx_state[1])))
        if self.lm:
            ntok = self.lm_logits.shape[1]
            pr.append(EbPhase(type=PH_COPY, S=R, N=ntok, x1=_ptr(self.lm_logits), y=_ptr(self._lm_logits_tmp)))
        pr.append(self._commit_phase(flush, self.n_out * self.max_symbols))
        pr.append(EbPhase(type=PH_GATHER, S=R, N=Hd, aux=2 * Ld, x1=_ptr(st[1]), y=_ptr(st[0]), K2=D,
                          x2=_ptr(self.dec_x[1]), y2=_ptr(self.dec_x[0]), src=_ptr(self.src)))
        if self.lm:
            pr.append(EbPhase(type=PH_GATHER, S=R, N=self._lst[0].shape[2], aux=self._lst[0].shape[0],
                              x1=_ptr(self._lst[1]), y=_ptr(self._lst[0]), K2=ntok, x2=_ptr(self._lm_logits_tmp),
                              y2=_ptr(self.lm_logits), src=_ptr(self.src)))

    def _state_views(self):
        v = dict(super()._state_views(), dec_state=self._st[0], dec_x=self.dec_x[0], logp=self.logp, seqs=self.seqs[0],
                 live=self.hist_live[:, -1])
        if self.lm:
            v.update(lm_state=self._lst[0], lm_logits=self.lm_logits)
        if self.ctx_state is not None:
            v.update(ctx_state=self.ctx_state[0])
        return v

    @torch.no_grad()
    def reset(self):
        """Every stream starts a new utterance: zero encoder state, one live slot of log p 0 with the empty sequence
        (at the phrase automaton's root with contextual biasing), predictor primed with <bos> and the LM with lm_bos
        from zeros."""
        for t in (self.enc_h, self.enc_c):
            if t is not None:
                t.zero_()
        beam_reset(self)
        self._reset_commits()
        self._run(self._prime, self.n_prime_phases)


class GRUStreamEngine(StreamEngine):
    """StreamEngine for a transducer with a GRU encoder (``Transducer(module_type='GRU')``, ResLayerNormGRU): the same
    arguments, ``step`` / ``reset`` / ``state`` / ``load_state`` / ``fingerprint`` / ``n_out`` and ``max_symbols``
    rounds with the ``<unk>`` rule.  The chunk program is encoder_phases' GRU encoder (per layer n GRU cell steps from
    the carried h) followed by StreamEngine's frames; the predictor stays an LSTM.  Every program runs through
    eb_decode_run_gru_rnnt, the decode kernel's instantiation with both cell phases.  The carried encoder state is
    ``enc_h`` alone: the state of an LSTM-encoder engine does not load here, nor this one's there.

    Per stream the ids are those of Transducer.greedy_decode (with the <unk> rule) on the concatenated chunks: every
    layer is a unidirectional GRU and the time reduction pairs frames inside a chunk of even length, so the chunks with
    h carried give the offline encoder output.  The matrix products are fp32-accurate (3xTF32)."""
    GRU = True


class GRUStreamBeamEngine(StreamBeamEngine):
    """StreamBeamEngine for a transducer with a GRU encoder: the same signature and contract (W, merge, the LM fusion
    arguments, max_pending and the forced collapse, max_symbols, ``step`` / ``flush`` / ``reset`` / ``state`` /
    ``load_state`` with the re-bound, ``context``).  The chunk program is encoder_phases' GRU encoder followed by
    StreamBeamEngine's beam frames and chunk end; every program (chunk, prime, flush, re-bound) runs through
    eb_decode_run_gru_rnnt.  The state carries ``enc_h`` and no ``enc_c``, so the state of an LSTM-encoder engine does
    not load here, nor this one's there."""
    GRU = True


def lm_cache_key(fusion):
    """What a phase program built for the fusion arguments ``fusion`` (check_lm_args' result, or None) depends on: the
    LM tensors' identity and version (a state_dict on another device is copied into the engine) and the scalars."""
    if fusion is None:
        return None
    lsd, lw, lb, bos, tmap = fusion
    return (tuple((k, v.data_ptr(), v.device, v.dtype, v._version) for k, v in sorted(lsd.items())), lw, lb, bos,
            tuple(tmap.tolist()))


class CTCBeamEngine:
    """Device-side CTC prefix beam search (Hannun et al., 2014) over log-probs [B, T', V], optionally with shallow
    fusion of the reference's LSTM language model, in ONE cooperative kernel launch (decode.cu, CTC_BEAM, which states
    the rule).  Row r = b*W + j holds slot j of utterance b; each slot carries a prefix with log P(prefix, path ends in
    blank) ``pb``, log P(prefix, ends in a non-blank) ``pnb`` and its accumulated fusion term ``f``.

    Without an LM nothing runs between frames but the selection, so the program is ``frames_per_phase`` frames per
    CTC_BEAM phase (0: all T' frames in one phase, no grid barrier per frame) and BEAM_FINAL.  With an LM every frame
    is one CTC_BEAM phase, the GATHER of the LM state by parent and the masked LM step and output Linear
    (predictor_phases resting on -1, as BeamEngine's LM), after a priming step on ``lm_bos``; frames_per_phase must
    then be 0 or 1.  BEAM_FINAL picks the best live slot by (pb (+) pnb) + f, lowest slot on ties, and walks the
    history, where a stay is recorded as blank.

    With ``context`` (a ContextGraph over V tokens) each slot carries its phrase-automaton state (``ctx_state``
    [2, R], parity t & 1 as ``state``), an extension by c adds the automaton's increment to f', and BEAM_FINAL ranks
    by (pb (+) pnb) + f minus the pending bonus of the slot's state.  An empty graph builds the program without it.

    With ``ngram`` (an NgramLM over V tokens) each slot carries its n-gram state (``ng_state`` [2, R], parity t & 1,
    the model's start state after ``run``'s reset), an extension by c adds the length bonus (without an LM) and
    ngram_weight * g(state, c) after the LM term, f' = ((f + LM term) + w g) + delta, and BEAM_FINAL ranks by
    ((pb (+) pnb) + f + w e(state)) - pending."""

    def __init__(self, batch, t_out, V, W, blank=0, lm=None, lm_weight=0.0, length_bonus=0.0, lm_bos=1,
                 lm_token_map=None, max_ctas=0, device=None, frames_per_phase=0, nbest=0, context=None, ngram=None,
                 ngram_weight=0.0):
        B, T, V, W, blank = (operator.index(v) for v in (batch, t_out, V, W, blank))
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        N = _engine_nbest(nbest, W)
        if B < 1 or T < 1 or V < 1:
            raise ValueError("batch, t_out and V must be positive, got %d, %d, %d" % (B, T, V))
        if not 0 <= blank < V:
            raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
        if W * V >= 2 ** 31:
            raise ValueError("beam width x vocabulary must stay below 2^31 (flat candidate index), got %d x %d" % (W, V))
        model = check_ngram(ngram, V, blank)
        ng_w = check_ngram_weight(model, ngram_weight)
        fusion = check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map, ngram=model is not None)
        graph = check_context(context, V, blank)
        n = operator.index(frames_per_phase)
        if n < 0 or (fusion is not None and n > 1):
            raise ValueError("frames_per_phase must be >= 0 (0: all), and 0 or 1 with an lm; got %d" % n)
        n = 1 if fusion is not None else (n or T)
        self.dev = torch.device("cuda") if device is None else torch.device(device)
        if self.dev.type != "cuda":
            raise RuntimeError("CTCBeamEngine runs on a CUDA device")
        f32, i32 = torch.float32, torch.int32
        R, LS = B * W, T + 5
        self.B, self.T, self.V, self.W, self.R, self.blank, self.max_ctas = B, T, V, W, R, blank, max_ctas
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=self.dev)
        self.lp, self.frames = z(B, T, V), z(B, dtype=i32)
        self.state = z(2, 3, R)                      # per parity: pb | pnb | f
        self.seqs = z(2, R, LS, dtype=i32)           # per parity: {len, hash lo / hi, parent hash lo / hi, tokens}
        self.score, self.src = z(R), z(R, dtype=i32)
        beam_history(self, B, T, W)
        final_outputs(self, B, N, T)
        self.lm = fusion is not None
        self._keep = []
        lm_sel, lm_step = lm_fusion(self, fusion, R) if self.lm else ({}, None)
        prog = []
        sel = dict(type=PH_CTC_BEAM, S=B, N=V, aux=W, aux2=blank, K1=LS, flags=F_LM if self.lm else 0,
                   x1=_ptr(self.lp), tok_in=_ptr(self.frames), c=_ptr(self.state), seq_out=_ptr(self.seqs),
                   y=_ptr(self.score), src=_ptr(self.src), hist=_ptr(self.hist), hist_ld=T, **lm_sel)
        # per parity: the context automaton state and the n-gram state of each slot
        self.ctx_state = z(2, R, dtype=i32) if graph is not None else None
        self.ng_state = z(2, R, dtype=i32) if model is not None else None
        cf = fusion_fields(self, sel, graph, self.ctx_state, model, self.ng_state, ng_w, length_bonus, R, V)
        ctx = None if cf is None else (cf, T & 1)        # frozen frames carry the states, so frame T-1 wrote them
        if self.lm:
            Ll, _, Hl = self.lm_htmp.shape
            self.lm_state = z(2, 2 * Ll, R, Hl)      # per parity: h of every layer, then c
            lm_step(prog, self.lm_state[0, :Ll], self.lm_state[0, Ll:], masked=False)   # prime with lm_bos from zeros
        for t0 in range(0, T, n):
            prog.append(EbPhase(hist_col=t0, ldw1=min(n, T - t0), **sel))
            if self.lm:                              # survivors inherit their parent's LM state, extensions step it
                p, q = t0 & 1, 1 - (t0 & 1)
                prog.append(EbPhase(type=PH_GATHER, S=R, N=Hl, aux=2 * Ll, x1=_ptr(self.lm_state[p]),
                                    y=_ptr(self.lm_state[q]), src=_ptr(self.src)))
                lm_step(prog, self.lm_state[q, :Ll], self.lm_state[q, Ll:], masked=True)
        prog.append(final_phase(self, W, self.score, 1, ctx))
        self.nphase = len(prog)
        self._prog = _upload(prog, self.dev)
        self._bar = torch.zeros(64, dtype=torch.int32, device=self.dev)

    @torch.no_grad()
    def run(self, log_probs, lengths):
        """log_probs [B, T', V] fp32 on the device (any strides), lengths int32 [B] on the device (frames each utterance
        decodes, clamped to [0, T']) -> (ids int32 [B, T']: the best prefix right-aligned, -1 before it; -score [B],
        the negated (pb (+) pnb) + f of that prefix).  Both stay on the device.  With ``nbest`` it returns
        ``nbest_out`` (nbest_lists reads it, L = T'), rank 0 of which holds those same values."""
        self.lp.copy_(log_probs)
        self.frames.copy_(lengths.clamp(0, self.T))
        self.state.zero_()
        self.state[0, :2].fill_(float("-inf"))
        self.state[0, 0].view(self.B, self.W)[:, 0] = 0.0        # the empty prefix: pb = 0, pnb = -inf, f = 0
        self.score.fill_(float("-inf"))
        self.score.view(self.B, self.W)[:, 0] = 0.0
        self.seqs[0].zero_()
        if self.ctx_state is not None:
            self.ctx_state[0].zero_()
        if self.ng_state is not None:
            self.ng_state[0].fill_(self.ng_start)
        if self.lm:
            self.lm_state[0].zero_()
            self.lm_tok.fill_(self.lm_bos)
        _launch("eb_decode_run_ctc", self._prog, self.nphase, self._bar, self.max_ctas)
        return self.nbest_out if self.nbest else (self.ids, self.nlogp)

    def hypotheses(self, b):
        """The live slots of utterance b after ``run``, in slot order: [(prefix tuple, pb, pnb, f)] on the host."""
        n = int(self.frames[b])
        live = int(self.hist_live[b, -1])
        st = self.state[n & 1, :, b * self.W:b * self.W + live].cpu()
        rows = self.seqs[n & 1, b * self.W:b * self.W + live].cpu()
        return [(tuple(int(x) for x in rows[j, 5:5 + int(rows[j, 0])]), float(st[0, j]), float(st[1, j]),
                 float(st[2, j])) for j in range(live)]


class CTCStreamEngine(_ChunkEngine):
    """Streaming greedy CTC decoding of a ``CTCEncoder`` (rnnt/models.py:272-310): S streams, one persistent kernel
    launch per chunk (eb_decode_run_ctc_stream).  The chunk program is encoder_phases' GRU encoder (LayerNorm, per layer
    n GRU cell steps from the carried h, residual LayerNorm, time reduction), the projection, the ``tovocab`` Linear
    over the chunk's n_out output frames, and CTC_EMIT.

    Per stream the emitted ids are those of ``CTCEncoder.greedy_decode`` on the concatenated chunks (every layer is a
    unidirectional GRU, LayerNorm works per frame and the time reduction pairs frames inside a chunk of even length, so
    streaming the chunks with h carried gives the offline log-probs): per frame the argmax of the log-probs (NaN first,
    ties to the lowest id), a frame equal to the previous frame's argmax dropped, including across a chunk boundary, and
    blanks dropped.  ``score()`` keeps greedy_decode's quirk: the sum of the WHOLE log-prob rows of the kept frames.
    The matrix products are fp32-accurate (3xTF32) whatever the model's precision setting.

    The carried state is ``enc_h`` [L, S, H], the previous frame's argmax ``prev`` [S] (-1 after ``reset``: it matches
    no token) and the running score ``score`` (fp64 on the device).  ``state()`` / ``load_state()`` move it to an engine
    rebuilt for another chunk length or for re-homed weights (``fingerprint``)."""
    GRU = True
    RUN = "eb_decode_run_ctc_stream"

    def __init__(self, ctc_model, n_streams, frames_per_chunk, blank=0, max_ctas=0, state=None, frontend=None,
                 samples_per_chunk=None):
        from .rnnt.models import CTCEncoder
        if not isinstance(ctc_model, CTCEncoder):
            raise TypeError("CTCStreamEngine streams a CTCEncoder, got %s" % type(ctc_model).__name__)
        enc, lin = ctc_model.model, ctc_model.tovocab[0]
        S, n, T = self._check_shape(enc, n_streams, frames_per_chunk, frontend, samples_per_chunk)
        V, blank = lin.weight.shape[0], operator.index(blank)
        if not 0 <= blank < V:
            raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
        i32 = torch.int32
        self.S, self.n, self.V, self.blank, self.max_ctas = S, n, V, blank, max_ctas
        prog = []
        E = self._build_encoder(prog, ctc_model, enc, S, n, T)
        assert lin.weight.shape[1] == E
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=self.dev)
        self.logits, self.logprobs = z(S * T, V), z(S * T, V)
        self.argmax = z(S, T, dtype=i32)                        # every frame's argmax (CTC_EMIT's seq_out)
        self.prev, self._score = z(S, dtype=i32), z(S, dtype=torch.float64)
        self._out = z(S * T + S, dtype=i32)                    # emitted ids [S, n_out] | counts [S]
        self._host = torch.zeros(self._out.shape, dtype=i32).pin_memory()
        prog.append(EbPhase(type=PH_LINEAR, S=S * T, N=V, K1=E, x1=_ptr(self.enc_out), ldx1=E, w1=_ptr(lin.weight),
                            ldw1=E, b1=_ptr(lin.bias), y=_ptr(self.logits), ldy=V))
        prog.append(EbPhase(type=PH_CTC_EMIT, S=S, N=V, aux=T, aux2=blank, x1=_ptr(self.logits), ldx1=V,
                            y=_ptr(self.logprobs), ldy=V, tok_out=_ptr(self.prev), hist=_ptr(self._out), hist_ld=T,
                            tok_out2=_ptr(self._out, S * T), y2=_ptr(self._score), seq_out=_ptr(self.argmax)))
        self._finish(prog, state)

    def _state_views(self):
        return dict(super()._state_views(), prev=self.prev, score=self._score)

    @torch.no_grad()
    def reset(self):
        """Every stream starts a new utterance: zero encoder state, no previous frame, score 0."""
        self.enc_h.zero_()
        self.prev.fill_(-1)
        self._score.zero_()

    def score(self):
        """The running score of every stream [S] (fp64, on the device): the sum of the whole log-prob rows of every
        frame kept since ``reset``, what ``CTCEncoder.greedy_decode`` returns negated."""
        return self._score

    @torch.no_grad()
    def step(self, chunk):
        """chunk [S, n, F] log-mel frames (device or pinned host), or with a front end fp32 audio [S, L] on the device,
        -> (ids int32 [S, n_out], counts int32 [S]) on the host: row s holds in its first counts[s] entries the ids stream s emitted in this chunk.  One device-to-host
        copy per chunk."""
        self._load(chunk)
        self._run(self._chunk, self.n_chunk_phases)
        ids, counts, _ = self._fetch(self.n_out)
        return ids, counts


class CTCStreamBeamEngine(_CommitEngine):
    """Streaming CTC prefix beam search of a ``CTCEncoder``, optionally with shallow fusion of the reference's LSTM
    language model: S streams of W prefixes each, carried from one chunk to the next, one persistent kernel launch per
    chunk (eb_decode_run_ctc_stream_beam).  Row r = s*W + slot; each slot carries its prefix with log P(prefix, ends in
    blank) ``pb``, log P(prefix, ends in a non-blank) ``pnb`` and its accumulated fusion term ``f`` (``beam`` [2][3][R],
    by parity).

    The chunk program is CTCStreamEngine's encoder and ``tovocab`` Linear, CTC_EMIT for the log-probs (``logprobs``
    [S*n_out, V]; its greedy outputs go to scratch), then CTCBeamEngine's search in streaming mode: without an LM one
    CTC_BEAM phase over the chunk's n_out frames, with an LM per frame CTC_BEAM, the GATHER of the LM state by parent and
    the masked LM step.  So how the audio is cut into chunks does not change which prefixes survive.

    After the chunk's last frame BEAM_COMMIT commits each stream's longest common prefix of its live prefixes, as
    StreamBeamEngine does: each slot stores only its uncommitted suffix, at most ``max_pending`` tokens, while its hash
    and parent hash describe the whole prefix.  When a suffix would hold more than ``max_pending - n_out`` tokens the
    beam collapses to its best slot (highest (pb (+) pnb) + f, lowest slot on ties), whose pb | pnb | f and LM state
    move to slot 0.  Each stream keeps its last committed token ``last`` [S] (-1 after ``reset``): a slot whose stored
    suffix is empty takes it as its last token, so a token held across a commit is not emitted twice.  ``flush()``,
    ``state()`` / ``load_state()`` (with the re-bound) and ``n_collapses`` are StreamBeamEngine's, and so is
    ``context``: each slot carries its phrase-automaton state (``ctx_state`` [2, R]) across chunks, an extension adds
    the automaton's increment to f', and collapses and ``flush`` use (pb (+) pnb) + f - pending[state], so the ids of
    the chunks plus ``flush`` are ctc.beam_search(context=...)'s on the concatenated log-probs."""
    GRU = True
    RUN = "eb_decode_run_ctc_stream_beam"

    def __init__(self, ctc_model, n_streams, frames_per_chunk, W, *, lm=None, lm_weight=0.0, length_bonus=0.0,
                 lm_bos=1, lm_token_map=None, max_pending=64, blank=0, max_ctas=0, state=None, frontend=None,
                 samples_per_chunk=None, context=None):
        from .rnnt.models import CTCEncoder
        if not isinstance(ctc_model, CTCEncoder):
            raise TypeError("CTCStreamBeamEngine streams a CTCEncoder, got %s" % type(ctc_model).__name__)
        enc, lin = ctc_model.model, ctc_model.tovocab[0]
        V, W, blank = lin.weight.shape[0], operator.index(W), operator.index(blank)
        if not 1 <= W <= BEAM_MAX_W:
            raise ValueError("beam width must be in [1, %d], got %d" % (BEAM_MAX_W, W))
        if W * V >= 2 ** 31:
            raise ValueError("beam width x vocabulary must stay below 2^31 (flat candidate index), got %d x %d" % (W, V))
        if not 0 <= blank < V:
            raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
        fusion = check_lm_args(lm, V, lm_weight, length_bonus, lm_bos, lm_token_map)
        graph = check_context(context, V, blank)
        S, n, T = self._check_shape(enc, n_streams, frames_per_chunk, frontend, samples_per_chunk)
        P = operator.index(max_pending)
        if P < T:
            raise ValueError("max_pending (%d) must be at least the encoder frames per chunk (%d): a chunk can add that "
                             "many tokens to a prefix" % (P, T))
        f32, i32 = torch.float32, torch.int32
        R, LS = S * W, P + 5
        self.S, self.n, self.V, self.W, self.R, self.blank, self.max_ctas, self.max_pending = \
            S, n, V, W, R, blank, max_ctas, P
        prog = []
        E = self._build_encoder(prog, ctc_model, enc, S, n, T)
        assert lin.weight.shape[1] == E
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=self.dev)
        self.logits, self.logprobs = z(S * T, V), z(S * T, V)
        self._emit = (z(S, dtype=i32), z(S, T, dtype=i32), z(S, dtype=i32), z(S, dtype=torch.float64))
        self.beam = z(2, 3, R)                       # per parity: pb | pnb | f
        self.seqs = z(2, R, LS, dtype=i32)           # per parity: {len, hash lo / hi, parent hash lo / hi, suffix}
        self.logp, self.src = z(R), z(R, dtype=i32)  # logp: the ranking value (pb (+) pnb) + f
        self.last = z(S, dtype=i32)
        self.frames = torch.full((S,), T, dtype=i32, device=self.dev)      # a stream never freezes
        beam_history(self, S, T, W)                  # hist_live's last column: the live count between launches
        self._commit_buffers()
        self.lm = fusion is not None
        lm_sel, lm_step = lm_fusion(self, fusion, R) if self.lm else ({}, None)
        prog.append(EbPhase(type=PH_LINEAR, S=S * T, N=V, K1=E, x1=_ptr(self.enc_out), ldx1=E, w1=_ptr(lin.weight),
                            ldw1=E, b1=_ptr(lin.bias), y=_ptr(self.logits), ldy=V))
        prev, ids, counts, score = self._emit
        prog.append(EbPhase(type=PH_CTC_EMIT, S=S, N=V, aux=T, aux2=blank, x1=_ptr(self.logits), ldx1=V,
                            y=_ptr(self.logprobs), ldy=V, tok_out=_ptr(prev), hist=_ptr(ids), hist_ld=T,
                            tok_out2=_ptr(counts), y2=_ptr(score)))
        sel = dict(type=PH_CTC_BEAM, S=S, N=V, aux=W, aux2=blank, K1=LS, flags=F_STREAM | (F_LM if self.lm else 0),
                   x1=_ptr(self.logprobs), tok_in=_ptr(self.frames), c=_ptr(self.beam), seq_out=_ptr(self.seqs),
                   y=_ptr(self.logp), src=_ptr(self.src), hist=_ptr(self.hist), hist_ld=T, y2=_ptr(self.last), **lm_sel)
        self.ctx_state = z(2, R, dtype=i32) if graph is not None else None   # per parity: each slot's automaton state
        self._context(graph, sel)
        prime = []
        if self.lm:
            Ll, _, Hl = self.lm_htmp.shape
            self.lm_state = z(2, 2 * Ll, R, Hl)      # per parity: h of every layer, then c
            self._lm_logits_tmp = z(R, self.lm_logits.shape[1])
            lm_step(prime, self.lm_state[0, :Ll], self.lm_state[0, Ll:], masked=False)   # lm_bos from zeros
            for t in range(T):
                prog.append(EbPhase(hist_col=t, ldw1=1, **sel))
                p, q = t & 1, 1 - (t & 1)
                prog.append(EbPhase(type=PH_GATHER, S=R, N=Hl, aux=2 * Ll, x1=_ptr(self.lm_state[p]),
                                    y=_ptr(self.lm_state[q]), src=_ptr(self.src)))
                lm_step(prog, self.lm_state[q, :Ll], self.lm_state[q, Ll:], masked=True)
        else:
            prog.append(EbPhase(hist_col=0, ldw1=T, **sel))
        self._prime, self.n_prime_phases = (_upload(prime, self.dev), len(prime)) if prime else (None, 0)
        self._commit_programs(prog, T % 2 == 0)      # where the frames left the state
        self._finish(prog, state)

    def _chunk_end(self, pr, in_parity0, flush):
        R, LS = self.R, self.seqs.shape[2]
        if in_parity0:
            pr.append(EbPhase(type=PH_COPY, S=3, N=R, x1=_ptr(self.beam[0]), y=_ptr(self.beam[1])))
            pr.append(EbPhase(type=PH_COPY, S=R, N=LS, x1=_ptr(self.seqs[0]), y=_ptr(self.seqs[1])))
            if self.lm:
                pr.append(EbPhase(type=PH_COPY, S=self.lm_state.shape[1] * R, N=self.lm_state.shape[3],
                                  x1=_ptr(self.lm_state[0]), y=_ptr(self.lm_state[1])))
            if self.ctx_state is not None:
                pr.append(EbPhase(type=PH_COPY, S=1, N=R, x1=_ptr(self.ctx_state[0]), y=_ptr(self.ctx_state[1])))
        if self.lm:
            ntok = self.lm_logits.shape[1]
            pr.append(EbPhase(type=PH_COPY, S=R, N=ntok, x1=_ptr(self.lm_logits), y=_ptr(self._lm_logits_tmp)))
        pr.append(self._commit_phase(flush, self.n_out, K2=CTC_SEQ_HEAD, y2=_ptr(self.last)))
        pr.append(EbPhase(type=PH_GATHER, S=R, N=1, aux=3, x1=_ptr(self.beam[1]), y=_ptr(self.beam[0]),
                          src=_ptr(self.src)))
        if self.lm:
            pr.append(EbPhase(type=PH_GATHER, S=R, N=self.lm_state.shape[3], aux=self.lm_state.shape[1],
                              x1=_ptr(self.lm_state[1]), y=_ptr(self.lm_state[0]), K2=ntok, x2=_ptr(self._lm_logits_tmp),
                              y2=_ptr(self.lm_logits), src=_ptr(self.src)))

    def _state_views(self):
        v = dict(super()._state_views(), beam=self.beam[0], logp=self.logp, seqs=self.seqs[0],
                 live=self.hist_live[:, -1], last=self.last)
        if self.lm:
            v.update(lm_state=self.lm_state[0], lm_logits=self.lm_logits)
        if self.ctx_state is not None:
            v.update(ctx_state=self.ctx_state[0])
        return v

    @torch.no_grad()
    def reset(self):
        """Every stream starts a new utterance: zero encoder state, one live slot holding the empty prefix (pb = 0,
        pnb = -inf, f = 0) at the phrase automaton's root with contextual biasing, no committed token (last = -1), and
        the LM primed with lm_bos from zeros."""
        S, W = self.S, self.W
        self.enc_h.zero_()
        if self.ctx_state is not None:
            self.ctx_state[0].zero_()
        self.beam[0].zero_()
        self.beam[0, :2].fill_(float("-inf"))
        self.beam[0, 0].view(S, W)[:, 0] = 0.0
        self.logp.fill_(float("-inf"))
        self.logp.view(S, W)[:, 0] = 0.0
        self.seqs[0].zero_()
        self.last.fill_(-1)
        self._reset_commits()
        if self.lm:
            self.lm_state[0].zero_()
            self.lm_tok.fill_(self.lm_bos)
            self._run(self._prime, self.n_prime_phases)

    def hypotheses(self, s):
        """The live slots of stream s between chunks, in slot order: [(stored suffix tuple, pb, pnb, f, hash, parent
        hash)] on the host; the committed tokens precede every suffix."""
        W, live = self.W, int(self.hist_live[s, -1])
        st = self.beam[0, :, s * W:s * W + live].cpu()
        rows = self.seqs[0, s * W:s * W + live].cpu()
        u = lambda lo, hi: (int(lo) & 0xffffffff) | ((int(hi) & 0xffffffff) << 32)
        return [(tuple(int(x) for x in rows[j, CTC_SEQ_HEAD:CTC_SEQ_HEAD + int(rows[j, 0])]), float(st[0, j]),
                 float(st[1, j]), float(st[2, j]), u(rows[j, 1], rows[j, 2]), u(rows[j, 3], rows[j, 4]))
                for j in range(live)]
