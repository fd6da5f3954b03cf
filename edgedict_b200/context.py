"""Contextual biasing: a phrase list compiled to a token automaton that the device beam searches score inside their
launch (``Transducer.beam_search(context=...)``, ``CTCEncoder.beam_search`` and ``ctc.beam_search``).

``ContextGraph(phrases, vocab_size, boost)`` builds, on the host, the deterministic automaton of the phrases as dense
tables.  Its states are the trie nodes of the phrases (their distinct prefixes, the root being the empty one); |s| is the
length of node s and P(s) = boost * |s| its pending bonus.  Appending a non-blank token k to a hypothesis in state s:

- u is the longest suffix of string(s) + [k] that is a trie node (the root if none is): the Aho-Corasick goto;
- if a suffix of string(u) is a whole phrase, the longest one, c, completes: boost * |c| is banked and the next state is
  the root (a phrase that is a prefix of a longer one therefore completes first and resets the state);
- otherwise the next state is u;
- the increment added to the hypothesis' value is delta(s, k) = (completes ? boost * |c| : boost * |u|) - P(s).

Blank (and a CTC stay, and a closed multi-symbol slot's stay) leaves the state alone and adds nothing, so during the
search a value includes banked + P(state); the final ranking and the returned scores subtract P(state), so a phrase
that is only partly matched earns nothing.  The state is a function of the token sequence alone, so merging equal
sequences stays exact.
"""
import hashlib
import math
import numbers

import numpy as np
import torch

MAX_TABLE = 1 << 24          # n_states * V entries at most: 128 MB of next (int32) + delta (fp32) tables


class ContextGraph:
    """The automaton of ``phrases`` (an iterable of non-empty sequences of token ids in [0, vocab_size), none equal to
    ``blank``; duplicates collapse) with one ``boost`` >= 0 per token.  Tables, numpy on the host:

    - ``next`` int32 [n_states, V]: the state after token k (the row of blank is the identity, never read);
    - ``delta`` float32 [n_states, V]: the increment of that step (0 for blank);
    - ``pending`` float32 [n_states]: P(s) = boost * |s|.

    State 0 is the root and ``nodes[s]`` the token string of state s.  ``fingerprint`` identifies the content (phrases, V, blank, boost); ``to(device)`` uploads
    the tables once per device.  Raises TypeError / ValueError for a malformed argument and for n_states * V above
    2^24 (MAX_TABLE), before any device work.  An empty phrase list is legal: it gives the search without context."""

    def __init__(self, phrases, vocab_size, boost, blank=0):
        if isinstance(vocab_size, bool) or not isinstance(vocab_size, numbers.Integral):
            raise TypeError("vocab_size must be an integer, got %r" % (vocab_size,))
        V = int(vocab_size)
        if V < 1:
            raise ValueError("vocab_size must be positive, got %d" % V)
        if isinstance(blank, bool) or not isinstance(blank, numbers.Integral):
            raise TypeError("blank must be an integer, got %r" % (blank,))
        blank = int(blank)
        if not 0 <= blank < V:
            raise ValueError("blank must lie in [0, %d), got %d" % (V, blank))
        if isinstance(boost, bool) or not isinstance(boost, numbers.Real):
            raise TypeError("boost must be a real number, got %r" % (boost,))
        beta = float(boost)
        if not math.isfinite(beta) or beta < 0:
            raise ValueError("boost must be finite and >= 0, got %r" % (boost,))
        if isinstance(phrases, (str, bytes)):
            raise TypeError("phrases must be an iterable of token-id sequences")
        uniq = set()
        for ph in phrases:
            if isinstance(ph, (str, bytes)):
                raise TypeError("a phrase must be a sequence of token ids, got %r" % (ph,))
            try:
                toks = list(ph)
            except TypeError:
                raise TypeError("a phrase must be a sequence of token ids, got %r" % (ph,)) from None
            ids = []
            for k in toks:
                if isinstance(k, (np.integer, torch.Tensor)) and getattr(k, "ndim", 0) == 0:
                    k = int(k)
                if isinstance(k, bool) or not isinstance(k, numbers.Integral):
                    raise TypeError("token ids must be integers, got %r" % (k,))
                ids.append(int(k))
            if not ids:
                raise ValueError("a phrase must not be empty")
            bad = [k for k in ids if not 0 <= k < V or k == blank]
            if bad:
                raise ValueError("phrase %s: token %d is blank or outside [0, %d)" % (ids, bad[0], V))
            uniq.add(tuple(ids))
        self.phrases = sorted(uniq)
        self.vocab_size, self.blank, self.boost = V, blank, beta
        # trie: node 0 the root, children by token, nodes numbered in insertion order
        child = [{}]
        depth = [0]
        for ph in self.phrases:
            s = 0
            for k in ph:
                if k not in child[s]:
                    child[s][k] = len(child)
                    child.append({})
                    depth.append(depth[s] + 1)
                s = child[s][k]
        n = len(child)
        self.nodes = [()] * n                                      # the token string of every state
        for s in sorted(range(n), key=lambda s: depth[s]):
            for k, c in child[s].items():
                self.nodes[c] = self.nodes[s] + (k,)
        if n * V > MAX_TABLE:
            raise ValueError("the context automaton has %d states x %d tokens = %d table entries, above the cap of 2^24 "
                             "(128 MB of tables); use fewer or shorter phrases" % (n, V, n * V))
        order = sorted(range(n), key=lambda s: depth[s])            # parents before children
        is_phrase = np.zeros(n, dtype=bool)
        for ph in self.phrases:
            s = 0
            for k in ph:
                s = child[s][k]
            is_phrase[s] = True
        # goto[s, k] = longest suffix of string(s) + [k] that is a node; fail[s] = longest proper suffix node of s;
        # out[s] = length of the longest suffix of string(s) that is a whole phrase (0: none)
        goto = np.zeros((n, V), dtype=np.int32)
        fail = np.zeros(n, dtype=np.int64)
        out = np.zeros(n, dtype=np.int64)
        dep = np.asarray(depth, dtype=np.int64)
        for s in order:
            if s == 0:
                row = np.zeros(V, dtype=np.int32)
            else:
                row = goto[fail[s]].copy()
                out[s] = dep[s] if is_phrase[s] else out[fail[s]]
            for k, c in child[s].items():
                fail[c] = row[k] if s != 0 else 0
                row[k] = c
            goto[s] = row
        P = (np.float32(beta) * dep.astype(np.float32)).astype(np.float32)
        done = out[goto]                                            # [n, V]: phrase completed by the step
        gain = np.where(done > 0, np.float32(beta) * done.astype(np.float32), P[goto]).astype(np.float32)
        nxt = np.where(done > 0, 0, goto)
        delta = (gain - P[:, None]).astype(np.float32)
        nxt[:, blank] = np.arange(n)
        delta[:, blank] = 0.0
        self.next = np.ascontiguousarray(nxt, dtype=np.int32)
        self.delta = np.ascontiguousarray(delta, dtype=np.float32)
        self.pending = P
        self.n_states = n
        h = hashlib.sha1()
        h.update(np.asarray([V, blank], dtype=np.int64).tobytes())
        h.update(np.float64(beta).tobytes())
        for ph in self.phrases:
            h.update(np.asarray([len(ph)] + list(ph), dtype=np.int64).tobytes())
        self.fingerprint = h.hexdigest()
        self._dev = {}

    def __len__(self):
        return len(self.phrases)

    def __repr__(self):
        return "ContextGraph(%d phrases, %d states, V=%d, boost=%g)" % (len(self.phrases), self.n_states,
                                                                        self.vocab_size, self.boost)

    def step(self, state, k):
        """(next state, increment) of appending token k in ``state`` (blank: (state, 0.0)), from the tables."""
        return int(self.next[state, k]), float(self.delta[state, k])

    def to(self, device):
        """The tables on ``device`` as one int32 buffer next | delta (fp32 bits) | pending (fp32 bits), uploaded once per
        device.  An empty graph has no tables: None."""
        if not self.phrases:
            return None
        dev = torch.device(device)
        key = str(dev)
        if key not in self._dev:
            flat = np.concatenate([self.next.reshape(-1), self.delta.view(np.int32).reshape(-1),
                                   self.pending.view(np.int32)])
            self._dev[key] = torch.from_numpy(flat).to(dev)
        return self._dev[key]


def check_context(context, V, blank):
    """Validate a beam search's ``context`` argument against the model's vocabulary V and blank: None or a ContextGraph
    with vocab_size V and the same blank.  Returns the graph when it has phrases, else None (an empty graph builds the
    search without context).  Raises TypeError / ValueError; touches no device."""
    if context is None:
        return None
    if not isinstance(context, ContextGraph):
        raise TypeError("context must be a ContextGraph, got %s" % type(context).__name__)
    if context.vocab_size != V:
        raise ValueError("context graph has vocab_size %d, the model %d" % (context.vocab_size, V))
    if context.blank != blank:
        raise ValueError("context graph was built for blank %d, the search uses %d" % (context.blank, blank))
    return context if context.phrases else None


def context_cache_key(graph):
    """What an engine built with the checked graph depends on: its content fingerprint (None without context)."""
    return None if graph is None else graph.fingerprint
