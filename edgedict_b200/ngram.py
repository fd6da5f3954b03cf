"""Token n-gram language models for shallow fusion in the device beam searches (``Transducer.beam_search(ngram=...)``,
``CTCEncoder.beam_search`` and ``ctc.beam_search``).

``NgramLM(arpa, vocab_size)`` reads an ARPA file whose words are the model's tokens and compiles it, on the host, to
sparse backoff tables the beam launches score inside the selection.  The rule, with every log10 value of the file
turned into a natural log once in float64 (``log10 * ln 10``) and rounded once to fp32, a missing backoff weight 0:

- a state is a token string h, |h| <= n - 1, that is an m-gram of order m < n in the file, or a proper prefix of one
  of its n-grams (backoff 0 then); the root is the empty history; suffix(h) is the longest proper suffix of h that is a
  state; the start state is [<s>] when it is a state, else the root;
- appending a non-blank token k to a hypothesis in state h scores, in fp32, innermost term first,
  g(h, k) = p(h k) when h k is an entry of the file, else bo(h) + g(suffix(h), k), and at the root the unigram
  ln P(k), or ln P(<unk>) when k has no unigram, or -100 ln 10 (KenLM's convention) without <unk> either;
- the next state is the longest suffix of h k that is a state (the root when k has no unigram);
- blank, a CTC stay and a closed multi-symbol slot's stay keep the state and add nothing;
- with a </s> unigram in the file the end term is e(h) = g(h, </s>) by the same rule; without one there is none.

The state is a function of the token sequence, so merging equal sequences stays exact.  The tables hold, per state,
its backoff, suffix, depth (suffix links to the root) and the CSR range of its children; per child its token (sorted
within the state), p and next state.  A history that is only a prefix is stored as a child of its context whose p is
the backoff value g(context, k) itself, so the row a state's chain builds and the walk that finds the next state see
every state the same way.
"""
import gzip
import hashlib
import math
import numbers

import numpy as np
import torch

MAX_ORDER = 8                  # the device walks at most MAX_ORDER - 1 suffix links
MAX_INDEX = 2 ** 31 - 1        # states and children are indexed by int32
LN10 = math.log(10.0)
KENLM_UNK = -100.0             # log10 of a token with neither a unigram nor <unk>
BOS, EOS, UNK = "<s>", "</s>", "<unk>"


def _ln(x):
    """ARPA log10 value -> fp32 natural log, one rounding."""
    return np.float32(x * LN10)


def _read_arpa(path):
    """{order: [(words tuple, log10 p, log10 bo or None)]} and the declared order of an ARPA file.  Raises ValueError
    for a malformed file."""
    opener = gzip.open if str(path).endswith(".gz") else open
    with opener(path, "rt", encoding="utf-8") as fh:
        lines = [ln.strip() for ln in fh]
    i = 0
    while i < len(lines) and lines[i] != "\\data\\":
        i += 1
    if i == len(lines):
        raise ValueError("%s: no \\data\\ section" % path)
    i += 1
    counts = {}
    while i < len(lines) and lines[i].startswith("ngram "):
        try:
            m, c = lines[i][6:].split("=")
            m, c = int(m), int(c)
        except ValueError:
            raise ValueError("%s: bad count line %r" % (path, lines[i])) from None
        if m != len(counts) + 1 or c < 0:
            raise ValueError("%s: bad count line %r" % (path, lines[i]))
        counts[m] = c
        i += 1
    if not counts:
        raise ValueError("%s: \\data\\ declares no n-gram counts" % path)
    n = len(counts)
    sections = {}
    for m in range(1, n + 1):
        while i < len(lines) and not lines[i]:
            i += 1
        if i == len(lines) or lines[i] != "\\%d-grams:" % m:
            raise ValueError("%s: expected the \\%d-grams: section" % (path, m))
        i += 1
        rows = []
        while i < len(lines) and lines[i] and not lines[i].startswith("\\"):
            f = lines[i].split()
            if len(f) not in ((m + 1, m + 2) if m < n else (m + 1,)):
                raise ValueError("%s: %d-gram line %r has %d fields" % (path, m, lines[i], len(f)))
            try:
                p = float(f[0])
                bo = float(f[m + 1]) if len(f) == m + 2 else None
            except ValueError:
                raise ValueError("%s: bad number in %r" % (path, lines[i])) from None
            if not math.isfinite(p) or (bo is not None and not math.isfinite(bo)):
                raise ValueError("%s: non-finite number in %r" % (path, lines[i]))
            rows.append((tuple(f[1:m + 1]), p, bo))
            i += 1
        if len(rows) != counts[m]:
            raise ValueError("%s: \\data\\ declares %d %d-grams, the section holds %d" % (path, counts[m], m, len(rows)))
        sections[m] = rows
    while i < len(lines) and not lines[i]:
        i += 1
    if i == len(lines) or lines[i] != "\\end\\":
        raise ValueError("%s: no \\end\\ after the %d-grams" % (path, n))
    return sections, n


class NgramLM:
    """The ARPA model ``arpa`` (a path; ``.gz`` is read through gzip) over ``vocab_size`` tokens, the rule in the module
    docstring.  ``vocab=None``: the ARPA words are decimal token ids; otherwise ``vocab[i]`` is the word of token i
    (None or "" for a token without one, such as blank).  An ARPA word that maps to no token is dropped with every
    n-gram that holds it (``n_dropped`` counts those n-grams); a word that maps to ``blank`` is a ValueError.

    Tables, numpy on the host: ``unigram`` fp32 [V] (the <unk> fill applied), per state ``bo`` fp32, ``suffix``,
    ``depth``, ``first``, ``count`` int32, per child ``tok`` int32, ``prob`` fp32, ``next`` int32, ``end`` fp32 per
    state (None without </s>) and ``start``.  ``step(state, k)`` scores one token on the host from the tables;
    ``fingerprint`` identifies the content; ``to(device)`` uploads the tables once per device.  Raises TypeError /
    ValueError before any device work for a malformed file or argument, an order above MAX_ORDER and a model whose
    states or children overflow int32 indices."""

    def __init__(self, arpa, vocab_size, vocab=None, blank=0):
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
        if vocab is not None:
            if isinstance(vocab, (str, bytes)):
                raise TypeError("vocab must be a sequence of %d strings" % V)
            vocab = list(vocab)
            if len(vocab) != V:
                raise ValueError("vocab has %d entries, the model %d tokens" % (len(vocab), V))
            word_id = {}
            for i, w in enumerate(vocab):
                if w is None or w == "":
                    continue
                if not isinstance(w, str):
                    raise TypeError("vocab entries must be strings or None, got %r" % (w,))
                if w in (BOS, EOS, UNK) or w in word_id:
                    raise ValueError("vocab word %r is reserved or repeated" % w)
                word_id[w] = i
            to_id = word_id.get
        else:
            def to_id(w):
                if not w.isdigit():
                    return None
                k = int(w)
                return k if k < V else None
        if not isinstance(arpa, (str, bytes)) and not hasattr(arpa, "__fspath__"):
            raise TypeError("arpa must be a path, got %s" % type(arpa).__name__)
        sections, n = _read_arpa(arpa)
        if n > MAX_ORDER:
            raise ValueError("the model has order %d, above the cap of %d" % (n, MAX_ORDER))
        self.order, self.vocab_size, self.blank = n, V, blank
        BOS_ID, EOS_ID = V, V + 1                        # internal ids of the sentence markers
        ids = {BOS: BOS_ID, EOS: EOS_ID}
        prob, bo = {}, {}
        unk = None
        dropped = 0
        for m in range(1, n + 1):
            for words, p, b in sections[m]:
                if m == 1 and words[0] == UNK:
                    unk = p
                    continue
                key = []
                for j, w in enumerate(words):
                    k = ids.get(w)
                    if k is None:
                        k = to_id(w)
                        if k == blank:
                            raise ValueError("ARPA word %r maps to blank (token %d)" % (w, blank))
                    elif (k == BOS_ID and j > 0) or (k == EOS_ID and j < m - 1):
                        k = None                         # a marker out of place: no history or token holds it
                    if k is None:
                        break
                    key.append(k)
                if len(key) < m:
                    dropped += 1
                    continue
                key = tuple(key)
                prob[key] = _ln(p)
                if b is not None:
                    bo[key] = _ln(b)
        self.n_dropped = dropped
        fill = _ln(unk if unk is not None else KENLM_UNK)
        unigram = np.full(V, fill, dtype=np.float32)
        for k in range(V):
            if (k,) in prob:
                unigram[k] = prob[(k,)]
        self.has_end = (EOS_ID,) in prob
        # states: the entries of order < n that end in a token or <s>, and every proper prefix of an entry
        states = {()}
        for key in prob:
            if len(key) < n and key[-1] != EOS_ID:
                states.add(key)
            for j in range(1, len(key)):
                states.add(key[:j])
        order = sorted(states, key=lambda h: (len(h), h))
        index = {h: i for i, h in enumerate(order)}
        S = len(order)

        def longest_state_suffix(h):
            for j in range(len(h) + 1):
                if h[j:] in index:
                    return index[h[j:]]
            return 0

        suffix = np.zeros(S, dtype=np.int32)
        depth = np.zeros(S, dtype=np.int32)
        bov = np.zeros(S, dtype=np.float32)
        for i, h in enumerate(order[1:], 1):
            suffix[i] = longest_state_suffix(h[1:])
            depth[i] = depth[suffix[i]] + 1
            bov[i] = bo.get(h, np.float32(0.0))

        def g(h, k):                                     # the backoff rule over the entries, fp32
            if h + (k,) in prob:
                return prob[h + (k,)]
            if not h:
                return unigram[k] if k < V else fill
            return np.float32(bov[index[h]] + g(order[suffix[index[h]]], k))

        children = [[] for _ in range(S)]
        for key in prob:
            if key[-1] < V and key[:-1] in index:
                children[index[key[:-1]]].append(key[-1])
        for h in order[1:]:                              # histories that are only prefixes
            if h[-1] < V and h not in prob:
                children[index[h[:-1]]].append(h[-1])
        count = np.array([len(c) for c in children], dtype=np.int64)
        if S > MAX_INDEX or int(count.sum()) > MAX_INDEX:
            raise ValueError("the model has %d states and %d children, above the int32 index cap of %d"
                             % (S, int(count.sum()), MAX_INDEX))
        first = np.zeros(S, dtype=np.int64)
        first[1:] = np.cumsum(count)[:-1]
        E = int(count.sum())
        tok = np.zeros(E, dtype=np.int32)
        pr = np.zeros(E, dtype=np.float32)
        nxt = np.zeros(E, dtype=np.int32)
        for i, h in enumerate(order):
            for j, k in enumerate(sorted(children[i])):
                c = int(first[i]) + j
                tok[c] = k
                pr[c] = g(h, k)
                nxt[c] = longest_state_suffix(h + (k,))
        self.unigram, self.bo, self.suffix, self.depth = unigram, bov, suffix, depth
        self.first, self.count = first.astype(np.int32), count.astype(np.int32)
        self.tok, self.prob, self.next = tok, pr, nxt
        self.end = np.array([g(h, EOS_ID) for h in order], dtype=np.float32) if self.has_end else None
        self.start = index.get((BOS_ID,), 0)
        self.n_states, self.n_children = S, E
        self.histories = order                           # the token string of every state (<s> as id V)
        h = hashlib.sha1()
        h.update(np.asarray([V, blank, n, self.start, self.has_end], dtype=np.int64).tobytes())
        for a in self._arrays():
            h.update(a.tobytes())
        self.fingerprint = h.hexdigest()
        self._dev = {}

    def __repr__(self):
        return "NgramLM(order %d, %d states, %d children, V=%d)" % (self.order, self.n_states, self.n_children,
                                                                  self.vocab_size)

    def _arrays(self):
        a = [self.unigram, self.bo, self.suffix, self.depth, self.first, self.count, self.tok, self.prob, self.next]
        return a + ([self.end] if self.has_end else [])

    @property
    def nbytes(self):
        """Bytes of the device tables."""
        return sum(a.nbytes for a in self._arrays())

    def _child(self, s, k):
        lo, hi = int(self.first[s]), int(self.first[s]) + int(self.count[s])
        c = lo + int(np.searchsorted(self.tok[lo:hi], k))
        return c if c < hi and self.tok[c] == k else -1

    def step(self, state, k):
        """(next state, g(state, k)) of appending the non-blank token k in ``state``, from the tables as the device
        reads them: the row of the chain's states from the root outward, and the walk down the suffix chain."""
        chain = [int(state)]
        while chain[-1] != 0:
            chain.append(int(self.suffix[chain[-1]]))
        v = self.unigram[k]
        for s in reversed(chain[:-1]):
            v = np.float32(self.bo[s] + v)
            c = self._child(s, k)
            if c >= 0:
                v = self.prob[c]
        for s in chain:
            c = self._child(s, k)
            if c >= 0:
                return int(self.next[c]), float(v)
        return 0, float(v)

    def to(self, device):
        """The tables on ``device`` as one int32 buffer in _arrays' order (fp32 as bits) and the element offset of
        each table in it, uploaded once per device."""
        dev = torch.device(device)
        key = str(dev)
        if key not in self._dev:
            parts, offs, o = [], [], 0
            for a in self._arrays():
                a = a.view(np.int32) if a.dtype == np.float32 else a.astype(np.int32)
                offs.append(o)
                pad = -len(a) % 64                       # 256-byte aligned tables
                parts += [a, np.zeros(pad, dtype=np.int32)]
                o += len(a) + pad
            self._dev[key] = (torch.from_numpy(np.concatenate(parts)).to(dev), offs)
        return self._dev[key]


def check_ngram(ngram, V, blank):
    """Validate a beam search's ``ngram`` argument against the model's vocabulary V and blank: None or an NgramLM
    with vocab_size V and the same blank.  Raises TypeError / ValueError; touches no device."""
    if ngram is None:
        return None
    if not isinstance(ngram, NgramLM):
        raise TypeError("ngram must be an NgramLM, got %s" % type(ngram).__name__)
    if ngram.vocab_size != V:
        raise ValueError("ngram model has vocab_size %d, the search %d" % (ngram.vocab_size, V))
    if ngram.blank != blank:
        raise ValueError("ngram model was built for blank %d, the search uses %d" % (ngram.blank, blank))
    return ngram


def check_ngram_weight(ngram, ngram_weight):
    """ngram_weight as a finite float; nonzero only with an ngram.  Raises TypeError / ValueError."""
    if isinstance(ngram_weight, bool) or not isinstance(ngram_weight, numbers.Real):
        raise TypeError("ngram_weight must be a real number, got %r" % (ngram_weight,))
    w = float(ngram_weight)
    if not math.isfinite(w):
        raise ValueError("ngram_weight must be finite, got %r" % (ngram_weight,))
    if ngram is None and w != 0.0:
        raise ValueError("ngram_weight needs an ngram")
    return w


def ngram_cache_key(ngram, ngram_weight, length_bonus=0.0):
    """What an engine built with the checked model depends on: its fingerprint, the weight and, without an LM, the
    length bonus the n-gram term carries (None without a model)."""
    return None if ngram is None else (ngram.fingerprint, float(ngram_weight), float(length_bonus))
