"""Pure-Python restatement of csrc/mwer.cu: the Levenshtein counts with the kernel's tie rule, the word segmentation of
a word table, the expected risk and its gradient in fp64; and, to pin the segmentation, the reference tokenizers'
decoding (CharTokenizer.decode, CharBPE decoding) with jiwer's default transform."""
import itertools
import math
import re

INSIDE, END, SEP, DROP = 0, 1, 2, 3
SPECIALS = ("<nul>", "<pad>", "<bos>", "<unk>")


def levenshtein(ref, hyp):
    """(errors, S, D, I) of hyp against ref (sequences of comparable units): D[i][j] takes the diagonal on ties, then
    the deletion D[i-1][j] + 1, then the insertion D[i][j-1] + 1, carrying the counts of the chosen predecessor."""
    prev = [(j, 0, 0, j) for j in range(len(hyp) + 1)]
    for i in range(1, len(ref) + 1):
        cur = [(i, 0, i, 0)]
        for j in range(1, len(hyp) + 1):
            d, s, dl, n = prev[j - 1]
            dia = (d, s, dl, n) if ref[i - 1] == hyp[j - 1] else (d + 1, s + 1, dl, n)
            d, s, dl, n = prev[j]
            dele = (d + 1, s, dl + 1, n)
            d, s, dl, n = cur[j - 1]
            ins = (d + 1, s, dl, n + 1)
            if dia[0] <= dele[0] and dia[0] <= ins[0]:
                cur.append(dia)
            elif dele[0] <= ins[0]:
                cur.append(dele)
            else:
                cur.append(ins)
        prev = cur
    return prev[len(hyp)]


def alignments(ref, hyp):
    """Every alignment of hyp to ref as (S, D, I): exhaustive, for short sequences."""
    out = set()

    def walk(i, j, s, d, n):
        if i == len(ref) and j == len(hyp):
            out.add((s, d, n))
            return
        if i < len(ref) and j < len(hyp):
            walk(i + 1, j + 1, s + (ref[i] != hyp[j]), d, n)
        if i < len(ref):
            walk(i + 1, j, s, d + 1, n)
        if j < len(hyp):
            walk(i, j + 1, s, d, n + 1)

    walk(0, 0, 0, 0, 0)
    return out


def words(ids, entries, chars):
    """The words (strings) of ids under a word table ({offset, count, class} per id, code points): a word is a
    maximal non-empty run of characters closed by a word end (its characters included), a separator or the end; dropped
    ids and ids outside the table vanish."""
    out, cur, is_open = [], [], False
    for k in ids:
        if not 0 <= k < len(entries):
            continue
        off, cnt, cls = entries[k]
        if cls in (INSIDE, END) and cnt > 0:
            cur.extend(chars[off:off + cnt])
            is_open = True
        if cls in (END, SEP):
            if is_open:
                out.append("".join(chr(c) for c in cur))
            cur, is_open = [], False
    if is_open:
        out.append("".join(chr(c) for c in cur))
    return out


def char_decode(ids, id2token):
    """CharTokenizer.decode: the tokens joined, the special tokens' strings removed."""
    text = "".join(id2token[k] for k in ids)
    for t in SPECIALS:
        text = text.replace(t, "")
    return text


def bpe_decode(ids, pieces, suffix="</w>"):
    """HuggingFaceTokenizer.decode (CharBPETokenizer, BPEDecoder): ids above 3 with a piece, the suffix turned into a
    space except in the last token."""
    toks = [pieces[k] for k in ids if k > 3 and k < len(pieces) and pieces[k] is not None]
    return "".join(t.replace(suffix, "" if i == len(toks) - 1 else " ") for i, t in enumerate(toks))


def jiwer_words(text):
    """jiwer's default wer transform: RemoveMultipleSpaces, Strip, ReduceToListOfListOfWords."""
    text = re.sub(r"\s\s+", " ", text).strip()
    return [w for w in text.split(" ") if w]


def risk(costs, errors, valid, g=1.0):
    """(loss, posteriors [B][N], d loss / d costs [B][N]) in fp64, the kernel's formulas and order."""
    B = len(costs)
    loss, post, grad = 0.0, [], []
    for c, e, v in zip(costs, errors, valid):
        idx = [i for i in range(len(c)) if v[i]]
        m = max((-float(c[i]) for i in idx), default=-math.inf)
        z = sum(math.exp(-float(c[i]) - m) for i in idx)
        ebar = sum(int(e[i]) for i in idx) / len(idx) if idx else 0.0
        p = [math.exp(-float(c[i]) - m) / z if v[i] else 0.0 for i in range(len(c))]
        r = sum(p[i] * (int(e[i]) - ebar) for i in idx)
        loss += r
        post.append(p)
        grad.append([-(p[i] * ((int(e[i]) - ebar) - r)) * g / B if v[i] else 0.0 for i in range(len(c))])
    return loss / B, post, grad


def min_distance(ref, hyp):
    return min(s + d + n for s, d, n in alignments(ref, hyp))


def pairs(alphabet, max_len):
    for n in range(max_len + 1):
        yield from itertools.product(alphabet, repeat=n)


def levenshtein_np(ref, hyp):
    """``levenshtein`` vectorised over anti-diagonals (numpy int64), for sequences of thousands of units."""
    import numpy as np
    r, h = np.asarray(ref, dtype=np.int64), np.asarray(hyp, dtype=np.int64)
    R, H = len(r), len(h)
    diags = {}
    for d in range(R + H + 1):
        i = np.arange(max(0, d - H), min(R, d) + 1)
        j = d - i
        v = np.zeros((4, len(i)), dtype=np.int64)                  # distance, S, D, I
        top, left = i == 0, (j == 0) & (i > 0)
        v[0, top], v[3, top] = j[top], j[top]
        v[0, left], v[2, left] = i[left], i[left]
        m = ~top & ~left
        if m.any():
            im, jm = i[m], j[m]
            p1, lo1 = diags[d - 1]
            p2, lo2 = diags[d - 2]
            dia = p2[:, im - 1 - lo2].copy()
            sub = r[im - 1] != h[jm - 1]
            dia[0] += sub
            dia[1] += sub
            dele = p1[:, im - 1 - lo1].copy()
            dele[0] += 1
            dele[2] += 1
            ins = p1[:, im - lo1].copy()
            ins[0] += 1
            ins[3] += 1
            take_dia = (dia[0] <= dele[0]) & (dia[0] <= ins[0])
            take_del = ~take_dia & (dele[0] <= ins[0])
            v[:, m] = np.where(take_dia, dia, np.where(take_del, dele, ins))
        diags[d] = (v, int(i[0]))
        diags.pop(d - 3, None)
    v, lo = diags[R + H]
    return tuple(int(x) for x in v[:, R - lo])
