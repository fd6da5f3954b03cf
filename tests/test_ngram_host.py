"""edgedict_b200.ngram on the host: the ARPA reader, the backoff tables and their walk against a brute-force
restatement over the n-gram dictionary (tests/ngram_oracle.py), normalisation, hand-written cases, refusals and the
fingerprint.  No GPU."""
import math

import numpy as np
import pytest
import torch

from edgedict_b200.ngram import MAX_ORDER, NgramLM, check_ngram, check_ngram_weight, ngram_cache_key
from tests import ngram_oracle as no

LN10 = math.log(10.0)


def _model(tmp_path, seed, order, V, n_sent=60, max_len=8):
    sents = no.corpus(seed, V, n_sent, max_len)
    m = no.estimate(sents, order, V)
    path = no.write_arpa(str(tmp_path / ("m%d_%d.arpa" % (seed, order))), m)
    return m, path


@pytest.mark.parametrize("seed,order,V", [(0, 2, 6), (1, 3, 7), (2, 4, 5), (3, 3, 12)])
def test_walk_equals_brute_force(tmp_path, seed, order, V):
    """step(h, k) is the fp32 backoff rule bit for bit and within 1e-6 of fp64; next states are the longest suffix
    of h k that is a state; the end term is g(h, </s>)."""
    m, path = _model(tmp_path, seed, order, V)
    ng = NgramLM(path, V)
    b32, b64 = no.Brute(m, V, np.float32), no.Brute(m, V, np.float64)
    assert set(ng.histories) == {tuple(V if w == no.BOS else w for w in h) for h in b32.states}
    index = {h: i for i, h in enumerate(ng.histories)}
    for s, h in enumerate(ng.histories):
        hb = tuple(no.BOS if w == V else w for w in h)
        for k in range(1, V):
            nxt, g = ng.step(s, k)
            assert np.float32(g).view(np.int32) == b32.g(hb, k).view(np.int32), (hb, k)
            assert abs(g - b64.g(hb, k)) <= 1e-6 * max(1.0, abs(g))
            want = b32.next(hb, k)
            assert nxt == index[tuple(V if w == no.BOS else w for w in want)], (hb, k)
        assert ng.end[s].view(np.int32) == b32.g(hb, no.EOS).view(np.int32)
    assert ng.histories[ng.start] == (V,)


@pytest.mark.parametrize("seed,order,V", [(4, 2, 6), (5, 3, 6), (6, 4, 5)])
def test_normalised(tmp_path, seed, order, V):
    """Vocabulary = the non-blank tokens and </s>: sum_k exp g(h, k) + exp e(h) = 1 in every state."""
    m, path = _model(tmp_path, seed, order, V)
    ng = NgramLM(path, V)
    b64 = no.Brute(m, V, np.float64)
    for h in b64.states:
        tot = sum(math.exp(b64.g(h, k)) for k in range(1, V)) + math.exp(b64.g(h, no.EOS))
        assert abs(tot - 1.0) < 1e-5, (h, tot)
    for s in range(ng.n_states):
        tot = sum(math.exp(ng.step(s, k)[1]) for k in range(1, V)) + math.exp(float(ng.end[s]))
        assert abs(tot - 1.0) < 1e-5


HAND = """
\\data\\
ngram 1=5
ngram 2=4
ngram 3=2

\\1-grams:
-1.0\t<s>\t-0.5
-0.5\t1\t-0.25
-0.75\t2\t-0.125
-1.25\t9
-0.6\t<unk>

\\2-grams:
-0.3\t<s> 1\t-0.1
-0.2\t1 2
-0.4\t2 1
-0.7\t9 1

\\3-grams:
-0.05\t<s> 1 2
-0.15\t1 2 1

\\end\\
"""


def _write(tmp_path, text, name="hand.arpa"):
    p = tmp_path / name
    p.write_text(text)
    return str(p)


def ln(x):
    return np.float32(x * LN10)


def test_hand_written(tmp_path):
    """<s> as the start state, a history without its own entry (1 2 exists only as the context of 1 2 1), <unk>,
    no </s>, and the word 9 outside V = 4: dropped with its bigram."""
    ng = NgramLM(_write(tmp_path, HAND), 4)
    assert ng.n_dropped == 2 and ng.end is None and not ng.has_end
    idx = {h: i for i, h in enumerate(ng.histories)}
    assert ng.start == idx[(4,)]
    # unigram fill: token 3 has no unigram, so it scores <unk>
    assert ng.unigram[3] == ln(-0.6) and ng.unigram[1] == ln(-0.5)
    s = ng.start
    s1, g = ng.step(s, 1)
    assert s1 == idx[(4, 1)] and g == ln(-0.3)
    s2, g = ng.step(s1, 2)
    assert s2 == idx[(1, 2)] and g == ln(-0.05)             # <s> 1 2 is top order: next is its suffix 1 2
    assert ng.bo[s2] == 0.0                                # 1 2 has no backoff (top-order context only... its bigram)
    s3, g = ng.step(s2, 1)
    assert s3 == idx[(2, 1)] and g == ln(-0.15)
    _, g = ng.step(s3, 3)                                  # 2 1 -> 3: bo(2 1) = 0, bo(1) + <unk>
    assert g == np.float32(np.float32(0.0) + np.float32(ln(-0.25) + ln(-0.6)))
    _, g = ng.step(idx[(1,)], 1)                           # bo(1) + p(1)
    assert g == np.float32(ln(-0.25) + ln(-0.5))


def test_unk_absent_and_orders(tmp_path):
    text = HAND.replace("-0.6\t<unk>\n", "").replace("ngram 1=5", "ngram 1=4")
    ng = NgramLM(_write(tmp_path, text), 4)
    assert ng.unigram[3] == np.float32(-100.0 * LN10)
    one = "\\data\\\nngram 1=3\n\n\\1-grams:\n-0.5\t1\n-0.25\t2\n-0.3\t</s>\n\n\\end\\\n"
    ng1 = NgramLM(_write(tmp_path, one, "one.arpa"), 3)
    assert ng1.n_states == 1 and ng1.start == 0 and ng1.end[0] == ln(-0.3)
    assert ng1.step(0, 2) == (0, float(ln(-0.25)))
    m, path = _model(tmp_path, 9, 5, 4, n_sent=40, max_len=10)
    ng5 = NgramLM(path, 4)
    assert ng5.order == 5 and int(ng5.depth.max()) <= 4


def test_vocab_words_and_gzip(tmp_path):
    import gzip
    names = {"1": "a", "2": "b"}
    text = "\n".join("\t".join([f[0], " ".join(names.get(w, w) for w in f[1].split())] + f[2:])
                     if len(f) > 1 else ln for ln in HAND.splitlines() for f in [ln.split("\t")])
    p = tmp_path / "w.arpa.gz"
    with gzip.open(p, "wt") as fh:
        fh.write(text)
    ng = NgramLM(str(p), 4, vocab=[None, "a", "b", ""])
    ref = NgramLM(_write(tmp_path, HAND), 4)
    assert ng.fingerprint == ref.fingerprint


def _bad(tmp_path, text, exc=ValueError, **kw):
    with pytest.raises(exc):
        NgramLM(_write(tmp_path, text, "bad.arpa"), kw.pop("V", 4), **kw)


def test_refusals(tmp_path, monkeypatch):
    _bad(tmp_path, HAND.replace("\\data\\", "data"))
    _bad(tmp_path, HAND.replace("ngram 2=4", "ngram 2=5"))
    _bad(tmp_path, HAND.replace("-0.2\t1 2", "-0.2\t1 2 2 2"))
    _bad(tmp_path, HAND.replace("-0.2\t1 2", "nan\t1 2"))
    _bad(tmp_path, HAND.replace("-0.2\t1 2", "-inf\t1 2"))
    _bad(tmp_path, HAND.replace("-0.5\t1\t-0.25", "-0.5\t0\t-0.25"))        # a word that maps to blank
    _bad(tmp_path, HAND, vocab=["", "1", "2"])                              # vocab of the wrong length
    _bad(tmp_path, HAND, blank=4)
    _bad(tmp_path, HAND, exc=TypeError, blank=1.0)
    _bad(tmp_path, HAND, exc=TypeError, V=4.0)
    many = "\\data\\\n" + "".join("ngram %d=1\n" % m for m in range(1, MAX_ORDER + 2)) + "".join(
        "\n\\%d-grams:\n-0.5\t%s\n" % (m, " ".join(["1"] * m)) for m in range(1, MAX_ORDER + 2)) + "\n\\end\\\n"
    _bad(tmp_path, many)
    import edgedict_b200.ngram as ngm
    monkeypatch.setattr(ngm, "MAX_INDEX", 3)
    _bad(tmp_path, HAND)


def test_check_ngram(tmp_path):
    ng = NgramLM(_write(tmp_path, HAND), 4)
    assert check_ngram(None, 4, 0) is None and check_ngram(ng, 4, 0) is ng
    with pytest.raises(ValueError):
        check_ngram(ng, 5, 0)
    with pytest.raises(ValueError):
        check_ngram(ng, 4, 1)
    with pytest.raises(TypeError):
        check_ngram("x.arpa", 4, 0)
    with pytest.raises(ValueError):
        check_ngram_weight(ng, float("inf"))
    with pytest.raises(ValueError):
        check_ngram_weight(None, 0.5)
    with pytest.raises(TypeError):
        check_ngram_weight(ng, True)
    assert ngram_cache_key(None, 0.0) is None
    assert ngram_cache_key(ng, 0.5) != ngram_cache_key(ng, 0.25)


def test_fingerprint_follows_content(tmp_path):
    a = NgramLM(_write(tmp_path, HAND, "a.arpa"), 4)
    assert a.fingerprint == NgramLM(_write(tmp_path, HAND, "b.arpa"), 4).fingerprint
    others = [NgramLM(_write(tmp_path, HAND.replace("-0.05", "-0.06"), "c.arpa"), 4),
              NgramLM(_write(tmp_path, HAND, "d.arpa"), 5), NgramLM(_write(tmp_path, HAND, "e.arpa"), 4, blank=3)]
    assert len({a.fingerprint} | {o.fingerprint for o in others}) == 1 + len(others)


def test_refusals_come_before_device_work(tmp_path, monkeypatch):
    """The public entries refuse a mismatched model or weight before touching the encoder or the device."""
    from edgedict_b200 import ctc
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer

    def boom(*a, **k):
        raise AssertionError("device work before the n-gram check")

    class Boom(torch.nn.Module):
        forward = staticmethod(boom)
    ng = NgramLM(_write(tmp_path, HAND), 4)
    m = Transducer(output_loss=False, vocab_embed_size=4, vocab_size=8, input_size=6, enc_hidden_size=8,
                   enc_layers=1, enc_dropout=0.0, enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0.0,
                   dec_proj_size=8, joint_size=8)
    monkeypatch.setattr(m, "encoder", Boom())
    with pytest.raises(ValueError, match="vocab_size"):
        m.beam_search(torch.zeros(1, 4, 6), W=2, ngram=ng)
    with pytest.raises(TypeError):
        m.beam_search(torch.zeros(1, 4, 6), W=2, ngram="m.arpa")
    with pytest.raises(ValueError, match="need an lm"):
        m.beam_search(torch.zeros(1, 4, 6), W=2, length_bonus=0.5)
    c = CTCEncoder(vocab_size=4, input_size=6, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0, proj_size=8)
    monkeypatch.setattr(c, "forward", boom)
    with pytest.raises(ValueError, match="finite"):
        c.beam_search(torch.zeros(1, 4, 6), W=2, ngram=ng, ngram_weight=float("nan"))
    with pytest.raises(ValueError, match="vocab_size"):
        ctc.beam_search(torch.zeros(1, 4, 8), [4], 2, ngram=ng)
