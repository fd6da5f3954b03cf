"""Minimum word error rate training without a GPU: the restatement (tests/mwer_oracle.py) against exhaustive alignment
enumeration and hand cases, the word segmentation of ``mwer.word_table`` against the reference tokenizers' decoding
followed by jiwer's transform, and every refusal raised on the host before any device work."""
import itertools
import random
import types

import pytest
import torch

from edgedict_b200 import mwer
from tests import mwer_oracle as mo

CHARS = ["<nul>", "<pad>", "<bos>", "<unk>", " ", "a", "b", "c", "'"]
BPE = ["<nul>", "<pad>", "<bos>", "<unk>", "a", "b", "c", "a</w>", "b</w>", "c</w>", "ab</w>", "ab", "bc</w>", "abc</w>",
       "'</w>"]


def _char_tok():
    return types.SimpleNamespace(id2token=list(CHARS))


def _bpe_tok(pieces=BPE):
    vocab = {p: i for i, p in enumerate(pieces)}
    return types.SimpleNamespace(tokenizer=types.SimpleNamespace(get_vocab=lambda: dict(vocab)))


def _words(table, ids):
    return mo.words(ids, table.entries.tolist(), table.chars.tolist())


# ---- the Levenshtein restatement --------------------------------------------------------------------------------------
def test_levenshtein_is_a_minimal_alignment():
    for ref in mo.pairs("ab", 4):
        for hyp in mo.pairs("ab", 4):
            e, s, d, n = mo.levenshtein(ref, hyp)
            al = mo.alignments(ref, hyp)
            assert e == s + d + n == min(x + y + z for x, y, z in al)
            assert (s, d, n) in al
            assert len(hyp) - len(ref) == n - d


@pytest.mark.parametrize("ref,hyp,want", [
    ("", "", (0, 0, 0, 0)),
    ("abc", "", (3, 0, 3, 0)),
    ("", "abc", (3, 0, 0, 3)),
    ("abc", "abc", (0, 0, 0, 0)),
    ("abc", "axc", (1, 1, 0, 0)),
    ("abc", "ac", (1, 0, 1, 0)),
    ("ac", "abc", (1, 0, 0, 1)),
    ("ab", "ba", (2, 2, 0, 0)),        # a tie between two substitutions and a deletion + insertion: the diagonal
    ("abcd", "bcde", (2, 0, 1, 1)),
    ("kitten", "sitting", (3, 2, 0, 1)),
])
def test_levenshtein_hand_cases(ref, hyp, want):
    assert mo.levenshtein(ref, hyp) == want


def test_levenshtein_tie_prefers_deletion_over_insertion():
    # D[1][1] of "a" vs "b" ties the diagonal (1) with neither step; "ab" vs "b": the diagonal path costs 2, a deletion 1
    assert mo.levenshtein("ab", "b") == (1, 0, 1, 0)
    assert mo.levenshtein("b", "ab") == (1, 0, 0, 1)


# ---- word segmentation against decode + jiwer -------------------------------------------------------------------------
def test_char_table_layout():
    t = mwer.word_table(_char_tok())
    assert t.vocab_size == len(CHARS)
    cls = t.entries[:, 2].tolist()
    assert cls[:4] == [mo.DROP] * 4 and cls[4] == mo.SEP and set(cls[5:]) == {mo.INSIDE}


def test_bpe_table_layout():
    t = mwer.word_table(_bpe_tok())
    e = t.entries.tolist()
    assert [c for _, _, c in e[:4]] == [mo.DROP] * 4
    assert e[BPE.index("ab</w>")][1:] == [2, mo.END] and e[BPE.index("ab")][1:] == [2, mo.INSIDE]
    off, cnt, _ = e[BPE.index("abc</w>")]
    assert t.chars[off:off + cnt].tolist() == [ord(c) for c in "abc"]


@pytest.mark.parametrize("seed", range(4))
def test_char_words_equal_decode_and_jiwer(seed):
    rng = random.Random(seed)
    t = mwer.word_table(_char_tok())
    for _ in range(400):
        ids = [rng.choice([0, 1, 2, 3, 4, 4, 5, 6, 7, 8]) for _ in range(rng.randint(0, 14))]
        assert _words(t, ids) == mo.jiwer_words(mo.char_decode(ids, CHARS))


@pytest.mark.parametrize("seed", range(4))
def test_bpe_words_equal_decode_and_jiwer(seed):
    rng = random.Random(seed)
    t = mwer.word_table(_bpe_tok())
    for _ in range(400):
        ids = [rng.randrange(len(BPE)) for _ in range(rng.randint(0, 12))]
        assert _words(t, ids) == mo.jiwer_words(mo.bpe_decode(ids, BPE))


def test_two_tokenisations_are_one_word():
    t = mwer.word_table(_bpe_tok())
    a = [BPE.index("ab</w>")]
    b = [BPE.index("a"), BPE.index("b</w>")]
    c = [BPE.index("a"), 0, BPE.index("b"), BPE.index("c</w>"), BPE.index("abc</w>")]
    assert _words(t, a) == _words(t, b) == ["ab"]
    assert _words(t, c) == ["abc", "abc"]
    assert mo.levenshtein(_words(t, a), _words(t, b)) == (0, 0, 0, 0)


def test_word_counts_equal_the_string_levenshtein_of_decoded_texts():
    rng = random.Random(7)
    for tok, dec, n in ((_char_tok(), lambda ids: mo.char_decode(ids, CHARS), len(CHARS)),
                        (_bpe_tok(), lambda ids: mo.bpe_decode(ids, BPE), len(BPE))):
        t = mwer.word_table(tok)
        for _ in range(300):
            r = [rng.randrange(n) for _ in range(rng.randint(0, 10))]
            h = [rng.randrange(n) for _ in range(rng.randint(0, 10))]
            assert mo.levenshtein(_words(t, r), _words(t, h)) == \
                mo.levenshtein(mo.jiwer_words(dec(r)), mo.jiwer_words(dec(h)))


def test_plain_pieces_and_ids_outside_the_table():
    t = mwer.word_table(["<nul>", "<pad>", "<bos>", "<unk>", "_", "x", "y", None], end_suffix=None, separators=("_",))
    assert _words(t, [5, 4, 4, 6, 7, 5, 99, -1, 6]) == ["x", "yxy"]


# ---- the risk restatement ---------------------------------------------------------------------------------------------
def test_risk_single_rank_and_equal_errors_are_zero():
    loss, post, grad = mo.risk([[3.0, 1.0, 2.0]], [[4, 1, 2]], [[1, 0, 0]])
    assert loss == 0.0 and post[0] == [1.0, 0.0, 0.0] and grad[0] == [0.0, 0.0, 0.0]
    loss, _, grad = mo.risk([[3.0, 1.0, 2.0]], [[2, 2, 2]], [[1, 1, 1]])
    assert loss == 0.0 and grad[0] == [0.0, 0.0, 0.0]


def test_risk_gradient_is_the_derivative():
    c, e, v = [[1.0, 2.5, 0.3, 4.0], [0.5, 0.7, 9.0, 9.0]], [[3, 1, 4, 1], [5, 9, 2, 6]], [[1, 1, 1, 1], [1, 1, 0, 0]]
    _, _, grad = mo.risk(c, e, v, g=1.0)
    for b, i in itertools.product(range(2), range(4)):
        h = 1e-6
        cp = [row[:] for row in c]
        cm = [row[:] for row in c]
        cp[b][i] += h
        cm[b][i] -= h
        fd = (mo.risk(cp, e, v)[0] - mo.risk(cm, e, v)[0]) / (2 * h)
        assert abs(fd - grad[b][i]) < 1e-8


# ---- refusals before any device work ----------------------------------------------------------------------------------
def _ids(*shape):
    return torch.zeros(*shape, dtype=torch.int32)


@pytest.mark.parametrize("args,kw,exc", [
    ((_ids(2, 3).float(), [1, 1], _ids(2, 3), [1, 1]), {}, TypeError),
    (([[1, 2]], [1], _ids(1, 3), [1]), {}, TypeError),
    ((_ids(2), [1, 1], _ids(2, 3), [1, 1]), {}, ValueError),
    ((_ids(2, 3), [1], _ids(2, 3), [1, 1]), {}, ValueError),
    ((_ids(2, 3), [1, 4], _ids(2, 3), [1, 1]), {}, ValueError),
    ((_ids(2, 3), [1, -1], _ids(2, 3), [1, 1]), {}, ValueError),
    ((_ids(2, 3), [1.5, 1], _ids(2, 3), [1, 1]), {}, TypeError),
    ((_ids(1, 5000), [4097], _ids(1, 3), [1]), {}, ValueError),
    ((_ids(2, 3), [1, 1], _ids(3, 3), [1, 1, 1]), {}, ValueError),
    ((_ids(2, 3), [1, 1], _ids(3, 3), [1, 1, 1]), {"ref_index": [0, 3]}, ValueError),
    ((_ids(2, 3), [1, 1], _ids(3, 3), [1, 1, 1]), {"ref_index": [0]}, ValueError),
    ((_ids(2, 3), [1, 1], _ids(2, 3), [1, 1]), {"word_table": [1, 2]}, TypeError),
    ((_ids(2, 3), [1, 1], _ids(2, 3), [1, 1]), {}, RuntimeError),       # valid, but on the CPU
])
def test_edit_distance_refusals(args, kw, exc):
    with pytest.raises(exc):
        mwer.edit_distance(*args, **kw)


def test_word_table_refusals():
    with pytest.raises(TypeError):
        mwer.word_table(3)
    with pytest.raises(TypeError):
        mwer.word_table(["a", 3])
    with pytest.raises(ValueError):
        mwer.word_table([])
    with pytest.raises(ValueError):
        mwer.word_table(["a"], end_suffix="")
    with pytest.raises(ValueError):
        mwer.check_word_table(mwer.word_table(["a", "b"]), 3)


@pytest.mark.parametrize("args,exc", [
    ((torch.zeros(2, 3, dtype=torch.float64), _ids(2, 3)), TypeError),
    ((torch.zeros(2, 3), torch.zeros(2, 3)), TypeError),
    ((torch.zeros(2, 3), _ids(2, 4)), ValueError),
    ((torch.zeros(3), _ids(3)), ValueError),
    ((torch.zeros(2, 1025), _ids(2, 1025)), ValueError),
    ((torch.zeros(2, 3), _ids(2, 3), _ids(3, 2)), ValueError),
    ((torch.zeros(2, 3), _ids(2, 3)), RuntimeError),
])
def test_expected_risk_refusals(args, exc):
    with pytest.raises(exc):
        mwer.expected_risk(*args)


@pytest.mark.parametrize("value,exc", [(True, TypeError), ("1", TypeError), (-0.1, ValueError),
                                       (float("nan"), ValueError), (float("inf"), ValueError)])
def test_ce_weight_refusals(value, exc):
    with pytest.raises(exc):
        mwer.check_ce_weight(value)


TINY = dict(vocab_embed_size=8, vocab_size=16, input_size=6, enc_hidden_size=8, enc_layers=1, enc_dropout=0.0,
            enc_proj_size=8, dec_hidden_size=8, dec_layers=1, dec_dropout=0.0, dec_proj_size=8, joint_size=8)


@pytest.mark.parametrize("kw,exc", [
    (dict(W=0), ValueError), (dict(W=1025), ValueError), (dict(W=4, nbest=5), ValueError),
    (dict(nbest=True), TypeError), (dict(ce_weight=-1.0), ValueError), (dict(max_symbols=0), ValueError),
    (dict(word_table=["a"]), TypeError), (dict(word_table=mwer.word_table(["a"] * 8)), ValueError),
])
def test_model_mwer_loss_refusals(kw, exc):
    from edgedict_b200.rnnt.models import CTCEncoder, Transducer
    xs, ys = torch.zeros(2, 8, 6), torch.ones(2, 3, dtype=torch.int32)
    xlen, ylen = torch.tensor([8, 6]), torch.tensor([3, 2])
    for m in (Transducer(**TINY), CTCEncoder(16, 6, 8, 1, 0.0, 8)):
        with pytest.raises(exc):
            m.mwer_loss(xs, ys, xlen, ylen, **kw)


def test_transducer_mwer_loss_refuses_fastemit():
    from edgedict_b200.rnnt.models import Transducer
    m = Transducer(fastemit_lambda=0.1, **TINY)
    with pytest.raises(ValueError):
        m.mwer_loss(torch.zeros(2, 8, 6), torch.ones(2, 3, dtype=torch.int32), torch.tensor([8, 6]),
                    torch.tensor([3, 2]))


def test_ctc_mwer_loss_refuses_several_symbols():
    from edgedict_b200.rnnt.models import CTCEncoder
    with pytest.raises(ValueError):
        CTCEncoder(16, 6, 8, 1, 0.0, 8).mwer_loss(torch.zeros(2, 8, 6), torch.ones(2, 3, dtype=torch.int32),
                                                  torch.tensor([8, 6]), torch.tensor([3, 2]), max_symbols=2)


def test_vectorised_levenshtein_equals_the_loop():
    rng = random.Random(3)
    for _ in range(300):
        r = [rng.randrange(3) for _ in range(rng.randint(0, 12))]
        h = [rng.randrange(3) for _ in range(rng.randint(0, 12))]
        assert mo.levenshtein_np(r, h) == mo.levenshtein(r, h)
