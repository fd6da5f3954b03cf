"""Minimum word error rate training on the device (csrc/mwer.cu, edgedict_b200/mwer.py, ``mwer_loss`` of the
transducer and CTC models): the edit distance exactly equal to the restatement (tests/mwer_oracle.py) in tokens and in
words, the C ABI's refusals, eb_nbest_pack against ``beam_search(nbest=N)``'s lists, the expected risk against fp64,
and both models' MWER loss and every parameter gradient against an fp64 torch restatement on the same hypotheses."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from edgedict_b200 import mwer, ops
from edgedict_b200._lib import lib
from oracle import model_torch as mt
from tests import mwer_oracle as mo
from tests.test_mwer_host import BPE, CHARS, _bpe_tok, _char_tok
from tests.util import load_tiny, to_t

pytestmark = pytest.mark.gpu


def _pad(rows, width=None):
    width = max([len(r) for r in rows] + [1]) if width is None else width
    out = torch.zeros(len(rows), width, dtype=torch.int32)
    for i, r in enumerate(rows):
        out[i, :len(r)] = torch.tensor(r, dtype=torch.int32)
    return out.cuda(), [len(r) for r in rows]


# ---- edit distance --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("vocab", [2, 5])
def test_tokens_equal_the_restatement(vocab):
    rng = random.Random(vocab)
    lens = [0, 1, 2, 3, 7, 31, 100, 257, 1000, 4096]
    pairs = [(rng.choice(lens), rng.choice(lens)) for _ in range(24)] + [(0, 0), (0, 4096), (4096, 0), (4096, 4096)]
    hyps = [[rng.randrange(vocab) for _ in range(a)] for a, _ in pairs]
    refs = [[rng.randrange(vocab) for _ in range(b)] for _, b in pairs]
    refs[-1] = hyps[-1][:4000] + refs[-1][:96]                          # a long near match
    h, hl = _pad(hyps)
    r, rl = _pad(refs)
    got = mwer.edit_distance(h, hl, r, rl).cpu().numpy()
    for k in range(len(pairs)):
        e, s, d, n = mo.levenshtein_np(refs[k], hyps[k])
        assert got[k].tolist() == [e, s, d, n, len(refs[k])], k


@pytest.mark.parametrize("style", ["char", "bpe"])
def test_words_equal_the_restatement(style):
    rng = random.Random(11)
    if style == "char":
        table, n = mwer.word_table(_char_tok()), len(CHARS)
        dec = lambda ids: mo.char_decode(ids, CHARS)          # noqa: E731
        draw = lambda: rng.choice([0, 1, 2, 3, 4, 4, 4, 5, 6, 7, 8])    # noqa: E731
    else:
        table, n = mwer.word_table(_bpe_tok()), len(BPE)
        dec = lambda ids: mo.bpe_decode(ids, BPE)             # noqa: E731
        draw = lambda: rng.randrange(n)                       # noqa: E731
    hyps = [[draw() for _ in range(rng.choice([0, 1, 5, 20, 300, 4096]))] for _ in range(40)]
    refs = [[draw() for _ in range(rng.choice([0, 1, 5, 20, 300, 4096]))] for _ in range(40)]
    if style == "bpe":                                        # another tokenisation of the same words
        a, b = BPE.index("ab</w>"), [BPE.index("a"), BPE.index("b</w>")]
        refs[0] = [a, BPE.index("c</w>"), a] * 5
        hyps[0] = (b + [BPE.index("c</w>")] + b) * 5
    h, hl = _pad(hyps)
    r, rl = _pad(refs)
    got = mwer.edit_distance(h, hl, r, rl, word_table=table).cpu().numpy()
    for k in range(len(hyps)):
        rw, hw = mo.words(refs[k], table.entries.tolist(), table.chars.tolist()), \
            mo.words(hyps[k], table.entries.tolist(), table.chars.tolist())
        assert rw == mo.jiwer_words(dec(refs[k])) and hw == mo.jiwer_words(dec(hyps[k]))
        ids = {w: i for i, w in enumerate(sorted(set(rw + hw)))}
        e, s, d, nn = mo.levenshtein_np([ids[w] for w in rw], [ids[w] for w in hw])
        assert got[k].tolist() == [e, s, d, nn, len(rw)], k
    if style == "bpe":
        assert got[0, 0] == 0 and got[0, 4] == 15


def test_error_rate_is_the_corpus_ratio():
    rng = random.Random(5)
    table = mwer.word_table(_char_tok())
    hyps = [[rng.choice([4, 5, 6, 7]) for _ in range(rng.randint(1, 40))] for _ in range(9)]
    refs = [[rng.choice([4, 5, 6, 7]) for _ in range(rng.randint(1, 40))] for _ in range(3)]
    h, hl = _pad(hyps)
    r, rl = _pad(refs)
    index = [k % 3 for k in range(9)]
    errs = units = 0
    for k in range(9):
        rw = mo.jiwer_words(mo.char_decode(refs[index[k]], CHARS))
        hw = mo.jiwer_words(mo.char_decode(hyps[k], CHARS))
        errs += mo.levenshtein(rw, hw)[0]
        units += len(rw)
    assert mwer.error_rate(h, hl, r, rl, index, table) == errs / units


def test_batch_and_row_order_invariance():
    rng = random.Random(2)
    hyps = [[rng.randrange(4) for _ in range(rng.randint(0, 600))] for _ in range(17)]
    refs = [[rng.randrange(4) for _ in range(rng.randint(0, 600))] for _ in range(5)]
    index = [rng.randrange(5) for _ in range(17)]
    h, hl = _pad(hyps, 700)
    r, rl = _pad(refs, 650)
    full = mwer.edit_distance(h, hl, r, rl, index)
    perm = list(range(17))
    rng.shuffle(perm)
    hp, hlp = _pad([hyps[p] for p in perm], 700)
    got = mwer.edit_distance(hp, hlp, r, rl, [index[p] for p in perm])
    assert torch.equal(got, full[perm])
    for k in (0, 9, 16):
        one = mwer.edit_distance(h[k:k + 1], hl[k:k + 1], r[index[k]:index[k] + 1], rl[index[k]:index[k] + 1])
        assert torch.equal(one[0], full[k])
    assert torch.equal(mwer.edit_distance(h, hl, r, rl, index), full)


def test_abi_refusals():
    h, hl = _pad([[1, 2, 3], [2]])
    r, rl = _pad([[1, 2], [3, 3, 3]])
    out = torch.full((2, 5), 7, dtype=torch.int32, device="cuda")
    table = mwer.word_table(_char_tok())
    wt, wc = table.device("cuda")

    def call(meta_h, n_hyp=2, n_ref=2, hyp=h, word=False, vocab=0, ld_h=3):
        meta = meta_h.cuda()
        return lib().eb_edit_distance(hyp.data_ptr() if hyp is not None else None, ld_h, r.data_ptr(), 3,
                                      meta.data_ptr(), meta_h.data_ptr(), n_hyp, n_ref,
                                      wt.data_ptr() if word else None, wc.data_ptr() if word else None,
                                      wt.shape[0] if word else 0, vocab, out.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream)

    ok = torch.tensor([3, 1, 2, 3, 0, 1], dtype=torch.int32)
    assert call(ok) == 0
    torch.cuda.synchronize()
    out.fill_(7)
    for bad in ([4, 1, 2, 3, 0, 1], [-1, 1, 2, 3, 0, 1], [3, 1, 4, 3, 0, 1], [3, 1, 2, -2, 0, 1], [3, 1, 2, 3, 0, 2],
                [3, 1, 2, 3, -1, 1]):
        assert call(torch.tensor(bad, dtype=torch.int32)) == 2
    assert call(ok, hyp=None) == 2
    assert call(ok, word=True, vocab=len(CHARS) + 1) == 2
    big = torch.tensor([4097, 1, 2, 3, 0, 1], dtype=torch.int32)
    assert call(big, ld_h=5000) == 2                                    # refused before the launch reads any row
    torch.cuda.synchronize()
    assert call(ok, word=True, vocab=len(CHARS)) == 0
    torch.cuda.synchronize()


# ---- N-best packing ---------------------------------------------------------------------------------------------------
# tiny.npz's sizes (12 input features, joint 28, V = 16) are below the bf16 GEMMs' multiple-of-8 rule: bf16 mode runs
# a model of the same depth at sizes it takes, on seeded inputs of tiny.npz's shapes and lengths
BF16_CFG = dict(vocab_embed_size=16, vocab_size=32, input_size=16, enc_hidden_size=32, enc_layers=3, enc_dropout=0,
                enc_proj_size=32, dec_hidden_size=32, dec_layers=2, dec_dropout=0, dec_proj_size=32, joint_size=32)


def _tiny(module_type="LSTM", seed=0, precision="fp32"):
    """(model on the device, xs, ys int32) -- tiny.npz's model and inputs in fp32 mode (a seeded GRU model of its sizes
    for module_type GRU), BF16_CFG's in bf16 mode."""
    from edgedict_b200.rnnt.models import Transducer
    z, cfg, sd, _ = load_tiny()
    xs, ys = torch.as_tensor(z["xs"]), torch.as_tensor(z["ys"]).to(torch.int32)
    torch.manual_seed(seed)
    if precision == "bf16":
        cfg = BF16_CFG
        g = torch.Generator().manual_seed(seed)
        xs = torch.randn(xs.shape[0], xs.shape[1], cfg["input_size"], generator=g)
        ys = torch.randint(4, cfg["vocab_size"], tuple(ys.shape), generator=g, dtype=torch.int32)
    m = Transducer(module_type=module_type, **cfg)
    if module_type == "LSTM" and precision == "fp32":
        m.load_state_dict(dict(to_t(sd)))
    m = m.cuda()
    m.set_precision(precision)
    return m, xs, ys


def test_nbest_pack_rows_are_the_beam_lists():
    from edgedict_b200.stream_engine import BeamEngine, nbest_lists
    m, xs, _ = _tiny()
    xs = xs.cuda()
    with torch.no_grad():
        h_enc, _ = m.encoder(xs)
    B, T = h_enc.shape[:2]
    W, N = 8, 6
    eng = BeamEngine(m, B, T, W, merge=True, nbest=N)
    frames = torch.tensor([T, 0, T - 2], dtype=torch.int32, device="cuda")
    buf = eng.run(h_enc, frames)
    L = eng.ids.shape[-1]
    lists = nbest_lists(buf, B, N, L)
    ref, rlen = _pad([[5, 6, 7], [], [9]], 4)
    n = B * N * L
    labels, lens, valid = ops.nbest_pack(buf[:n].view(B, N, L), buf[2 * n + B * N:], ref,
                                         torch.tensor(rlen, dtype=torch.int32, device="cuda"), max(L, 4))
    labels, lens, valid = labels.cpu(), lens.cpu(), valid.cpu()
    assert len(lists[1]) == 1                                           # ranks past the count
    for b in range(B):
        for i in range(N):
            row = b * (N + 1) + i
            want = lists[b][i].tokens.tolist() if i < len(lists[b]) else []
            assert int(lens[row]) == len(want) and labels[row, :len(want)].tolist() == want
            assert not labels[row, len(want):].any()
            assert int(valid[b, i]) == (i < len(lists[b]))
        row = b * (N + 1) + N
        assert int(lens[row]) == rlen[b] and labels[row, :rlen[b]].tolist() == ref[b, :rlen[b]].tolist()


# ---- expected risk ----------------------------------------------------------------------------------------------------
def _risk_inputs(B=7, N=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    c = (torch.rand(B, N, generator=g) * 6).float()
    e = torch.randint(0, 9, (B, N), generator=g, dtype=torch.int32)
    cnt = torch.randint(1, N + 1, (B,), generator=g)
    v = (torch.arange(N)[None] < cnt[:, None]).to(torch.int32)
    return c, e, v


def test_expected_risk_against_fp64():
    c, e, v = _risk_inputs()
    cc = c.cuda().requires_grad_(True)
    loss, post = mwer.expected_risk(cc, e.cuda(), v.cuda())
    (loss * 1.7).sum().backward()
    want, wpost, wgrad = mo.risk(c.tolist(), e.tolist(), v.tolist(), g=1.7)
    assert abs(float(loss) - want) <= 1e-6 * max(1.0, abs(want))
    assert np.allclose(post.cpu().numpy(), np.array(wpost), rtol=0, atol=1e-7)
    assert np.allclose(cc.grad.cpu().numpy(), np.array(wgrad), rtol=1e-6, atol=1e-9)


def test_expected_risk_zero_cases():
    c, e, v = _risk_inputs(B=4, N=5, seed=3)
    v[:] = 0
    v[:, 0] = 1                                                          # one valid rank
    cc = c.cuda().requires_grad_(True)
    loss, post = mwer.expected_risk(cc, e.cuda(), v.cuda())
    loss.sum().backward()
    assert float(loss) == 0.0 and not cc.grad.any() and torch.equal(post[:, 0].cpu(), torch.ones(4))
    e[:] = 3                                                             # equal errors
    cc = c.cuda().requires_grad_(True)
    loss, _ = mwer.expected_risk(cc, e.cuda())
    loss.sum().backward()
    assert float(loss) == 0.0 and not cc.grad.any()


def test_expected_risk_is_bitwise_repeatable():
    c, e, v = _risk_inputs(B=33, N=16, seed=9)
    outs = []
    for _ in range(3):
        cc = c.cuda().requires_grad_(True)
        loss, post = mwer.expected_risk(cc, e.cuda(), v.cuda())
        loss.sum().backward()
        outs.append((loss.detach().cpu(), post.cpu(), cc.grad.cpu()))
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(o, outs[0]))


# ---- Transducer.mwer_loss ---------------------------------------------------------------------------------------------
def _risk64(costs, errors, valid):
    mask = valid.bool()
    c = costs[:, :errors.shape[1]]
    p = torch.softmax((-c).masked_fill(~mask, float("-inf")), 1).masked_fill(~mask, 0.0)
    e = errors.double()
    ebar = (e * mask).sum(1) / mask.sum(1)
    return (p * (e - ebar[:, None])).sum(1).mean()


def _hyp_rows(lists, ys, ylen, N):
    rows, lens = [], []
    for b, hyps in enumerate(lists):
        for i in range(N):
            t = hyps[i].tokens.tolist() if i < len(hyps) else []
            rows.append(t)
        rows.append(ys[b, :int(ylen[b])].tolist())
    return rows


def _grads_close(model, sd64, bar):
    worst = 0.0
    for k, p in model.named_parameters():
        g, r = p.grad.double().cpu(), sd64[k].grad
        if r is None:
            r = torch.zeros_like(g)
        worst = max(worst, float((g - r).norm() / (r.norm() + 1e-12)))
    assert worst < bar, worst
    return worst


def _transducer_case(module_type, precision, K, xlen, ylen, N=4, W=4, ce=0.3):
    m, xs, ys = _tiny(module_type, seed=5, precision=precision)
    loss = m.mwer_loss(xs.cuda(), ys.cuda(), xlen, ylen, W=W, nbest=N, ce_weight=ce, max_symbols=K)
    loss.backward()
    last = {k: v.cpu() for k, v in m.last_mwer.items()}
    with torch.no_grad():
        lists = m.beam_search(xs[:, :int(xlen.max())].cuda(), xlen, W=W, merge=True, nbest=N, max_symbols=K)
    B = xs.shape[0]
    assert last["count"].tolist() == [len(x) for x in lists]
    rows = _hyp_rows(lists, ys, ylen, N)
    for b in range(B):
        for i in range(len(lists[b])):
            assert int(last["errors"][b, i]) == mo.levenshtein(rows[b * (N + 1) + N], rows[b * (N + 1) + i])[0]
    # the fp64 restatement of the whole loss on the same hypotheses
    sd = {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}
    xs64 = xs[:, :int(xlen.max())].double()
    if module_type == "LSTM":
        h_enc, _ = mt.encoder(sd, xs64)
    else:
        h_enc, _ = mt.encoder_gru(sd, xs64)
    labels = torch.zeros(len(rows), max(max(len(r) for r in rows), 1), dtype=torch.int64)
    for k, r in enumerate(rows):
        labels[k, :len(r)] = torch.tensor(r, dtype=torch.int64)
    lens = torch.tensor([len(r) for r in rows], dtype=torch.int32)
    labels = labels[:, :int(lens.max())]
    h_dec, _ = mt.decoder(sd, labels)
    idx = torch.arange(B).repeat_interleave(N + 1)
    xl = mt.scale_length(h_enc.shape[1], xlen)[idx]
    logits = mt.joint(sd, h_enc[idx], h_dec)
    costs = mt.rnnt_loss(logits, labels.int(), xl, lens, 0, "none", use_ref=False).view(B, N + 1)
    valid = torch.arange(N)[None] < last["count"][:, None]
    ref_loss = _risk64(costs, last["errors"], valid) + ce * costs[:, N].sum() / B
    ref_loss.backward()
    c32 = last["costs"].double()
    cbar = 2e-5 if precision == "fp32" else 2e-2
    assert float((c32 - costs.detach()).abs().max() / costs.detach().abs().max()) < cbar
    assert abs(float(loss) - float(ref_loss)) <= cbar * max(1.0, abs(float(ref_loss)))
    return m, sd, last, loss, (xs, ys)


@pytest.mark.parametrize("module_type", ["LSTM", "GRU"])
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("K", [1, 2])
def test_transducer_mwer_loss_against_fp64(module_type, precision, K):
    z = load_tiny()[0]
    xlen, ylen = torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"])
    m, sd, last, _, _ = _transducer_case(module_type, precision, K, xlen, ylen)
    assert (last["count"] >= 2).any()                                   # the risk term is not empty
    _grads_close(m, sd, 2e-3 if precision == "fp32" else 5e-2)


def test_transducer_ragged_batch_with_an_empty_transcript():
    z = load_tiny()[0]
    xlen = torch.as_tensor(z["xlen"]).clone()
    xlen[1] = 2
    ylen = torch.as_tensor(z["ylen"]).clone()
    ylen[1] = 0
    m, sd, _, _, _ = _transducer_case("LSTM", "fp32", 1, xlen, ylen)
    _grads_close(m, sd, 2e-3)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_transducer_nbest1_is_ce_times_forward(precision):
    z = load_tiny()[0]
    xlen, ylen = torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"])
    m, xs, ys = _tiny(precision=precision)
    xs, ys = xs.cuda(), ys.cuda()
    loss = m.mwer_loss(xs, ys, xlen, ylen, W=4, nbest=1, ce_weight=0.25)
    loss.backward()
    g1 = {k: p.grad.clone() for k, p in m.named_parameters()}
    assert not m.last_mwer["posteriors"].ne(1).any()
    m.zero_grad()
    fwd = m(xs, ys, xlen, ylen)
    (0.25 * fwd).backward()
    bar = 1e-5 if precision == "fp32" else 1e-3
    assert abs(float(loss) - 0.25 * float(fwd)) <= bar * abs(0.25 * float(fwd))
    for k, p in m.named_parameters():
        assert float((g1[k] - p.grad).norm()) <= 10 * bar * float(p.grad.norm()) + 1e-9, k


def test_transducer_word_level_errors():
    z = load_tiny()[0]
    xlen, ylen = torch.as_tensor(z["xlen"]), torch.as_tensor(z["ylen"])
    m, xs, ys = _tiny()
    xs, ys, cfg = xs.cuda(), ys.cuda(), load_tiny()[1]
    pieces = ["<nul>", "<pad>", "<bos>", "<unk>", " "] + [chr(ord("a") + k) for k in range(cfg["vocab_size"] - 5)]
    table = mwer.word_table(pieces)
    m.mwer_loss(xs, ys, xlen, ylen, W=4, word_table=table)
    lists = m.beam_search(xs, xlen, W=4, merge=True, nbest=4)
    got = m.last_mwer["errors"].cpu()
    for b, hyps in enumerate(lists):
        rw = mo.jiwer_words(mo.char_decode(ys[b, :int(ylen[b])].tolist(), pieces))
        for i, h in enumerate(hyps):
            assert int(got[b, i]) == mo.levenshtein(rw, mo.jiwer_words(mo.char_decode(h.tokens.tolist(), pieces)))[0]


# ---- CTCEncoder.mwer_loss ---------------------------------------------------------------------------------------------
def _ctc_case(precision, xlen, ylen, N=4, W=6, ce=0.2):
    from edgedict_b200.rnnt.models import CTCEncoder, _ctc_frames
    torch.manual_seed(1)
    V, F_in = (12, 10) if precision == "fp32" else (16, 16)          # bf16 GEMMs take multiples of 8
    m = CTCEncoder(vocab_size=V, input_size=F_in, enc_hidden_size=16 if precision == "fp32" else 32, enc_layers=2,
                   enc_dropout=0.0, proj_size=16).cuda()
    m.set_precision(precision)
    g = torch.Generator().manual_seed(2)
    xs = torch.randn(len(xlen), int(max(xlen.max(), 1)), F_in, generator=g)
    ys = torch.randint(4, V, (len(xlen), 5), generator=g, dtype=torch.int32)
    loss = m.mwer_loss(xs.cuda(), ys.cuda(), xlen, ylen, W=W, nbest=N, ce_weight=ce)
    loss.backward()
    last = {k: v.cpu() for k, v in m.last_mwer.items()}
    with torch.no_grad():
        lists = m.beam_search(xs.cuda(), xlen, W=W, nbest=N)
    B = xs.shape[0]
    rows = _hyp_rows(lists, ys, ylen, N)
    assert last["count"].tolist() == [len(x) for x in lists]
    sd = {k: v.detach().double().cpu().requires_grad_(True) for k, v in m.state_dict().items()}
    h, _ = mt.encoder_gru(sd, xs.double(), pre="model.")
    lp = F.log_softmax(F.linear(h, sd["tovocab.0.weight"], sd["tovocab.0.bias"]), -1)
    idx = torch.arange(B).repeat_interleave(N + 1)
    frames = _ctc_frames(lp.shape[1], xlen, B)[idx]
    labels = torch.zeros(len(rows), max(max(len(r) for r in rows), 1), dtype=torch.int64)
    for k, r in enumerate(rows):
        labels[k, :len(r)] = torch.tensor(r, dtype=torch.int64)
    lens = torch.tensor([len(r) for r in rows])
    costs = F.ctc_loss(lp[idx].transpose(0, 1), labels, frames, lens, reduction="none").view(B, N + 1)
    valid = torch.arange(N)[None] < last["count"][:, None]
    for b in range(B):
        for i in range(len(lists[b])):
            assert int(last["errors"][b, i]) == mo.levenshtein(rows[b * (N + 1) + N], rows[b * (N + 1) + i])[0]
    ref_loss = _risk64(costs, last["errors"], valid) + ce * costs[:, N].sum() / B
    ref_loss.backward()
    cbar = 2e-5 if precision == "fp32" else 2e-2
    assert float((last["costs"].double() - costs.detach()).abs().max() / costs.detach().abs().max()) < cbar
    assert abs(float(loss) - float(ref_loss)) <= cbar * max(1.0, abs(float(ref_loss)))
    _grads_close(m, sd, 2e-3 if precision == "fp32" else 5e-2)
    return m, last


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_ctc_mwer_loss_against_fp64(precision):
    _, last = _ctc_case(precision, torch.tensor([24, 17, 9]), torch.tensor([5, 3, 2]))
    assert (last["count"] >= 2).any()


def test_ctc_ragged_batch_with_a_length0_utterance():
    _ctc_case("fp32", torch.tensor([24, 0, 13]), torch.tensor([4, 0, 2]))


def test_ctc_nbest1_is_ce_times_the_ctc_loss():
    from edgedict_b200 import ctc
    from edgedict_b200.rnnt.models import CTCEncoder, _ctc_frames
    torch.manual_seed(1)
    m = CTCEncoder(vocab_size=12, input_size=10, enc_hidden_size=16, enc_layers=2, enc_dropout=0.0, proj_size=16).cuda()
    xs = torch.randn(3, 20, 10).cuda()
    ys = torch.randint(4, 12, (3, 5), dtype=torch.int32).cuda()
    xlen, ylen = torch.tensor([20, 14, 9]), torch.tensor([5, 3, 2])
    loss = m.mwer_loss(xs, ys, xlen, ylen, W=3, nbest=1, ce_weight=0.5)
    loss.backward()
    g1 = {k: p.grad.clone() for k, p in m.named_parameters()}
    m.zero_grad()
    lp = m(xs)
    ref = ctc.ctc_loss(lp.transpose(0, 1), ys, _ctc_frames(lp.shape[1], xlen, 3), ylen, reduction="sum") * 0.5 / 3
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    for k, p in m.named_parameters():
        assert float((g1[k] - p.grad).norm()) <= 1e-4 * float(p.grad.norm()) + 1e-9, k
