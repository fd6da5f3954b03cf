"""Generates tests/golden/*.npz by running the REFERENCE itself (only possible where its sources are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden.py [tiny|e4d1|ref_loss ...]

* model: ``rnnt.models.Transducer`` imported from $EDGEDICT_REFERENCE (torch CPU fp32);
* loss : the reference's CPU library compiled by oracle/Makefile (oracle/_ref, make WARP_TRANSDUCER_DIR=...),
  driven exactly like warprnnt_pytorch._RNNT does on CPU tensors (log_softmax first, 'mean' = /B).

The committed fixtures are what the tests see; nothing at test time reads the reference.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import loss as ol  # noqa: E402

assert ol.have_ref(), "build oracle/_ref first (make -C oracle WARP_TRANSDUCER_DIR=<warp-transducer tree>)"


def Transducer(**kw):
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from rnnt.models import Transducer as T  # (the reference)
    return T(**kw)


class RefLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, acts, labels, act_lens, label_lens):
        lp = torch.log_softmax(acts, -1)
        costs, grads = ol.ref_cpu(lp.detach().numpy(), labels.numpy(), act_lens.numpy(), label_lens.numpy())
        B = acts.shape[0]
        p = lp.exp()
        g = torch.from_numpy(grads) / B
        ctx.g = g - p * g.sum(-1, keepdim=True)      # chain through log_softmax, as autograd would
        return torch.tensor([costs.sum() / B])

    @staticmethod
    def backward(ctx, go):
        return ctx.g * go.view(-1, 1, 1, 1), None, None, None


def run_case(model, xs, ys, xlen, ylen, want_param_grads=True):
    model.zero_grad()
    acts = []
    x = model.encoder.norm(xs[:, :xlen.max()])
    hs = None
    # per-layer encoder activations, rnnt/models.py:55-75
    with torch.no_grad():
        xx = x
        for i, (lstm, proj) in enumerate(zip(model.encoder.lstm.lstms, model.encoder.lstm.projs)):
            y, _ = lstm(xx)
            xx = proj(y if i == 0 else xx + y)
            acts.append(xx.numpy().copy())
    logits = model(xs, ys, xlen, ylen)
    logits.retain_grad()
    xl = model.scale_length(logits, xlen)
    loss = RefLoss.apply(logits, ys[:, :ylen.max()].contiguous().int(), xl, ylen.int())
    loss.backward()
    out = dict(logits=logits.detach().numpy(), loss=loss.detach().numpy(), xlen_scaled=xl.numpy(),
               dlogits=logits.grad.numpy(), layer_acts=acts)
    if want_param_grads:
        out["pgrads"] = {k: p.grad.numpy().copy() for k, p in model.named_parameters()}
    with torch.no_grad():
        h_enc, (eh, ec) = model.encoder(xs[:, :xlen.max()])
        h_dec, (dh, dc) = model.decoder(ys[:, :ylen.max()])
    out.update(h_enc=h_enc.numpy(), h_dec=h_dec.numpy(), enc_h=eh.numpy(), enc_c=ec.numpy(),
               dec_h=dh.numpy(), dec_c=dc.numpy())
    return out


def stream_ref(model, chunks, unk_id=3):
    """rnnt/stream.py:78-120 driven with the reference modules on synthetic log-mel chunks."""
    enc, dec, jnt = model.encoder, model.decoder, model.joint
    L, H = len(enc.lstm.lstms), enc.lstm.hidden_size
    Ld, Hd = dec.lstm.num_layers, dec.lstm.hidden_size
    with torch.no_grad():
        eh, ec = torch.zeros(L, 1, H), torch.zeros(L, 1, H)
        dx, (dh, dc) = dec(torch.ones(1, 1).long() * 2, (torch.zeros(Ld, 1, Hd), torch.zeros(Ld, 1, Hd)))
        out = []
        for ch in chunks:
            ex, (eh, ec) = enc(ch, (eh, ec))
            toks = []
            for k in range(ex.shape[1]):
                prob = jnt(ex[:, k], dx[:, 0])
                pred = prob.argmax(-1).item()
                if pred == unk_id:
                    prob[:, pred] = 0
                    pred = prob.argmax(-1).item()
                if pred != 0:
                    dx, (dh, dc) = dec(torch.ones(1, 1).long() * pred, (dh, dc))
                    toks.append(pred)
            out.append(toks)
    return out


def tiny():
    torch.manual_seed(1234)
    cfg = dict(vocab_embed_size=8, vocab_size=16, input_size=12, enc_hidden_size=24, enc_layers=3,
               enc_dropout=0, enc_proj_size=20, dec_hidden_size=16, dec_layers=2, dec_dropout=0,
               dec_proj_size=12, joint_size=28)
    m = Transducer(output_loss=False, **cfg)
    # make weights larger than the default init so that greedy / stream decode emit non-blanks
    with torch.no_grad():
        for p in m.parameters():
            p.mul_(3.0)
    xs = torch.randn(3, 11, 12)
    ys = torch.randint(4, 16, (3, 4), dtype=torch.int32)
    xlen = torch.tensor([11, 9, 6], dtype=torch.int32)
    ylen = torch.tensor([4, 2, 3], dtype=torch.int32)
    r = run_case(m, xs, ys, xlen, ylen)
    m.eval()
    with torch.no_grad():
        ids, nlp = m.greedy_decode(xs, xlen)
    chunks = [torch.randn(1, 2, 12) for _ in range(40)]
    toks = stream_ref(m, chunks)
    save = {"cfg_" + k: np.array(v) for k, v in cfg.items()}
    save.update({"sd." + k: v.numpy() for k, v in m.state_dict().items()})
    save.update({"pgrad." + k: v for k, v in r.pop("pgrads").items()})
    for i, a in enumerate(r.pop("layer_acts")):
        save["layer_act.%d" % i] = a
    save.update(r)
    save.update(xs=xs.numpy(), ys=ys.numpy(), xlen=xlen.numpy(), ylen=ylen.numpy())
    save["greedy_ids"] = np.stack([np.pad(i, (0, 6 - len(i)), constant_values=-1) for i in ids])
    save["greedy_nlp"] = nlp.numpy()
    save["stream_chunks"] = torch.cat(chunks, 0).numpy()
    save["stream_tokens"] = np.array([t[0] if t else -1 for t in toks], dtype=np.int32)
    assert all(len(t) <= 1 for t in toks)
    np.savez_compressed(os.path.join(HERE, "tiny.npz"), **save)
    print("tiny: loss", r["loss"], "greedy nonblank", sum(int((i != 0).sum()) for i in ids),
          "stream emitted", int((save["stream_tokens"] >= 0).sum()))


def e4d1():
    """BASELINE.json configs[0]; recipe of SURVEY.md section 8(d)."""
    torch.manual_seed(10)
    m = Transducer(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=320,
                   enc_layers=4, enc_dropout=0, enc_proj_size=320, dec_hidden_size=320, dec_layers=1,
                   dec_dropout=0, dec_proj_size=320, joint_size=320, output_loss=False)
    torch.manual_seed(0)
    xs = torch.randn(2, 200, 240)
    ys = torch.randint(4, 1024, (2, 40), dtype=torch.int32)
    save = {}
    sd = m.state_dict()
    save["sd_keys"] = np.array(list(sd.keys()))
    save["sd_sum"] = np.array([float(v.double().sum()) for v in sd.values()])
    save["sd_abs"] = np.array([float(v.double().abs().sum()) for v in sd.values()])
    save["xs_sum"] = np.array(float(xs.double().sum()))
    save["ys"] = ys.numpy()
    for tag, xl, yl in (("full", [200, 200], [40, 40]), ("ragged", [200, 180], [40, 33])):
        xlen = torch.tensor(xl, dtype=torch.int32)
        ylen = torch.tensor(yl, dtype=torch.int32)
        r = run_case(m, xs, ys, xlen, ylen)
        save[tag + ".loss"] = r["loss"]
        save[tag + ".xlen_scaled"] = r["xlen_scaled"]
        save[tag + ".h_enc"] = r["h_enc"].astype(np.float32)
        save[tag + ".h_dec"] = r["h_dec"].astype(np.float32)
        save[tag + ".logits_sub"] = r["logits"][:, ::9, ::5, ::16].copy()
        save[tag + ".dlogits_sub"] = r["dlogits"][:, ::9, ::5, ::16].copy()
        save[tag + ".dlogits_abs_sum"] = np.array(float(np.abs(r["dlogits"]).astype(np.float64).sum()))
        for i, a in enumerate(r["layer_acts"]):
            save[tag + ".layer_act_sub.%d" % i] = a[:, ::7, ::3].copy()
        for k, g in r["pgrads"].items():
            save[tag + ".pgrad_norm." + k] = np.array(float(np.linalg.norm(g.astype(np.float64))))
            save[tag + ".pgrad_head." + k] = g.reshape(-1)[:32].copy()
        print("e4d1", tag, "loss", r["loss"])
    m.eval()
    with torch.no_grad():
        ids, nlp = m.greedy_decode(xs, torch.tensor([200, 200]))
    save["greedy_ids"] = np.stack(ids)
    save["greedy_nlp"] = nlp.numpy()
    np.savez_compressed(os.path.join(HERE, "e4d1.npz"), **save)


# problems of tests/test_oracle_loss.py: (B, T, U, V, ragged), inputs drawn there from RandomState(B * 1000 + T)
REF_LOSS_CASES = [(1, 2, 3, 5, False), (3, 17, 6, 11, True), (2, 50, 16, 20, True), (4, 10, 6, 5, True)]


def ref_loss_inputs(B, T, U, V, ragged):
    rng = np.random.RandomState(B * 1000 + T)
    acts = rng.uniform(0, 1, size=(B, T, U, V)).astype(np.float32)
    labels = rng.randint(1, V, size=(B, U - 1)).astype(np.int32)
    tl = np.full(B, T, np.int32)
    ul = np.full(B, U - 1, np.int32)
    if ragged:
        tl[1:] = rng.randint(1, T + 1, size=B - 1)
        ul[1:] = rng.randint(0, U, size=B - 1)
    return acts, labels, tl, ul


def ref_loss():
    """Costs and log-prob gradients of the reference's CPU loss library on the problems of test_oracle_loss.py."""
    from tests.golden import loss_kat as K
    save = {}
    for case in REF_LOSS_CASES:
        acts, labels, tl, ul = ref_loss_inputs(*case)
        lp, _ = ol.log_softmax(acts)
        c, g = ol.ref_cpu(lp, labels, tl, ul)
        tag = "%d_%d_%d_%d" % case[:4]
        save[tag + ".costs"], save[tag + ".grads"] = c, g
    lp, _ = ol.log_softmax(K.SMALL_ACTS)
    save["small_kat.costs"], _ = ol.ref_cpu(lp, K.SMALL_LABELS, [2], [2])
    np.savez_compressed(os.path.join(HERE, "ref_loss.npz"), **save)


if __name__ == "__main__":
    for name in sys.argv[1:] or ("tiny", "e4d1", "ref_loss"):
        globals()[name]()
    for f in ("tiny.npz", "e4d1.npz", "ref_loss.npz"):
        print(f, os.path.getsize(os.path.join(HERE, f)) // 1024, "KiB")
