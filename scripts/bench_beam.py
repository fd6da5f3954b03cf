"""E6D2_LARGE batched beam search through the public API: Transducer.beam_search for several beam widths and
greedy_decode as an anchor, B = 32 synthetic utterances of T = 500 input frames (60 ms each after stacking and
downsampling, 30 s of audio; T' = 250 encoder frames), weights x 2 so that symbols appear.  Each call ends in a device
synchronise; every width is warmed up once before it is timed.  Prints one JSON line (card name and power limit
read in the same run).

--lm adds shallow fusion of a random language model of cli/train_lm.py's shape, LMModel(1024, 64, 1024, 2), at
LM_WEIGHT / LENGTH_BONUS: every width is then timed with and without the LM in the same run, the two calls alternating
rep by rep so that both see the same state of the shared machine."""
import argparse, copy, json, os, subprocess, sys, time
import torch
sys.path.insert(0, os.getcwd())
from edgedict_b200.rnnt.models import Transducer

LARGE = dict(vocab_embed_size=64, vocab_size=1024, input_size=240, enc_hidden_size=1024, enc_layers=6, enc_dropout=0.0,
             enc_proj_size=640, dec_hidden_size=512, dec_layers=2, dec_dropout=0.1, dec_proj_size=640, joint_size=640)
FRAME_SEC = 0.060

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--frames", type=int, default=500)
ap.add_argument("--widths", default="1,4,8")
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--lm", action="store_true")
args = ap.parse_args()
LM_WEIGHT, LENGTH_BONUS = 0.5, 1.0

torch.manual_seed(10)
model = Transducer(output_loss=False, **LARGE).eval()
with torch.no_grad():
    for p in model.parameters():
        p.mul_(2.0)
model.cuda()
g = torch.Generator().manual_seed(0)
xs = torch.randn(args.batch, args.frames, 240, generator=g).cuda()
xlen = torch.full((args.batch,), args.frames, dtype=torch.int32)
audio = args.batch * args.frames * FRAME_SEC


def timed(*fns):
    """Times each of fns args.reps times, the calls alternating; returns [(min s, median s, last output)] per fn."""
    for fn in fns:
        fn()                                          # warm-up: engine build, module load
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    outs = [None] * len(fns)
    for _ in range(args.reps):
        for i, fn in enumerate(fns):
            t0 = time.perf_counter()
            outs[i] = fn()
            torch.cuda.synchronize()
            ts[i].append(time.perf_counter() - t0)
    return [(min(t), sorted(t)[len(t) // 2], o) for t, o in zip(ts, outs)]


lm = None
if args.lm:
    torch.manual_seed(11)
    lm = torch.nn.Module()                            # the layout of the reference's LMModel(1024, 64, 1024, 2)
    lm.encoder = torch.nn.Embedding(1024, 64)
    lm.rnn = torch.nn.LSTM(64, 1024, 2, batch_first=True)
    lm.decoder = torch.nn.Linear(1024, 1024)
    lm = lm.eval().cuda()
# the fused calls go through a shallow copy of the model (same parameters, its own engine cache): Transducer keeps one
# resident beam engine, and alternating calls on one model would rebuild it every time
model_lm = copy.copy(model)


res = dict(config="E6D2_LARGE beam search, B=%d x T=%d input frames (%.0f s of audio)" % (args.batch, args.frames, audio))
[(best, med, (ids, _))] = timed(lambda: model.greedy_decode(xs, xlen))
res["greedy"] = dict(min_s=round(best, 4), median_s=round(med, 4), audio_sec_per_sec=round(audio / med, 1),
                     nonblank=int(sum(int((i != 0).sum()) for i in ids)))
for W in [int(w) for w in args.widths.split(",")]:
    fns = [lambda: model.beam_search(xs, xlen, W=W)]
    if lm is not None:
        fns.append(lambda: model_lm.beam_search(xs, xlen, W=W, lm=lm, lm_weight=LM_WEIGHT, length_bonus=LENGTH_BONUS))
    for tag, (best, med, (seqs, nlp)) in zip(("beam_W%d" % W, "beam_lm_W%d" % W), timed(*fns)):
        res[tag] = dict(min_s=round(best, 4), median_s=round(med, 4), audio_sec_per_sec=round(audio / med, 1),
                        nonblank=sum(len(s) for s in seqs), mean_neg_logp=round(float(nlp.mean()), 4))
if lm is not None:
    res["lm"] = dict(shape="LMModel(1024, 64, 1024, 2), random init", lm_weight=LM_WEIGHT, length_bonus=LENGTH_BONUS)
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
res["gpu"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()
res["reps"] = args.reps
print(json.dumps(res))
