"""oracle.ctc (the fp64-capable restatement of CTCEncoder) reproduces tests/golden/ctc_tiny.npz, which the reference's
own CTCEncoder produced (torch CPU fp32)."""
import os

import numpy as np
import torch

from oracle import ctc as oc
from tests.util import GOLDEN, rel_err


def load_ctc_tiny():
    z = np.load(os.path.join(GOLDEN, "ctc_tiny.npz"))
    cfg = {k[4:]: int(z[k]) for k in z.files if k.startswith("cfg_")}
    sd = {k[3:]: z[k] for k in z.files if k.startswith("sd.")}
    return z, cfg, sd


def _ids(z):
    return [row[:n] for row, n in zip(z["greedy_ids"], z["greedy_counts"])]


def test_oracle_forward_matches_reference_logprobs():
    z, _, sd = load_ctc_tiny()
    for dt, bar in ((torch.float32, 2e-6), (torch.float64, 2e-6)):
        sdt = {k: torch.as_tensor(v, dtype=dt) for k, v in sd.items()}
        lp = oc.ctc_encoder_forward(sdt, torch.as_tensor(z["xs"], dtype=dt))
        assert lp.shape == z["logprobs"].shape
        assert rel_err(lp.numpy(), z["logprobs"]) < bar


def test_oracle_greedy_decode_matches_reference():
    z, _, sd = load_ctc_tiny()
    sdt = {k: torch.as_tensor(v) for k, v in sd.items()}
    ids, nlp = oc.ctc_greedy_decode(sdt, torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"]))
    for got, want in zip(ids, _ids(z)):
        assert got.dtype == np.int64 and got.tolist() == want.tolist()
    assert rel_err(nlp.numpy(), z["greedy_nlp"]) < 1e-6
    # the fixture's shapes of interest: a collapsed constant utterance and xlen above T'
    assert int(z["xlen"].max()) > z["logprobs"].shape[1]
    assert 0 < len(ids[2]) < z["logprobs"].shape[1]


def test_oracle_all_blank_decode_matches_reference():
    z, _, sd = load_ctc_tiny()
    sdt = {k: torch.as_tensor(v) for k, v in sd.items()}
    sdt["tovocab.0.bias"] = sdt["tovocab.0.bias"].clone()
    sdt["tovocab.0.bias"][0] += 100.0
    ids, nlp = oc.ctc_greedy_decode(sdt, torch.as_tensor(z["xs"]), torch.as_tensor(z["xlen"]))
    assert all(len(i) == 0 for i in ids)
    assert np.array_equal(nlp.numpy(), z["blank_bias_nlp"])
