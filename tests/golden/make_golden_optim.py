"""Generates tests/golden/optim_tiny.npz by running the REFERENCE's optimizers themselves (only possible where its sources
are):

    EDGEDICT_REFERENCE=<reference checkout> python tests/golden/make_golden_optim.py

* optimizers: ``SM3``, ``AdamW`` and ``Novograd`` of $EDGEDICT_REFERENCE's ``modules/optimizer.py`` and
  ``torch.optim.SGD(momentum=0.9, weight_decay=...)`` (what cli/train.py builds without ``--optim adam``), torch CPU fp32;
  AdamW once with one group and once with two groups, weight decay on the rank >= 2 tensors and 0.0 on the others, as
  cli/pretrain_wav2vec.py splits them;
* parameters: ranks 0, 1, 2 and 3 with odd sizes (bucket padding), one of them a Conv1d weight [C_out, C_in, k];
* 6 steps of seeded gradients, the lr of every group changed after step 3;
* recorded after every step: the parameters and the full ``state_dict()``.

Keys: ``shapes``, ``init.<i>``, ``grad.<step>.<i>`` (steps 1-6), ``<case>.p.<step>.<i>`` and
``<case>.s.<step>.<i>.<key>`` (state tensors and numbers), ``<case>.lr`` = [lr of steps 1-3, lr of steps 4-6].
The committed fixture is what the tests see; nothing at test time reads the reference.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SHAPES = [(), (7,), (5, 9), (6, 3, 5), (11,)]            # (6, 3, 5): a Conv1d weight, 3 input channels, 5 taps
STEPS, LR_CHANGE = 6, 3
CASES = {
    # name: (constructor name, kwargs, two groups, lr after step 3)
    "sgd": ("SGD", dict(lr=0.05, momentum=0.9, weight_decay=1e-2), False, 0.02),
    "sm3": ("SM3", dict(lr=0.1), False, 0.03),
    "adamw": ("AdamW", dict(lr=1e-2, weight_decay=1e-2), False, 3e-3),
    "adamw2": ("AdamW", dict(lr=1e-2, weight_decay=5e-2), True, 4e-3),
    "novograd": ("Novograd", dict(lr=1e-2, weight_decay=1e-3), False, 5e-3),
}


def init_params():
    g = torch.Generator().manual_seed(11)
    return [torch.randn(s, generator=g) for s in SHAPES]


def grads(step):
    g = torch.Generator().manual_seed(1000 + step)
    return [torch.randn(s, generator=g) * (1.0 + i) for i, s in enumerate(SHAPES)]


def reference_classes():
    sys.path.insert(0, os.environ["EDGEDICT_REFERENCE"])
    from modules import optimizer   # (the reference)
    return {"SM3": optimizer.SM3, "AdamW": optimizer.AdamW, "Novograd": optimizer.Novograd, "SGD": torch.optim.SGD}


def groups_of(params, wd, two):
    if not two:
        return params
    return [{"params": [p for p in params if p.dim() >= 2], "weight_decay": wd},
            {"params": [p for p in params if p.dim() < 2], "weight_decay": 0.0}]


def main():
    classes = reference_classes()
    save = {"shapes": np.array([str(s) for s in SHAPES])}
    for i, p in enumerate(init_params()):
        save["init.%d" % i] = p.numpy().copy()
    for step in range(1, STEPS + 1):
        for i, g in enumerate(grads(step)):
            save["grad.%d.%d" % (step, i)] = g.numpy().copy()
    for case, (cls, kw, two, lr2) in CASES.items():
        params = [p.clone().requires_grad_(True) for p in init_params()]
        opt = classes[cls](groups_of(params, kw.get("weight_decay", 0.0), two), **kw)
        order = [id(p) for g in opt.param_groups for p in g["params"]]
        for step in range(1, STEPS + 1):
            if step == LR_CHANGE + 1:
                for g in opt.param_groups:
                    g["lr"] = lr2
            for p, g in zip(params, grads(step)):
                p.grad = g.clone()
            opt.step()
            for i, p in enumerate(params):
                save["%s.p.%d.%d" % (case, step, i)] = p.detach().numpy().copy()
            sd = opt.state_dict()
            for k, st in sd["state"].items():
                i = [id(p) for p in params].index(order[k])       # state index -> parameter of SHAPES
                for key, v in st.items():
                    save["%s.s.%d.%d.%s" % (case, step, i, key)] = \
                        v.numpy().copy() if torch.is_tensor(v) else np.float64(v)
        save["%s.lr" % case] = np.array([kw["lr"], lr2])
        print(case, "ok")
    np.savez_compressed(os.path.join(HERE, "optim_tiny.npz"), **save)


if __name__ == "__main__":
    main()
    print("optim_tiny.npz", os.path.getsize(os.path.join(HERE, "optim_tiny.npz")) // 1024, "KiB")
