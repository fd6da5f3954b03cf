"""Flat-bucket optimizer state for data-parallel training (SURVEY.md 8(e), "next" row N3).

All parameters of a module are re-homed into ONE contiguous fp32 buffer (``flat_params``) and
their gradients into another (``flat_grads``): the gradient all-reduce is a single NCCL call on
``flat_grads`` and the Adam update is a single launch of ``eb_adam_step`` over the bucket
(replaces torch.optim.Adam in cli/baseline.py:141-156,239-245; clip_grad_norm_ via ``eb_sumsq``).

``SGD``, ``SM3``, ``AdamW`` and ``Novograd`` (``FlatOptimizer``) are the optimizers the reference's other trainers build,
as ``torch.optim.Optimizer``s with parameter groups and checkpointable state over the same kind of bucket (csrc/optim.cu).
"""
import math

import torch

from . import _lib, ops


class FlatAdam:
    """torch.optim.Adam over the flat bucket.  ``step(grad_scale, lr, max_norm)``: grad_scale multiplies every
    gradient (1 / loss_scale, 1 / accumulation steps); max_norm applies ``clip_grad_norm_`` semantics on the
    device (cli/baseline.py:239-245) with no host read of the norm; with clipping or loss scaling active a
    non-finite gradient norm skips the update (apex's overflow rule).  ``adamw=True`` selects the reference's own
    AdamW update (modules/optimizer.py:195-292)."""

    def __init__(self, module, lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, adamw=False):
        params = [p for p in module.parameters() if p.requires_grad]
        if not params:
            raise ValueError("no parameters")
        dev = params[0].device
        if dev.type != "cuda":
            raise RuntimeError("FlatAdam needs the module on a CUDA device")
        # every parameter starts on a 16-byte boundary of the bucket (vector loads, TMA-friendly)
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.n = n
        self.flat_params = torch.zeros(n, dtype=torch.float32, device=dev)
        self.flat_grads = torch.zeros(n, dtype=torch.float32, device=dev)
        self.m = torch.zeros(n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(n, dtype=torch.float32, device=dev)
        with torch.no_grad():
            for p, off in zip(params, offs):
                k = p.numel()
                self.flat_params[off:off + k].copy_(p.reshape(-1))
                p.data = self.flat_params[off:off + k].view(p.shape)
                p.grad = self.flat_grads[off:off + k].view(p.shape)
        self.params = params
        self.lr, self.betas, self.eps, self.weight_decay, self.adamw = lr, betas, eps, weight_decay, adamw
        self.step_count = 0
        self._norm = torch.zeros(1, dtype=torch.float32, device=dev)

    def zero_grad(self):
        self.flat_grads.zero_()
        for p in self.params:                       # autograd may have replaced .grad: re-home it
            if p.grad is None or p.grad.data_ptr() < self.flat_grads.data_ptr() or \
                    p.grad.data_ptr() >= self.flat_grads.data_ptr() + 4 * self.n:
                raise RuntimeError("parameter gradient left the flat bucket")

    def grad_norm(self):
        self._norm.zero_()
        ops.sumsq(self.flat_grads, self._norm)
        return self._norm.sqrt()

    def step(self, grad_scale=1.0, lr=None, max_norm=None, check_overflow=False):
        self.step_count += 1
        lr = self.lr if lr is None else lr
        if max_norm or check_overflow or self.adamw:
            ss = None
            if max_norm or check_overflow:
                self._norm.zero_()
                ops.sumsq(self.flat_grads, self._norm)
                ss = self._norm
            ops.adam_step_ex(self.flat_params, self.flat_grads, self.m, self.v, lr, self.betas[0], self.betas[1],
                             self.eps, self.weight_decay, self.step_count, grad_scale, ss, max_norm or 0.0, self.adamw)
        else:
            ops.adam_step(self.flat_params, self.flat_grads, self.m, self.v, lr, self.betas[0], self.betas[1],
                          self.eps, self.weight_decay, self.step_count, grad_scale)


class FlatAdamW(FlatAdam):
    """The reference's AdamW (modules/optimizer.py:195-292) over the flat bucket."""

    def __init__(self, module, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        super().__init__(module, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, adamw=True)


# ---------------------------------------------------------------------------------------------------------------------
# The reference trainers' optimizers (SGD, SM3, AdamW, Novograd) as torch.optim.Optimizers over one flat bucket
# ---------------------------------------------------------------------------------------------------------------------
TILE_ELEMS, TILE_COLS, TILE_ROWS = 16384, 4096, 1024      # csrc/optim.cu: SM3_COLS, SM3_ROWS


def _tiles(seg_index, shape, numel):
    """Contiguous ranges of one tensor cut from its own shape: whole rows of its last dimension (at most TILE_ROWS rows
    and TILE_ELEMS elements), or pieces of TILE_COLS columns of one row when the last dimension is longer."""
    C = shape[-1] if len(shape) else 1
    if numel == 0:
        return []
    R = numel // C
    out = []
    if C <= TILE_COLS:
        rb = max(1, min(TILE_ROWS, TILE_ELEMS // C))
        for r0 in range(0, R, rb):
            out.append((seg_index, r0 * C, min(rb, R - r0) * C, r0, 0, C))
    else:
        for r in range(R):
            for c0 in range(0, C, TILE_COLS):
                k = min(TILE_COLS, C - c0)
                out.append((seg_index, r * C + c0, k, r, c0, k))
    return out


def bucket_tables(group_shapes):
    """The bucket of tensors given as one list of shapes per parameter group, in order: (seg, tiles, offs, n, nacc).
    seg holds one eb_opt_seg row per tensor (off, numel, rank, group, tile_begin, tile_end, shape[4], acc[4]), tiles
    the eb_opt_tile rows of every tensor in order (``_tiles``), offs each tensor's offset (a multiple of 4), n the
    bucket's length and nacc the length of SM3's accumulator buffer (rank <= 1: one per element, at least one; rank >= 2:
    one per index of every dimension)."""
    seg, tiles, offs, n, nacc = [], [], [], 0, 0
    for gi, shapes in enumerate(group_shapes):
        for shape in shapes:
            i, shape = len(offs), tuple(shape)
            k = math.prod(shape)
            acc = [0, 0, 0, 0]
            if len(shape) <= 1:
                acc[0] = nacc
                nacc += max(k, 1)
            else:
                for d, nd in enumerate(shape):
                    acc[d] = nacc
                    nacc += nd
            t = _tiles(i, shape, k)
            seg.append([n, k, len(shape), gi, len(tiles), len(tiles) + len(t)] + list(shape) +
                       [0] * (4 - len(shape)) + acc)
            tiles.extend(t)
            offs.append(n)
            n += (k + 3) // 4 * 4
    return seg, tiles, offs, n, nacc


class FlatOptimizer(torch.optim.Optimizer):
    """Base of the flat-bucket optimizers: a ``torch.optim.Optimizer`` whose parameters live in one fp32 bucket.

    Construction re-homes every parameter into ``flat_params`` and every gradient into ``flat_grads``, each tensor on a
    16-byte boundary, so ``dist.allreduce_bucket(opt.flat_grads)`` is one call.  The step is a few launches over the
    bucket (csrc/optim.cu); the hyperparameters are read from ``param_groups`` at every step (schedulers and warm-up
    writes to ``param_groups[g]['lr']`` take effect at the next step) and passed by value, with no host-device copy
    and no host sync.

    ``step(closure=None, *, grad_scale=1.0, max_norm=None, check_overflow=False)`` follows ``FlatAdam.step``:
    grad_scale multiplies every gradient, max_norm clips like ``clip_grad_norm_``, and with clipping or overflow checking
    a non-finite norm skips the step.  The norm is summed in a fixed order, so clipped steps are bitwise repeatable.
    The step counters live on the device, one per group, and advance only when the step is taken; a skipped step leaves
    every state unchanged.

    Gradients are never None inside the bucket: a parameter that received no gradient takes a zero-gradient step,
    where the reference classes skip it.

    ``state_dict()`` uses the reference classes' keys and returns compact per-parameter tensors; ``load_state_dict``
    copies into the bucket and accepts what the reference class (or ``torch.optim.SGD``) saved.

    Refused: parameters not on a CUDA device (RuntimeError), tensors of rank > 4, more than 16 groups, a parameter in
    two groups (ValueError), and ``add_param_group`` after construction (RuntimeError: the bucket is fixed).
    """

    _state_keys = ()            # state_dict keys held in the bucket, besides 'step'
    _has_step = True            # the reference class stores state['step']

    def __init__(self, params, defaults):
        self._built = False
        super().__init__(params, defaults)
        ps = [p for g in self.param_groups for p in g["params"]]
        for p in ps:
            if not p.is_cuda:
                raise RuntimeError("%s needs its parameters on a CUDA device (got %s)" % (type(self).__name__, p.device))
        dev = ps[0].device
        if any(p.device != dev for p in ps):
            raise RuntimeError("%s needs every parameter on one device" % type(self).__name__)
        seg, tiles, offs, n, nacc = bucket_tables([[p.shape for p in g["params"]] for g in self.param_groups])
        self.n = n
        self.flat_params = torch.zeros(n, dtype=torch.float32, device=dev)
        self.flat_grads = torch.zeros(n, dtype=torch.float32, device=dev)
        self._params = ps
        self._offs = offs
        self._grad_views = []
        with torch.no_grad():
            for p, off in zip(ps, offs):
                k = p.numel()
                self.flat_params[off:off + k].copy_(p.reshape(-1))
                if p.grad is not None:
                    self.flat_grads[off:off + k].copy_(p.grad.reshape(-1))
                p.data = self.flat_params[off:off + k].view(p.shape)
                gv = self.flat_grads[off:off + k].view(p.shape)
                p.grad = gv
                self._grad_views.append(gv)
        self._grad_ptrs = [gv.data_ptr() for gv in self._grad_views]
        self._seg_host = seg
        self._seg = torch.tensor(seg, dtype=torch.int64).to(dev)
        # a bucket of empty tensors has no tile: step() then runs only the prologue (the sum of squares is 0)
        self._ntiles = len(tiles)
        self._tiles = torch.tensor(tiles, dtype=torch.int64).reshape(-1, 6).to(dev)
        self._nacc = nacc
        self._partial = torch.zeros(len(tiles), dtype=torch.float32, device=dev)
        self._segsum = torch.zeros(len(ps), dtype=torch.float32, device=dev)
        self._total = torch.zeros(1, dtype=torch.float32, device=dev)
        self._ctl = torch.zeros(2, dtype=torch.float32, device=dev)
        self._steps = torch.zeros(len(self.param_groups), dtype=torch.int32, device=dev)
        self._init_state(dev)
        self._built = True

    # -- construction ---------------------------------------------------------------------------------------------
    def add_param_group(self, param_group):
        if getattr(self, "_built", False):
            raise RuntimeError("%s: add_param_group after construction is not supported (the flat bucket is fixed)"
                               % type(self).__name__)
        super().add_param_group(param_group)
        if len(self.param_groups) > _lib.OPT_MAX_GROUPS:
            raise ValueError("%s supports at most %d parameter groups" % (type(self).__name__, _lib.OPT_MAX_GROUPS))
        group = self.param_groups[-1]
        self._check_group(group)
        for p in group["params"]:
            if p.dim() > 4:
                raise ValueError("%s supports tensors of rank <= 4 (got shape %s)" % (type(self).__name__,
                                                                                     tuple(p.shape)))

    def _check_group(self, group):
        """Raise ValueError for an option value the flat kernels do not implement (DESIGN.md §8)."""

    def _refuse(self, option, why):
        raise ValueError("%s: %s is not supported (%s); see DESIGN.md §8" % (type(self).__name__, option, why))

    def _init_state(self, dev):
        raise NotImplementedError

    # -- the step -------------------------------------------------------------------------------------------------
    def _hyper(self, group):
        """(lr, weight decay, b1, b2, eps) of one group."""
        raise NotImplementedError

    def _hyper_struct(self):
        h = _lib.OptHyper()
        for gi, g in enumerate(self.param_groups):
            h.lr[gi], h.wd[gi], h.b1[gi], h.b2[gi], h.eps[gi] = (float(x) for x in self._hyper(g))
        return h

    _needs_segsum = False

    @torch.no_grad()
    def step(self, closure=None, *, grad_scale=1.0, max_norm=None, check_overflow=False):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for p, ptr in zip(self._params, self._grad_ptrs):
            if p.grad is None or p.grad.data_ptr() != ptr:
                raise RuntimeError("parameter gradient left the flat bucket")
        h = self._hyper_struct()
        clip = bool(max_norm) or bool(check_overflow)
        if (clip or self._needs_segsum) and self._ntiles:
            ops.opt_seg_sumsq(self.flat_grads, self._seg, self._tiles, self._partial, self._segsum,
                              self._total if clip else None)
        ops.opt_prologue(self._total if clip else None, grad_scale, max_norm if max_norm else 0.0, self._steps,
                         self._ctl)
        if self._ntiles:
            self._update(h)
        return loss

    def _update(self, h):
        raise NotImplementedError

    def zero_grad(self, set_to_none=True):
        """Zeroes ``flat_grads`` in one memset.  ``set_to_none`` is accepted and ignored: the gradients stay views of
        the bucket (a gradient that autograd replaced is re-homed)."""
        self.flat_grads.zero_()
        for p, gv in zip(self._params, self._grad_views):
            if p.grad is not gv:
                p.grad = gv

    def grad_norm(self):
        """The gradient norm, summed in the same fixed order as the clip."""
        if self._ntiles:
            ops.opt_seg_sumsq(self.flat_grads, self._seg, self._tiles, self._partial, self._segsum, self._total)
        return self._total.sqrt()

    # -- checkpoints ----------------------------------------------------------------------------------------------
    def _views(self, i, group):
        """State key -> view of the bucket-held state of parameter i (in ``group``), in the reference's shape."""
        raise NotImplementedError

    def _extra_state(self):
        return {}

    def state_dict(self):
        steps = self._steps.tolist()
        state, groups, i = {}, [], 0
        for gi, g in enumerate(self.param_groups):
            packed = {k: v for k, v in g.items() if k != "params"}
            packed["params"] = list(range(i, i + len(g["params"])))
            groups.append(packed)
            for _ in g["params"]:
                views = self._views(i, g)
                if steps[gi] > 0 and (views or self._has_step):
                    st = {"step": steps[gi]} if self._has_step else {}
                    st.update(self._extra_state())
                    st.update({k: v.detach().clone() for k, v in views.items()})
                    state[i] = st
                i += 1
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict):
        saved = state_dict["param_groups"]
        if len(saved) != len(self.param_groups):
            raise ValueError("loaded state dict has a different number of parameter groups")
        if any(len(s["params"]) != len(g["params"]) for s, g in zip(saved, self.param_groups)):
            raise ValueError("loaded state dict contains a parameter group that doesn't match the size of "
                             "optimizer's group")
        new_groups = []
        for s, g in zip(saved, self.param_groups):
            ng = dict(self.defaults)
            ng.update({k: v for k, v in s.items() if k != "params"})
            ng["params"] = g["params"]
            self._check_group(ng)
            new_groups.append(ng)
        saved_state = state_dict["state"]
        plan, steps, i = [], [], 0
        for gi, (s, ng) in enumerate(zip(saved, new_groups)):
            t = 0
            for pid in s["params"]:
                st = saved_state.get(pid, {})
                views = self._views(i, ng)
                for k, view in views.items():
                    x = st.get(k)
                    if x is not None:                     # absent (no step taken yet): the state starts at zero
                        x = torch.as_tensor(x)
                        if tuple(x.shape) != tuple(view.shape):
                            raise ValueError("loaded state %r of parameter %d has shape %s, expected %s"
                                             % (k, i, tuple(x.shape), tuple(view.shape)))
                    plan.append((view, x))
                if self._has_step:
                    t = max(t, int(st.get("step", 0)))
                elif any(st.get(k) is not None for k in views):
                    t = 1
                i += 1
            steps.append(t)
        with torch.no_grad():
            for view, x in plan:
                if x is None:
                    view.zero_()
                else:
                    view.copy_(x)
            self._steps.copy_(torch.tensor(steps, dtype=torch.int32))
        for g, ng in zip(self.param_groups, new_groups):
            g.clear()
            g.update(ng)

    def _param_view(self, buf, i):
        p, off = self._params[i], self._offs[i]
        return buf[off:off + p.numel()].view(p.shape)


class SGD(FlatOptimizer):
    """``torch.optim.SGD`` over the flat bucket (cli/train.py:135-140, cli/baseline.py:141-146): d = g + wd p; with
    momentum buf = d on the group's first step and buf = momentum buf + d after it; p -= lr buf.  ``foreach`` and
    ``fused`` are accepted and ignored; dampening != 0, nesterov, maximize and differentiable are refused."""

    _has_step = False

    def __init__(self, params, lr=1e-3, momentum=0, dampening=0, weight_decay=0, nesterov=False, *, maximize=False,
                 foreach=None, differentiable=False, fused=None):
        if lr < 0.0:
            raise ValueError(f"Invalid learning rate: {lr}")
        if momentum < 0.0:
            raise ValueError(f"Invalid momentum value: {momentum}")
        if weight_decay < 0.0:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = dict(lr=lr, momentum=momentum, dampening=dampening, weight_decay=weight_decay, nesterov=nesterov,
                        maximize=maximize, foreach=foreach, differentiable=differentiable, fused=fused)
        self._check_group(defaults)
        super().__init__(params, defaults)

    def _check_group(self, group):
        if group["dampening"] != 0:
            self._refuse("dampening != 0", "no reference caller sets it")
        if group["nesterov"]:
            self._refuse("nesterov=True", "no reference caller sets it")
        if group["maximize"]:
            self._refuse("maximize=True", "no reference caller sets it")
        if group["differentiable"]:
            self._refuse("differentiable=True", "the step runs outside autograd")

    def _init_state(self, dev):
        self.momentum_buffer = None

    def _buf(self):
        if self.momentum_buffer is None:      # allocated once some group has momentum
            self.momentum_buffer = torch.zeros_like(self.flat_params)
        return self.momentum_buffer

    def _hyper(self, group):
        return group["lr"], group["weight_decay"], group["momentum"], 0.0, 0.0

    def _update(self, h):
        buf = self._buf() if any(g["momentum"] != 0 for g in self.param_groups) else None
        ops.opt_sgd_step(self.flat_params, self.flat_grads, buf, self._seg, self._tiles, h, self._steps, self._ctl)

    def _views(self, i, group):
        if group["momentum"] == 0:
            return {}
        return {"momentum_buffer": self._param_view(self._buf(), i)}


class SM3(FlatOptimizer):
    """The reference's SM3 (modules/optimizer.py:4-189) over the flat bucket, momentum = beta = 0: per tensor of rank r
    one accumulator per dimension, u = min_i acc_i + g^2, acc_i = the max of u over every other dimension,
    p -= lr g / sqrt(u + eps).  The accumulators of a rank-2 tensor hold rows + columns floats, not rows x columns.
    momentum > 0 (a full-size buffer, which defeats SM3) and beta > 0 are refused; sparse gradients do not occur."""

    def __init__(self, params, lr=0.1, momentum=0.0, beta=0.0, eps=1e-30):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {0}".format(lr))
        if not 0.0 <= momentum < 1.0:
            raise ValueError("Invalid momentum: {0}".format(momentum))
        if not 0.0 <= beta < 1.0:
            raise ValueError("Invalid beta: {0}".format(beta))
        if not 0.0 <= eps:
            raise ValueError("Invalid eps: {0}".format(eps))
        defaults = {'lr': lr, 'momentum': momentum, 'beta': beta, 'eps': eps}
        self._check_group(defaults)
        super().__init__(params, defaults)

    def _check_group(self, group):
        if group["momentum"] > 0:
            self._refuse("momentum > 0", "it needs a full-size buffer, which defeats SM3")
        if group["beta"] > 0:
            self._refuse("beta > 0", "no reference caller sets it")

    def _init_state(self, dev):
        self._acc = [torch.zeros(self._nacc, dtype=torch.float32, device=dev) for _ in range(2)]
        self._cur = 0

    def _hyper(self, group):
        return group["lr"], 0.0, 0.0, 0.0, group["eps"]

    def _update(self, h):
        ops.opt_sm3_step(self.flat_params, self.flat_grads, self._acc[self._cur], self._acc[1 - self._cur], self._seg,
                         self._tiles, h, self._steps, self._ctl)
        self._cur = 1 - self._cur          # a skipped step copied the accumulators, so the swap is always right

    def _extra_state(self):
        return {"momentum_buffer": 0.}

    def _views(self, i, group):
        acc, row = self._acc[self._cur], self._seg_host[i]
        shape = tuple(self._params[i].shape)
        if len(shape) == 0:
            return {"accumulator_0": acc[row[10]:row[10] + 1].view(())}
        if len(shape) == 1:
            return {"accumulator_0": acc[row[10]:row[10] + shape[0]]}
        r = len(shape)
        return {"accumulator_%d" % d: acc[row[10 + d]:row[10 + d] + n].view([1] * d + [n] + [1] * (r - 1 - d))
                for d, n in enumerate(shape)}


class AdamW(FlatOptimizer):
    """The reference's AdamW (modules/optimizer.py:195-292) over the flat bucket, with parameter groups (wav2vec's
    decay / no-decay split): m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2,
    p -= lr sqrt(bc2)/bc1 (wd p + m / (sqrt(v) + eps)), the bias corrections from the device step counter.
    amsgrad=True is refused."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad)
        self._check_group(defaults)
        super().__init__(params, defaults)

    def _check_group(self, group):
        if group["amsgrad"]:
            self._refuse("amsgrad=True", "no reference caller sets it")

    def _init_state(self, dev):
        self.exp_avg = torch.zeros_like(self.flat_params)
        self.exp_avg_sq = torch.zeros_like(self.flat_params)

    def _hyper(self, group):
        return group["lr"], group["weight_decay"], group["betas"][0], group["betas"][1], group["eps"]

    def _update(self, h):
        ops.opt_adamw_step(self.flat_params, self.flat_grads, self.exp_avg, self.exp_avg_sq, self._seg, self._tiles, h,
                           self._steps, self._ctl)

    def _views(self, i, group):
        return {"exp_avg": self._param_view(self.exp_avg, i), "exp_avg_sq": self._param_view(self.exp_avg_sq, i)}


class Novograd(FlatOptimizer):
    """The reference's Novograd (modules/optimizer.py:294-399) over the flat bucket: per tensor n = sum g^2 (summed in
    a fixed order on the device, with no host sync), v = n on the first nonzero step and b2 v + (1-b2) n after it;
    g' = g / (sqrt(v) + eps) + wd p, m = b1 m + g', p -= lr m.  The reference also divides ``p.grad`` in place; that
    side effect is not reproduced (``flat_grads`` keeps the gradients).  amsgrad=True and grad_averaging=True are
    refused."""

    _needs_segsum = True

    def __init__(self, params, lr=1e-3, betas=(0.95, 0), eps=1e-8, weight_decay=0, grad_averaging=False,
                 amsgrad=False):
        if not 0.0 <= lr:
            raise ValueError("Invalid learning rate: {}".format(lr))
        if not 0.0 <= eps:
            raise ValueError("Invalid epsilon value: {}".format(eps))
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError("Invalid beta parameter at index 0: {}".format(betas[0]))
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError("Invalid beta parameter at index 1: {}".format(betas[1]))
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, grad_averaging=grad_averaging,
                        amsgrad=amsgrad)
        self._check_group(defaults)
        super().__init__(params, defaults)

    def _check_group(self, group):
        if group["amsgrad"]:
            self._refuse("amsgrad=True", "no reference caller sets it")
        if group["grad_averaging"]:
            self._refuse("grad_averaging=True", "no reference caller sets it")

    def _init_state(self, dev):
        self.exp_avg = torch.zeros_like(self.flat_params)
        self.exp_avg_sq = torch.zeros(len(self._params), dtype=torch.float32, device=dev)

    def _hyper(self, group):
        return group["lr"], group["weight_decay"], group["betas"][0], group["betas"][1], group["eps"]

    def _update(self, h):
        ops.opt_novograd_step(self.flat_params, self.flat_grads, self.exp_avg, self.exp_avg_sq, self._segsum,
                              self._seg, self._tiles, h, self._steps, self._ctl)

    def _views(self, i, group):
        return {"exp_avg": self._param_view(self.exp_avg, i), "exp_avg_sq": self.exp_avg_sq[i:i + 1].view(())}
