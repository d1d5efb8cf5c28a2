"""Optimizer / grad-norm helpers of ``galvatron/core/runtime/utils.py`` (:124-167).

The optimizer itself is out of the hot-path scope (SURVEY 2.1 row 9: "keep torch/apex"): apex ``FusedAdam`` (AdamW mode)
becomes ``torch.optim.AdamW(fused=True)`` over the fp32 flat shards the sharded units expose.
"""
import math

import torch


class FusedShardedAdamW(torch.optim.Optimizer):
    """AdamW whose update runs inside each layer's gradient reduce-scatter kernel (SURVEY 8f-3): when a layer's last
    backward of the step finishes, ONE kernel pulls the peers' gradient slices, sums them and applies the AdamW step to
    the fp32 shard -- the fp32 gradient buffer is never materialised (30 GiB less at Llama-3-8B on one GPU) and the
    optimizer's own pass over the state disappears.  ``step()`` only advances the step counter and fences the reduce
    stream; hyper-parameters take effect for the NEXT forward_backward.  Same rule as torch.optim.AdamW.

    ``clip_grad`` > 0 (Megatron's ``--clip-grad``) defers the update so that ``clip_grad_norm`` can scale it by the job-wide
    gradient norm, still without an fp32 gradient buffer: the layer's reduction at the end of its backward becomes a norm pass
    (the same reduce-scatter, whose epilogue only writes per-warp sums of squares of the reduced gradient), and ``step()``
    re-runs the AdamW reduce-scatter over the untouched unsharded gradient with the clip coefficient, a device scalar that
    ``clip_grad_norm`` sets and ``step()`` resets to 1.  Pooled zero3 units hand their gradient buffer back after the
    reduction: their norm pass also writes the fp32 gradient shard, and ``step()`` applies the same clipped rule to it."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, clip_grad=0.0):
        params = list(model.parameters())
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self.units = list(model.model.units)
        self.step_count = 0
        self._fallback = None
        self.deferred = clip_grad > 0
        plain = []
        for u in self.units:
            u.fused_opt = self
            if u.uses_fused_optimizer():
                u.exp_avg = torch.zeros_like(u.flat_param.data)
                u.exp_avg_sq = torch.zeros_like(u.flat_param.data)
            else:
                plain.append(u.flat_param)
        if self.deferred:
            from .backend import get_backend
            be = get_backend()
            self.partials = be.clip_partials(len(self.units))      # row i: unit i's sums of squares of this step
            self.clip_coef = torch.ones((), dtype=torch.float32, device=self.partials.device)
            self._row = {id(u): i for i, u in enumerate(self.units)}
            self._skip = {id(u): _shard_skip_ranges(u, be.rank) for u in self.units if u.uses_fused_optimizer()}
            self._stepping = []         # units whose norm pass ran this step, in reduction order: their step passes
        if plain:   # replicated DDP layers: ordinary AdamW on their fp32 gradients
            g = self.param_groups[0]
            self._fallback = torch.optim.AdamW(plain, lr=g["lr"], betas=g["betas"], eps=g["eps"], weight_decay=g["weight_decay"],
                                               fused=all(p.is_cuda for p in plain))

    def hyper(self):
        g = self.param_groups[0]
        return g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self.step_count + 1

    def norm_pass(self, unit):
        """Deferred clipping: the unit's reduction at the end of its backward (called by ``ShardedUnit.reduce_now``)."""
        unit.be.unit_reduce_sumsq(unit, self.partials[self._row[id(unit)]], self._skip[id(unit)], into_master=unit.g_pool is not None)
        self._stepping.append(unit)

    def sum_of_squares(self):
        """Device scalar: the sum of squares of this rank's share of the fused units' gradients, as the next update will see
        them (scaled by the clip coefficient set so far)."""
        return self.partials.sum() * self.clip_coef * self.clip_coef

    @torch.no_grad()
    def step(self, closure=None):
        from .backend import get_backend
        be = get_backend()
        be.finish_reductions()
        if self.deferred:
            # the step passes, in the order of the norm passes (the same on every member of each group: they are collectives)
            for u in self._stepping:
                if u.g_pool is not None:
                    be.unit_adamw_clipped(u, self, self.clip_coef)
                else:
                    be.unit_reduce_adamw(u, self, clip_coef=self.clip_coef)
                    u._reduce_event = be.reduce_done_event()      # the next backward may overwrite G only after this read
            self._stepping = []
            be.finish_reductions()
            self.partials.zero_()
            self.clip_coef.fill_(1.0)
        if self._fallback is not None:
            for gsrc, gdst in zip(self.param_groups, self._fallback.param_groups):
                gdst["lr"] = gsrc["lr"]
            self._fallback.step()
        self.step_count += 1

    def zero_grad(self, set_to_none=True):
        if self._fallback is not None:
            self._fallback.zero_grad(set_to_none)

    def state_dict(self):
        """Per-rank optimizer state (what ``optimizer/<rank>.pt`` of a distributed checkpoint holds): the moments live on the
        sharded units, next to the fp32 shard the reduce-scatter epilogue updates."""
        return {"fused_sharded_adamw": 1, "step_count": self.step_count,
                "param_groups": [{k: v for k, v in g.items() if k != "params"} for g in self.param_groups],
                "units": {u.name: {"exp_avg": u.exp_avg.detach().cpu(), "exp_avg_sq": u.exp_avg_sq.detach().cpu()}
                          for u in self.units if u.uses_fused_optimizer()},
                "fallback": None if self._fallback is None else self._fallback.state_dict()}

    def load_state_dict(self, state):
        if not state.get("fused_sharded_adamw"):
            raise ValueError("not a FusedShardedAdamW state (saved with --optimizer torch?)")
        self.step_count = int(state["step_count"])
        for g, saved in zip(self.param_groups, state["param_groups"]):
            g.update(saved)
        for u in self.units:
            if u.uses_fused_optimizer():
                rec = state["units"][u.name]
                u.exp_avg.copy_(rec["exp_avg"])
                u.exp_avg_sq.copy_(rec["exp_avg_sq"])
        if self._fallback is not None and state.get("fallback") is not None:
            self._fallback.load_state_dict(state["fallback"])


class OptimizerParamScheduler:
    """LR warm-up / decay and weight-decay ramp with the semantics and the ``state_dict`` keys of Megatron's scheduler
    (``megatron/training/optimizer_param_scheduler.py:9-229``, built by ``training.py:434-480`` and used by
    ``galvatron/core/runtime/utils.py:151``), so ``opt_param_scheduler.json`` moves between the two runtimes unchanged.
    Pinned to the reference class by tests/golden/opt_param_scheduler.json (oracle/gen_golden_sched.py).

    ``step(increment)`` advances by ``increment`` samples (the reference steps by the global batch size) and writes ``lr`` and
    ``weight_decay`` into every param group (scaled by the group's ``lr_mult`` / ``wd_mult``).  Schedule, with n = steps so far:
      n <= warmup (warmup > 0):  init_lr + (max_lr - init_lr) * n / warmup
      constant:                  max_lr
      n > decay_steps:           min_lr
      inverse-square-root:       max(min_lr, max_lr * sqrt(max(warmup, 1)) / sqrt(max(n, 1)))
      linear / cosine:           min_lr + c * (max_lr - min_lr),  r = (n - warmup) / (decay_steps - warmup),
                                 c = 1 - r  /  (cos(pi r) + 1) / 2
    weight decay: end_wd beyond wd_incr_steps; constant; linear r; cosine (cos(pi (1 - r)) + 1) / 2 between start_wd and end_wd."""

    _LR_COEFF = {"linear": lambda r: 1.0 - r, "cosine": lambda r: 0.5 * (math.cos(math.pi * r) + 1.0)}
    _WD_COEFF = {"linear": lambda r: r, "cosine": lambda r: 0.5 * (math.cos(math.pi * (1.0 - r)) + 1.0)}
    _STATE = ("max_lr", "lr_warmup_steps", "num_steps", "lr_decay_style", "lr_decay_steps", "min_lr", "start_wd", "end_wd",
              "wd_incr_style", "wd_incr_steps")
    # older checkpoints name some fields differently (optimizer_param_scheduler.py:176-212)
    _ALIASES = {"max_lr": ("start_lr",), "lr_warmup_steps": ("warmup_iter", "warmup_steps"), "lr_decay_steps": ("end_iter", "decay_steps"),
                "lr_decay_style": ("decay_style",), "num_steps": ("num_iters",)}

    def __init__(self, optimizer, init_lr, max_lr, min_lr, lr_warmup_steps, lr_decay_steps, lr_decay_style, start_wd, end_wd,
                 wd_incr_steps, wd_incr_style, use_checkpoint_opt_param_scheduler=True, override_opt_param_scheduler=False):
        if not (0.0 <= min_lr <= float(max_lr) and init_lr <= float(max_lr)):
            raise ValueError("need 0 <= min_lr <= max_lr and init_lr <= max_lr")
        if not (lr_decay_steps > 0 and lr_warmup_steps < lr_decay_steps):
            raise ValueError("need 0 <= lr_warmup_steps < lr_decay_steps")
        if not 0.0 <= start_wd <= end_wd:
            raise ValueError("need 0 <= start_wd <= end_wd")
        if override_opt_param_scheduler and use_checkpoint_opt_param_scheduler:
            raise ValueError("both override and use-checkpoint are set.")
        self.optimizer = optimizer
        self.init_lr, self.max_lr, self.min_lr = init_lr, float(max_lr), min_lr
        self.lr_warmup_steps, self.lr_decay_steps, self.lr_decay_style = lr_warmup_steps, lr_decay_steps, lr_decay_style
        self.start_wd, self.end_wd, self.wd_incr_steps, self.wd_incr_style = start_wd, end_wd, wd_incr_steps, wd_incr_style
        self.use_checkpoint, self.override = use_checkpoint_opt_param_scheduler, override_opt_param_scheduler
        self.num_steps = 0
        self.step(0)

    def get_wd(self):
        if self.num_steps > self.wd_incr_steps:
            return self.end_wd
        if self.wd_incr_style == "constant":
            if self.start_wd != self.end_wd:
                raise ValueError("constant weight decay needs start_wd == end_wd")
            return self.end_wd
        if self.wd_incr_style not in self._WD_COEFF:
            raise ValueError("{} weight decay increment style is not supported.".format(self.wd_incr_style))
        ratio = float(self.num_steps) / float(self.wd_incr_steps)
        return self.start_wd + self._WD_COEFF[self.wd_incr_style](ratio) * (self.end_wd - self.start_wd)

    def get_lr(self, param_group=None):
        group = param_group or {}
        max_lr, min_lr, n = group.get("max_lr", self.max_lr), group.get("min_lr", self.min_lr), self.num_steps
        if self.lr_warmup_steps > 0 and n <= self.lr_warmup_steps:
            return self.init_lr + (max_lr - self.init_lr) * float(n) / float(self.lr_warmup_steps)
        if self.lr_decay_style == "constant":
            return max_lr
        if n > self.lr_decay_steps:
            return min_lr
        if self.lr_decay_style == "inverse-square-root":
            return max(min_lr, max_lr * max(self.lr_warmup_steps, 1) ** 0.5 / (max(n, 1) ** 0.5))
        if self.lr_decay_style not in self._LR_COEFF:
            raise ValueError("{} decay style is not supported.".format(self.lr_decay_style))
        ratio = float(n - self.lr_warmup_steps) / float(self.lr_decay_steps - self.lr_warmup_steps)
        return min_lr + self._LR_COEFF[self.lr_decay_style](ratio) * (max_lr - min_lr)

    def step(self, increment=1):
        self.num_steps += increment
        wd = self.get_wd()
        for group in self.optimizer.param_groups:
            group["lr"] = self.get_lr(group) * group.get("lr_mult", 1.0)
            group["weight_decay"] = wd * group.get("wd_mult", 1.0)

    def state_dict(self):
        return {k: getattr(self, k) for k in self._STATE}

    def load_state_dict(self, sd):
        if "lr_lambdas" in sd or "_last_lr" in sd:
            raise ValueError("this is a torch LambdaLR state (written by round 1 of this runtime), not an OptimizerParamScheduler state")

        def pick(name):
            for key in self._ALIASES.get(name, ()) + (name,):
                if key in sd:
                    return sd[key]
            raise KeyError("opt_param_scheduler state lacks %r" % name)

        def settle(name):
            mine, saved = getattr(self, name), pick(name)
            if self.override:
                return mine
            if not self.use_checkpoint and mine != saved:
                raise ValueError("OptimizerParamScheduler: class input value %r and checkpoint value %r for %s do not match" % (mine, saved, name))
            return saved

        for name in ("max_lr", "min_lr", "lr_warmup_steps", "lr_decay_steps", "lr_decay_style"):
            setattr(self, name, settle(name))
        self.step(increment=pick("num_steps"))
        if "start_wd" in sd:
            for name in ("start_wd", "end_wd", "wd_incr_steps", "wd_incr_style"):
                setattr(self, name, settle(name))


def get_optimizer_param_scheduler(optimizer, args):
    """``training.py:434-480``: iteration-based (``train_iters``) or sample-based (``train_samples``) schedule lengths; without
    either -- the random-data scripts of this runtime pass neither -- a constant schedule at ``args.lr`` / ``args.adam_weight_decay``."""
    gbs = args.global_train_batch_size
    style = getattr(args, "lr_decay_style", None)
    if getattr(args, "train_iters", None):
        decay_iters = getattr(args, "lr_decay_iters", None) or args.train_iters
        decay, wd_steps = decay_iters * gbs, args.train_iters * gbs
        frac = getattr(args, "lr_warmup_fraction", None)
        warmup = frac * decay if frac is not None else getattr(args, "lr_warmup_iters", 0) * gbs
        style = style or "linear"
    elif getattr(args, "train_samples", None):
        decay = getattr(args, "lr_decay_samples", None) or args.train_samples
        wd_steps = args.train_samples
        frac = getattr(args, "lr_warmup_fraction", None)
        warmup = frac * decay if frac is not None else getattr(args, "lr_warmup_samples", 0)
        style = style or "linear"
    else:
        decay, wd_steps, warmup, style = 1, 1, 0, "constant"
    wd = args.adam_weight_decay
    start_wd, end_wd = getattr(args, "start_weight_decay", None), getattr(args, "end_weight_decay", None)
    return OptimizerParamScheduler(
        optimizer, init_lr=getattr(args, "lr_warmup_init", 0.0), max_lr=args.lr, min_lr=getattr(args, "min_lr", 0.0),
        lr_warmup_steps=warmup, lr_decay_steps=decay, lr_decay_style=style, start_wd=wd if start_wd is None else start_wd,
        end_wd=wd if end_wd is None else end_wd, wd_incr_steps=wd_steps, wd_incr_style=getattr(args, "weight_decay_incr_style", "constant"),
        use_checkpoint_opt_param_scheduler=getattr(args, "use_checkpoint_opt_param_scheduler", True),
        override_opt_param_scheduler=getattr(args, "override_opt_param_scheduler", False))


def get_optimizer_and_param_scheduler(model, args):
    """``core/runtime/utils.py:140-167``: AdamW over the fp32 flat shards + Megatron's LR / weight-decay scheduler; with
    ``--distributed_checkpoint`` both resume from ``<load>/iter_<load_iteration>/{optimizer/<rank>.pt, opt_param_scheduler.json}``
    (:152-165) -- and, as in the reference, a missing file is an error, not a silent fresh start."""
    if getattr(args, "fused_optimizer", False):
        optimizer = FusedShardedAdamW(model, lr=args.lr, betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)),
                                      eps=getattr(args, "adam_eps", 1e-8), weight_decay=args.adam_weight_decay,
                                      clip_grad=float(getattr(args, "clip_grad", 0.0) or 0.0))
    else:
        params = list(model.parameters())
        optimizer = torch.optim.AdamW(params, lr=args.lr, weight_decay=args.adam_weight_decay,
                                      betas=(getattr(args, "adam_beta1", 0.9), getattr(args, "adam_beta2", 0.999)),
                                      eps=getattr(args, "adam_eps", 1e-8), fused=all(p.is_cuda for p in params))
    scheduler = get_optimizer_param_scheduler(optimizer, args)
    if getattr(args, "distributed_checkpoint", False) and getattr(args, "load", None):
        import json
        import os
        from .backend import get_backend
        root = os.path.join(args.load, "iter_%d" % int(getattr(args, "load_iteration", 0)))
        opt_file = os.path.join(root, "optimizer", "%d.pt" % get_backend().rank)
        sched_file = os.path.join(root, "opt_param_scheduler.json")
        for path in (opt_file, sched_file):
            if not os.path.exists(path):
                raise FileNotFoundError("--distributed_checkpoint: %s is missing (the checkpoint holds no optimizer / scheduler state "
                                        "for this rank)" % path)
        state = torch.load(opt_file, map_location="cpu", weights_only=True)
        if isinstance(optimizer, FusedShardedAdamW) != bool(isinstance(state, dict) and state.get("fused_sharded_adamw")):
            raise ValueError("%s was written by a different optimizer layout (fused_sharded_adamw=%s); per-rank optimizer state of a "
                             "reference-written checkpoint (apex FusedAdam over FSDP flat parameters) cannot be re-sharded here: load "
                             "the weights without --distributed_checkpoint's optimizer state, or save with this runtime"
                             % (opt_file, bool(isinstance(state, dict) and state.get("fused_sharded_adamw"))))
        optimizer.load_state_dict(state)
        with open(sched_file) as f:
            saved = json.load(f)
        if saved:
            scheduler.load_state_dict(saved)
    return optimizer, scheduler


def _tp_replicated_ranges(unit):
    """[(offset, numel)] inside the unit's flat buffer of the parameters that every rank of the unit's tensor-parallel group
    holds in full (norm weights, the row-parallel bias): Megatron counts those once (``param_is_not_tensor_parallel_duplicate``,
    clip_grads.py:61-75); parameters marked ``tensor_model_parallel`` (column / row / vocabulary-parallel weights, the
    column-parallel bias; layers.py:95-105) are a different slice on every tensor-parallel rank."""
    return [(off, n) for p, off, n in zip(unit.params, unit.offsets, unit.numels) if not getattr(p, "tensor_model_parallel", False)]


def _shard_skip_ranges(unit, rank):
    """Shard-relative [lo, hi) element ranges of a fused unit's gradient that this rank must leave out of the global norm: the
    tensor-parallel duplicates (``_tp_replicated_ranges``) on tensor-parallel ranks other than 0, rounded out to the 8-element
    parameter alignment (the padding between parameters holds zero gradients) and merged where they touch."""
    tp = unit.tp_group
    if tp is None or tp.size == 1 or tp.rank_in_group(rank) == 0:
        return []
    lo = unit.rank_in_group * unit.shard_elems         # this rank's window of the flat buffer
    hi = lo + unit.shard_elems
    out = []
    for off, n in _tp_replicated_ranges(unit):
        a, b = max(off, lo), min((off + n + 7) // 8 * 8, hi)
        if a >= b:
            continue
        if out and out[-1][1] == a - lo:
            out[-1] = (out[-1][0], b - lo)
        else:
            out.append((a - lo, b - lo))
    return out


def clip_grad_norm(model, max_norm, norm_type=2):
    """Global L2 norm of the gradients over the job, then scale them by min(1, max_norm / (norm + 1e-6))
    (utils.py:124-133 -> megatron ``clip_grad_norm_fp32``, clip_grads.py:47-132).  Every parameter is counted exactly once:
      * a sharded unit's fp32 gradient shards partition its flat parameter over the SDP group;
      * a replicated (DDP) unit holds the same reduced gradient on every member: divided by the group size;
      * tensor-parallel ranks hold different slices of the parallel weights, but the SAME norm weights / row-parallel bias
        (after the sequence-parallel gradient all-reduce): those are counted on tensor-parallel rank 0 only.
    Every rank enters the world all-reduce, whether or not it holds gradients.  With ``--fused_optimizer`` the gradient is consumed
    inside the reduce-scatter kernel and there is nothing left to clip, unless the optimizer was built with ``clip_grad`` > 0: the
    fused units' squares then come from the norm passes, and the coefficient is stored on the device for ``step()`` (a second
    call multiplies it, as scaling the gradients twice does)."""
    from .backend import get_backend
    if norm_type != 2:
        raise ValueError("clip_grad_norm: only the L2 norm is implemented")
    be = get_backend()
    units = list(model.model.units)
    fused = next((u.fused_opt for u in units if u.uses_fused_optimizer()), None)
    if fused is not None and not fused.deferred:
        raise RuntimeError("clip_grad_norm cannot be combined with --fused_optimizer unless clip_grad > 0: the AdamW step runs inside "
                           "the gradient reduce-scatter kernel, no gradient tensor survives it (set args.clip_grad to defer the "
                           "update until the norm is known, or use the unfused optimizer to clip)")
    device = units[0].flat_param.device if units else be.device
    total = torch.zeros((), dtype=torch.float32, device=device)
    if fused is not None:
        be.finish_reductions()          # the norm passes have written their partial sums
        total = total + fused.sum_of_squares()
    grads = []
    for u in units:
        g = u.flat_param.grad
        if g is None:
            continue
        grads.append(g)
        gf = g.float()
        sq = gf.pow(2).sum()
        if u.tp_group is not None and u.tp_group.size > 1 and u.tp_group.rank_in_group(be.rank) != 0:
            lo = 0 if u.dp_type == "ddp" else u.rank_in_group * u.shard_elems       # this rank's window of the flat buffer
            hi = lo + gf.numel()
            for off, n in _tp_replicated_ranges(u):
                a, b = max(off, lo), min(off + n, hi)
                if a < b:
                    sq = sq - gf[a - lo:b - lo].pow(2).sum()
        if u.dp_type == "ddp":
            sq = sq / u.group.size
        total = total + sq
    buf = torch.zeros(8, dtype=torch.float32, device=device)
    buf[0] = total
    if be.world > 1:
        if be.world_group is None:
            raise RuntimeError("clip_grad_norm over %d ranks needs the world group reserved at model construction "
                               "(construct_hybrid_parallel_model_api does it; worlds beyond one NVSwitch domain are out of scope)" % be.world)
        buf = be.all_reduce(buf, be.world_group)
    norm = buf[0].sqrt()
    coef = (max_norm / (norm + 1e-6)).clamp(max=1.0)
    for g in grads:
        g.mul_(coef.to(g.dtype))
    if fused is not None:
        fused.clip_coef.mul_(coef)
    return float(norm)
