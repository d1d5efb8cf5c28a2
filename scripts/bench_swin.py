"""Swin on one GPU: training steps of Swin-H/224 through the public API, and the Swin kernels alone next to the eager torch sequence
each replaces (CUDA events, warm-up).
Usage: python scripts/bench_swin.py [--steps N] [--warmup W] [--batch B] [--skip-steps] [--relative-position-bias]
  -> JSON lines on stdout.

  * "card": the GPU's name, power limit and maximum SM clock, read in the same run as the numbers.
  * "kernel": each Swin kernel at Swin-H/224 shapes (micro-batch B): time per call and achieved bytes/s, the bytes being what the
    kernel must read and write (computed from the shapes below), against the data sheet's 3.35 TB/s of HBM3; "eager_ms" is the torch
    sequence the reference runs for the same job (roll + window partition + contiguous; strided slices + cat + LayerNorm; mean).
  * "attention": the window-attention library calls of one step (forward + backward of every block at its stage's shape), timed
    alone, and their share of the step.
  * "step": s/step, images/s, torch peak memory and the peer-memory arena at batch B (no padding tokens when 196 B and 49 B are
    multiples of 8) and at batch B - 1 (stages 2 and 3 then run 200 and 56 tokens), each measured in a process of its own.
  * --relative-position-bias: also the two bias kernels at every stage's shape (bytes: the bf16 mask written / its gradient read),
    the window attention of one step with the bias ("attention_bias": the memory-efficient kernel, the bias gradient included)
    next to the plain one, and the step at batch B without and with the bias, alternated twice."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BF = torch.bfloat16
HBM_TBPS = 3.35
SPEC = "swin-huge-patch4-window7-224"


def timeit(fn, iters=30, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    print(json.dumps({"card": q.stdout.strip() or torch.cuda.get_device_name(0)}), flush=True)


def _emit(name, stage, ms, nbytes, eager_ms=None):
    tbps = nbytes / (ms * 1e-3) / 1e12
    rec = dict(kernel=name, stage=stage, ms=round(ms, 4), bytes=nbytes, TBps=round(tbps, 3), of_hbm=round(tbps / HBM_TBPS, 3))
    if eager_ms is not None:
        rec["eager_ms"] = round(eager_ms, 4)
    print(json.dumps(rec), flush=True)


def kernels(batch, rel_bias=False):
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    from hetu_galvatron_b200.swin import config_from_meta
    from hetu_galvatron_b200.swin.SwinModel_tensor_parallel import WindowLayout
    be = CudaBackend(arena_bytes=64 << 20)
    config = config_from_meta(SPEC)
    attn_ms = attn_bias_ms = 0.0
    for k, st in enumerate(config.stages):
        res, c, heads, ws = st["res"], st["width"], st["heads"], st["window"]
        hn, t = c // heads, st["tokens"]
        lay = WindowLayout(res, ws, st["shift"])
        tmap, inv = lay.maps("cuda")
        x = torch.randn(t, batch, c, device="cuda").to(BF)
        mixed = torch.randn(t * batch, 3 * c, device="cuda").to(BF)
        bias = torch.randn(3 * c, device="cuda").to(BF)
        q, kk, v = be.swin_window_qkv_fwd(mixed, bias, tmap, inv, lay.n_windows, batch, heads, hn)
        act = t * batch * c * 2

        def eager_qkv():                  # the reference: bias add, roll, window partition, contiguous q / k / v
            m = (mixed.view(res, res, batch, 3 * c) + bias)
            m = torch.roll(m, shifts=(-st["shift"], -st["shift"]), dims=(0, 1)) if st["shift"] else m
            m = m.view(res // ws, ws, res // ws, ws, batch, heads, 3, hn).permute(4, 0, 2, 1, 3, 5, 6, 7)
            return [m[..., i, :].reshape(-1, ws * ws, heads, hn).contiguous() for i in range(3)]
        _emit("swin_window_qkv_fwd", k, timeit(lambda: be.swin_window_qkv_fwd(mixed, bias, tmap, inv, lay.n_windows, batch, heads, hn)),
              6 * act, timeit(eager_qkv))
        _emit("swin_window_qkv_bwd", k, timeit(lambda: be.swin_window_qkv_bwd(q, kk, v, tmap, inv, lay.n_windows, batch, t)),
              6 * act + min(be.norm_partials, t * batch) * 3 * c * 4)

        def eager_merge():
            o = q.view(batch, res // ws, res // ws, ws, ws, c).permute(1, 3, 2, 4, 0, 5).reshape(res, res, batch, c)
            o = torch.roll(o, shifts=(st["shift"], st["shift"]), dims=(0, 1)) if st["shift"] else o
            return o.contiguous()
        _emit("swin_window_merge_fwd", k, timeit(lambda: be.swin_window_merge_fwd(q, tmap, inv, lay.n_windows, batch, t)), 2 * act,
              timeit(eager_merge))
        _emit("swin_window_merge_bwd", k, timeit(lambda: be.swin_window_merge_bwd(x, tmap, inv, lay.n_windows, batch, heads, hn)),
              2 * act)
        mask = lay.attn_mask(batch, "cuda", BF)
        qg, kg, vg = [u.detach().requires_grad_(True) for u in (q, kk, v)]

        def attn():
            o = be.attention(qg, kg, vg, False, hn ** -0.5, window_mask=mask) if mask is not None else \
                be.attention(qg, kg, vg, False, hn ** -0.5)
            o.backward(torch.ones_like(o))
        attn_ms += st["depth"] * timeit(attn, iters=10, warm=2)
        if rel_bias:
            index, smask, cells, offsets = lay.rel_maps("cuda")
            table = (0.02 * torch.randn((2 * ws - 1) ** 2, heads, device="cuda")).to(BF)
            rb = be.swin_rel_bias_fwd(table, index, smask, batch, lay.n_windows, ws)
            nbytes = rb.numel() // (ws * ws) * ((ws * ws + 7) // 8 * 8) * 2
            _emit("swin_rel_bias_fwd", k, timeit(lambda: be.swin_rel_bias_fwd(table, index, smask, batch, lay.n_windows, ws)), nbytes)
            _emit("swin_rel_bias_bwd", k, timeit(lambda: be.swin_rel_bias_bwd(rb, cells, offsets, lay.n_windows, ws)), nbytes)
            rbg = rb.detach().requires_grad_(True)

            def attn_bias():
                o = be.attention(qg, kg, vg, False, hn ** -0.5, window_bias=rbg)
                o.backward(torch.ones_like(o))
            attn_bias_ms += st["depth"] * timeit(attn_bias, iters=10, warm=2)
        if k + 1 < len(config.stages):
            w4, b4 = torch.ones(4 * c, device="cuda").to(BF), torch.zeros(4 * c, device="cuda").to(BF)
            to = t // 4
            y, mean, rstd = be.swin_merge_ln_fwd(x, None, w4, b4, 1e-5, batch, res, res, 2, False, to)

            def eager_merge_ln():
                h = x.view(res, res, batch, c)
                cat = torch.cat([h[0::2, 0::2], h[1::2, 0::2], h[0::2, 1::2], h[1::2, 1::2]], dim=-1).view(to, batch, 4 * c)
                return F.layer_norm(cat, (4 * c,), w4, b4, 1e-5)
            _emit("swin_merge_ln_fwd", k, timeit(lambda: be.swin_merge_ln_fwd(x, None, w4, b4, 1e-5, batch, res, res, 2, False, to)),
                  2 * act, timeit(eager_merge_ln))
            _emit("swin_merge_ln_bwd", k, timeit(lambda: be.swin_merge_ln_bwd(y, x, None, w4, mean, rstd, batch, res, res, 2, False)),
                  3 * act)
        if k == 0:
            pb = torch.randn(c, device="cuda").to(BF)
            w1, b1 = torch.ones(c, device="cuda").to(BF), torch.zeros(c, device="cuda").to(BF)
            _emit("swin_merge_ln_fwd_embedding", k, timeit(lambda: be.swin_merge_ln_fwd(mixed[:, :c].contiguous(), pb, w1, b1, 1e-5, batch,
                                                                                         res, res, 1, True, t)), 2 * act)
            res_t = torch.randn_like(x)
            _emit("drop_path_add_fwd", k, timeit(lambda: be.drop_path_add_fwd(x, pb, res_t, 0.1, 1, 0, 4, 0)), 3 * act,
                  timeit(lambda: res_t + (x + pb) * (torch.rand(1, batch, 1, device="cuda") >= 0.1) / 0.9))
            _emit("drop_path_add_bwd", k, timeit(lambda: be.drop_path_add_bwd(x, 0.1, 1, 0, 4, 0, True)), 2 * act)
        if k == len(config.stages) - 1:
            rows = (batch + 7) // 8 * 8
            _emit("swin_mean_pool_fwd", k, timeit(lambda: be.swin_mean_pool_fwd(x, t, rows)), act + rows * c * 2,
                  timeit(lambda: x.mean(0)))
            dy = torch.randn(rows, c, device="cuda").to(BF)
            _emit("swin_mean_pool_bwd", k, timeit(lambda: be.swin_mean_pool_bwd(dy, t, t, batch)), act + rows * c * 2)
    be.close()
    return attn_ms, attn_bias_ms


def steps(batch, n_steps, warmup, rel_bias=False):
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.backend import reset_backend
    from hetu_galvatron_b200.core.runtime.utils import get_optimizer_and_param_scheduler
    from hetu_galvatron_b200.swin import config_from_meta, set_model_config, swin_model_hp
    reset_backend()
    args = sm.tiny_args(global_train_batch_size=batch, chunks=1, default_dp_type="zero2", init_method_std=0.02, lr=1e-4)
    config = set_model_config(config_from_meta(SPEC), args)
    config.relative_position_bias = rel_bias
    model = swin_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    g = torch.Generator(device="cuda").manual_seed(0)
    pixels = torch.randn(batch, 3, 224, 224, device="cuda", generator=g)
    labels = torch.randint(0, 1000, (batch,), device="cuda", generator=g)
    losses = []

    def step(it):
        losses.append(model.forward_backward([pixels], it, None, loss_func=None, labels=labels, attention_mask=None))
        opt.step()
        opt.zero_grad()

    for it in range(warmup):
        step(it)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for it in range(warmup, warmup + n_steps):
        step(it)
    e.record()
    torch.cuda.synchronize()
    sec = s.elapsed_time(e) / 1e3 / n_steps
    rec = dict(step="swin-h/224", relative_position_bias=rel_bias, batch=batch, tokens_run=config.tokens_run, s_per_step=round(sec, 4), images_per_s=round(batch / sec, 1),
               first_loss=round(losses[0], 4), last_loss=round(losses[-1], 4),
               torch_peak_GiB=round(torch.cuda.max_memory_allocated() / 2**30, 1), arena_GiB=round(args.arena_bytes / 2**30, 2))
    print(json.dumps(rec), flush=True)
    del model, opt
    reset_backend()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return sec


def _steps_in_child(batch, n_steps, warmup, rel_bias=False):
    """one step measurement in a process of its own, so that nothing the previous model allocated or cached counts in its memory"""
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--only-steps", "--batch", str(batch), "--steps", str(n_steps),
                          "--warmup", str(warmup)] + (["--relative-position-bias"] if rel_bias else []), capture_output=True, text=True,
                         check=True).stdout
    rec = json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])
    print(json.dumps(rec), flush=True)
    return rec["s_per_step"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--relative-position-bias", action="store_true", help="also measure the model with HF's relative-position bias")
    ap.add_argument("--only-steps", action="store_true", help="(internal) one step measurement at --batch in this process")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_swin.py measures on a GPU"
    if a.only_steps:
        steps(a.batch, a.steps, a.warmup, a.relative_position_bias)
        return
    card()
    attn_ms, attn_bias_ms = kernels(a.batch, a.relative_position_bias)
    torch.cuda.empty_cache()
    if a.skip_steps:
        return
    sec = _steps_in_child(a.batch, a.steps, a.warmup)
    print(json.dumps(dict(attention="window attention fwd + bwd of every block, timed alone", batch=a.batch, ms=round(attn_ms, 2),
                          share_of_step=round(attn_ms / (sec * 1e3), 4))), flush=True)
    if a.relative_position_bias:
        sec_bias = _steps_in_child(a.batch, a.steps, a.warmup, True)
        print(json.dumps(dict(attention_bias="window attention fwd + bwd of every block with the relative-position bias (memory-"
                              "efficient kernel), timed alone", batch=a.batch, ms=round(attn_bias_ms, 2),
                              share_of_step=round(attn_bias_ms / (sec_bias * 1e3), 4))), flush=True)
        _steps_in_child(a.batch, a.steps, a.warmup)
        _steps_in_child(a.batch, a.steps, a.warmup, True)
    _steps_in_child(a.batch - 1, a.steps, a.warmup)


if __name__ == "__main__":
    main()
