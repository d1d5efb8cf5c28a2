"""ViT on one GPU: training steps of ViT-H/16 through the public API, and the four ViT kernels alone (CUDA events, warm-up).
Usage: python scripts/bench_vit.py [--steps N] [--warmup W] [--batch B] [--layers L] [--skip-steps]  -> JSON lines on stdout.

  * "card": the GPU's name, power limit and maximum SM clock, read in the same run as the numbers.
  * "kernel": each ViT kernel at ViT-H/16 shapes (h 1280, 224 px, patch 16, batch B): time per call and achieved bytes/s, the bytes
    being what the kernel must read and write (computed from the shapes below), against the data sheet's 3.35 TB/s of HBM3.
  * "embedding": the embedding row's work in one step at the step's shape (patchify twice, the patch GEMM and its wgrad, the embed
    forward and backward kernels), timed alone.
  * "step": s/step and images/s at batch B (micro-batch B: 197 x B rows, a multiple of 8 when B is, so no padding tokens) and at
    batch B - 1 (the layers then run 200 tokens, 3 of them masked padding), and the time per real token of each."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from hetu_galvatron_b200 import _bg as bg  # noqa: E402

BF = torch.bfloat16
HBM_TBPS = 3.35
H, IMG, PATCH, C, N_PATCHES = 1280, 224, 16, 3, 196


def timeit(fn, iters=50, warm=5):
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


def kernels(batch):
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    be = CudaBackend(arena_bytes=64 << 20)
    s, rows_pad = N_PATCHES + 1, (batch * N_PATCHES + 7) // 8 * 8
    k = PATCH * PATCH * C
    pixels = torch.randn(batch, C, IMG, IMG, device="cuda")
    patch_out = torch.randn(rows_pad, H, device="cuda").to(BF)
    bias, cls, pos = [torch.randn(*sh, device="cuda").to(BF) for sh in ((H,), (H,), (s, H))]
    w = torch.randn(H, k, device="cuda").to(BF)
    pooled = torch.randn((batch + 7) // 8 * 8, H, device="cuda").to(BF)
    dpool = torch.randn_like(pooled)
    out = {}
    for s_run in (s, 200):
        dy = torch.randn(s_run, batch, H, device="cuda").to(BF)
        npart = min(be.norm_partials, N_PATCHES)
        for p in (0.0, 0.1):
            cases = {
                "vit_patchify_fp32": (lambda: be.vit_patchify(pixels, PATCH, rows_pad), pixels.numel() * 4 + rows_pad * k * 2),
                "vit_embed_fwd": (lambda: be.vit_embed_fwd(patch_out, bias, cls, pos, batch, s_run, p, 1, 0, 0, 0),
                                  (batch * N_PATCHES + 2 * s + 1) * H * 2 + s_run * batch * H * 2),
                "vit_embed_bwd": (lambda: be.vit_embed_bwd(dy, N_PATCHES, rows_pad, p, 1, 0, 0, 0),
                                  s * batch * H * 2 + rows_pad * H * 2 + s * H * 4 + npart * H * 4),
                "bias_tanh_fwd": (lambda: be.bias_tanh_fwd(pooled, bias), 2 * pooled.numel() * 2 + H * 2),
                "bias_tanh_bwd": (lambda: be.bias_tanh_bwd(dpool, pooled, bias), 3 * pooled.numel() * 2 + H * 2),
            }
            for name, (fn, nbytes) in cases.items():
                if (name.startswith("vit_embed") or p == 0.0) and (name.startswith("vit_embed") or s_run == s):
                    ms = timeit(fn)
                    tbps = nbytes / (ms * 1e-3) / 1e12
                    rec = dict(kernel=name, batch=batch, h=H, s_run=s_run if name.startswith("vit_embed") else None,
                               dropout=p if name.startswith("vit_embed") else None, ms=round(ms, 4), bytes=nbytes,
                               TBps=round(tbps, 3), of_hbm=round(tbps / HBM_TBPS, 3))
                    print(json.dumps(rec), flush=True)
                    out[(name, s_run, p)] = ms
    # the embedding row of one step at s_run = 197 without dropout: patchify (forward, and again for the wgrad), the patch GEMM,
    # its wgrad, the embed forward and backward
    dy = torch.randn(s, batch, H, device="cuda").to(BF)
    patches = be.vit_patchify(pixels, PATCH, rows_pad)
    dpatch = torch.randn(rows_pad, H, device="cuda").to(BF)
    gemm_ms = timeit(lambda: be.gemm(patches, w, "tn")) + timeit(lambda: be.gemm(dpatch, patches, "nt"))
    emb_ms = 2 * out[("vit_patchify_fp32", s, 0.0)] + gemm_ms + out[("vit_embed_fwd", s, 0.0)] + out[("vit_embed_bwd", s, 0.0)]
    be.close()
    return emb_ms


def steps(batch, n_steps, warmup, layers):
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.backend import reset_backend
    from hetu_galvatron_b200.core.runtime.utils import get_optimizer_and_param_scheduler
    from hetu_galvatron_b200.vit_hf import config_from_meta, set_model_config, vit_model_hp
    reset_backend()
    args = sm.tiny_args(global_train_batch_size=batch, chunks=1, default_dp_type="zero2", init_method_std=0.02, lr=1e-4)
    spec = dict(hidden_size=H, num_hidden_layers=layers, num_attention_heads=16, intermediate_size=4 * H, image_size=IMG,
                patch_size=PATCH, num_channels=C, num_labels=1000)
    config = set_model_config(config_from_meta(spec), args)
    model = vit_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    g = torch.Generator(device="cuda").manual_seed(0)
    pixels = torch.randn(batch, C, IMG, IMG, device="cuda", generator=g)
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
    rec = dict(step="vit-h/16" if layers == 32 else "vit-h/16 x %d layers" % layers, batch=batch, s_run=config.seq_run,
               s_per_step=round(sec, 4), images_per_s=round(batch / sec, 1), us_per_real_token=round(sec / (batch * 197) * 1e6, 4),
               first_loss=round(losses[0], 4), last_loss=round(losses[-1], 4), max_mem_GiB=round(torch.cuda.max_memory_allocated() / 2**30, 1))
    print(json.dumps(rec), flush=True)
    del model, opt
    reset_backend()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return sec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--skip-steps", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vit.py measures on a GPU"
    card()
    emb_ms = kernels(a.batch)
    if a.skip_steps:
        return
    sec = steps(a.batch, a.steps, a.warmup, a.layers)
    print(json.dumps(dict(embedding="row work of one step, timed alone", batch=a.batch, ms=round(emb_ms, 3),
                          share_of_step=round(emb_ms / (sec * 1e3), 4))), flush=True)
    steps(a.batch - 1, a.steps, a.warmup, a.layers)


if __name__ == "__main__":
    main()
