"""T5 on one GPU: training steps of T5-large (24 + 24 layers, d_model 1024, d_ff 4096, 16 heads, encoder and decoder 512 tokens)
through the public API with ZeRO-2 and the fused AdamW, and the cross-attention relayout kernels alone (CUDA events, warm-up).
Usage: python scripts/bench_t5.py [--steps N] [--warmup W] [--batch B]  -> JSON lines on stdout.

  * "card": the GPU's name, power limit and maximum SM clock, read in the same run as the numbers.
  * "kernel": bg_cross_attn_qkv_fwd / _bwd at T5-large shapes (batch B): time per call and achieved bytes/s, the bytes being what the
    kernel must read and write (computed from the shapes below), against the data sheet's 3.35 TB/s of HBM3.
  * "attention": the attention library calls of one step (forward + backward of every encoder self-, decoder self- and decoder
    cross-attention at its shape), timed alone, and their share of the step.
  * "step": s/step, encoder and decoder tokens/s counted separately, torch peak memory and the peer-memory arena, measured in a
    process of its own."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

BF = torch.bfloat16
HBM_TBPS = 3.35
SPEC = "t5-large"


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


def _emit(name, ms, nbytes):
    tbps = nbytes / (ms * 1e-3) / 1e12
    print(json.dumps(dict(kernel=name, ms=round(ms, 4), bytes=nbytes, TBps=round(tbps, 3), of_hbm=round(tbps / HBM_TBPS, 3))), flush=True)


def kernels(batch):
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    from hetu_galvatron_b200.t5 import config_from_meta
    be = CudaBackend(arena_bytes=64 << 20)
    c = config_from_meta(SPEC)
    heads, hn, s_e, s_d, h = c.num_attention_heads, c.d_kv, c.n_positions, c.n_decoder_positions, c.hidden_size
    qm = torch.randn(s_d, batch, heads * hn, device="cuda").to(BF)
    kvm = torch.randn(s_e, batch, 2 * heads * hn, device="cuda").to(BF)
    qb, kvb = torch.randn(heads * hn, device="cuda").to(BF), torch.randn(2 * heads * hn, device="cuda").to(BF)
    q, k, v = be.cross_attn_qkv_fwd(qm, qb, kvm, kvb, heads, hn)
    act = (s_d + 2 * s_e) * batch * heads * hn * 2                       # bf16 elements of q + k + v
    _emit("cross_attn_qkv_fwd", timeit(lambda: be.cross_attn_qkv_fwd(qm, qb, kvm, kvb, heads, hn)), 2 * act + 3 * heads * hn * 2)
    npart = min(be.norm_partials, max(s_e, s_d) * batch)
    _emit("cross_attn_qkv_bwd", timeit(lambda: be.cross_attn_qkv_bwd(q, k, v)), 2 * act + npart * 3 * heads * hn * 4)
    attn_ms = 0.0
    scale = hn ** -0.5
    for n_layers, sq, sk, causal in ((c.num_layers, s_e, s_e, False), (c.num_decoder_layers, s_d, s_d, True),
                                     (c.num_decoder_layers, s_d, s_e, False)):
        qg = torch.randn(batch, sq, heads, hn, device="cuda").to(BF).requires_grad_(True)
        kg, vg = [torch.randn(batch, sk, heads, hn, device="cuda").to(BF).requires_grad_(True) for _ in range(2)]

        def attn():
            o = be.attention(qg, kg, vg, causal, scale)
            o.backward(torch.ones_like(o))
        attn_ms += n_layers * timeit(attn, iters=10, warm=2)
    be.close()
    return attn_ms


def steps(batch, n_steps, warmup):
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.backend import reset_backend
    from hetu_galvatron_b200.core.runtime.utils import get_optimizer_and_param_scheduler
    from hetu_galvatron_b200.t5 import config_from_meta, set_model_config, t5_model_hp
    reset_backend()
    args = sm.tiny_args(global_train_batch_size=batch, chunks=1, default_dp_type="zero2", init_method_std=0.02, lr=1e-4,
                        fused_optimizer=True)
    config = set_model_config(config_from_meta(SPEC), args)
    model = t5_model_hp(config, args)
    opt, _ = get_optimizer_and_param_scheduler(model, args)
    g = torch.Generator(device="cuda").manual_seed(0)
    V, s_e, s_d = config.vocab_size, config.n_positions, config.n_decoder_positions
    enc = torch.randint(0, V, (batch, s_e), device="cuda", generator=g)
    dec = torch.randint(0, V, (batch, s_d), device="cuda", generator=g)
    labels = torch.randint(0, V, (batch, s_d), device="cuda", generator=g)
    losses = []

    def step(it):
        losses.append(model.forward_backward([enc], it, None, loss_func=None, dec_tokens=dec, dec_labels=labels))
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
    rec = dict(step=SPEC, batch=batch, s_per_step=round(sec, 4), encoder_tokens_per_s=round(batch * s_e / sec),
               decoder_tokens_per_s=round(batch * s_d / sec), first_loss=round(losses[0], 4), last_loss=round(losses[-1], 4),
               torch_peak_GiB=round(torch.cuda.max_memory_allocated() / 2**30, 1), arena_GiB=round(args.arena_bytes / 2**30, 2))
    print(json.dumps(rec), flush=True)
    return sec


def _steps_in_child(batch, n_steps, warmup):
    """the step measurement in a process of its own, so that nothing the kernel timings allocated counts in its memory"""
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--only-steps", "--batch", str(batch), "--steps", str(n_steps),
                          "--warmup", str(warmup)], capture_output=True, text=True, check=True).stdout
    rec = json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])
    print(json.dumps(rec), flush=True)
    return rec["s_per_step"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--only-steps", action="store_true", help="(internal) the step measurement in this process")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_t5.py measures on a GPU"
    if a.only_steps:
        steps(a.batch, a.steps, a.warmup)
        return
    card()
    attn_ms = kernels(a.batch)
    torch.cuda.empty_cache()
    sec = _steps_in_child(a.batch, a.steps, a.warmup)
    print(json.dumps(dict(attention="encoder self-, decoder self- and cross-attention fwd + bwd of every layer, timed alone",
                          batch=a.batch, ms=round(attn_ms, 2), share_of_step=round(attn_ms / (sec * 1e3), 4))), flush=True)


if __name__ == "__main__":
    main()
