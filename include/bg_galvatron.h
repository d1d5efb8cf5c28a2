/*
 * bg_galvatron.h -- C ABI of the H100-native hot path behind Hetu-Galvatron's per-layer strategy API.
 *
 * The reference (PKU-DAIR/Hetu-Galvatron v2.4.1) has no FFI at this seam: every per-layer collective is a
 * torch.distributed (ProcessGroupNCCL) call made from Python.  Each entry point below names the reference
 * call site it replaces (file:line under /root/reference unless prefixed torch/).  The host side that binds
 * these (ctypes) is hetu-galvatron_b200/_bg.py; INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions: plain pointers and sizes, no torch types; every call returns 0 on success or a negative
 * BG_E* code (message via bg_last_error()); nothing throws across the ABI.  All device work is asynchronous
 * on the cudaStream_t passed as `stream` (void*).  One bg_ctx per rank (one process per GPU; several ctx in
 * one process = "virtual ranks" on one device, used by the single-GPU parity tests).  Thread-compatible:
 * callable from the main and the autograd thread; per-(group,lane) ordering is the caller's stream order.
 *
 * Peer memory model: each rank owns ONE symmetric arena (cudaMalloc, exported with cudaIpcGetMemHandle,
 * mapped by its peers once).  A "symmetric buffer" is an array of per-member arena offsets (group order).
 * Cross-rank synchronisation is device-side: per-(group,lane,CTA) flags in the arena head, CAS put/wait
 * with release/acquire at .sys scope; no host sync, no NCCL on these paths.
 */
#ifndef BG_GALVATRON_H
#define BG_GALVATRON_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BG_ABI_VERSION 1
#define BG_MAX_PEERS 8      /* one NVSwitch domain */
#define BG_MAX_WORLD 64
#define BG_LANES 6          /* independent barrier lanes per group: unshard / grad-reduce / activations / misc / fused-op push / cp ring */
#define BG_MAX_CHANNELS 256 /* max CTAs of a cross-rank kernel (one barrier channel per CTA; the default is one slim CTA per SM) */

typedef struct bg_ctx* bg_ctx_t;

enum bg_dtype { BG_BF16 = 0, BG_F32 = 1 };
enum bg_redop { BG_SUM = 0, BG_MAX = 1 };
enum bg_err {
    BG_OK = 0, BG_EINVAL = -1, BG_ECUDA = -2, BG_ENOMEM = -3, BG_ENOTMAPPED = -4, BG_EGROUP = -5, BG_ETIMEOUT = -6,
    BG_EUNSUPPORTED = -7
};

/* ---- library ------------------------------------------------------------------------------------------ */
int bg_abi_version(void);
const char* bg_last_error(void);                       /* thread-local message of the last failing call */
/* "comm_ctas" (CTAs of a cross-rank kernel, default 132 = one 128-thread / <=64-register CTA per SM), "local_ctas", "timeout_ms",
 * "oneshot_bytes", "nvls_min_bytes" (multicast paths above this size), "nvls_min_ranks" (... and from this group size on), "nvls_gather" [0] / "nvls_reduce" [1]
 * (multimem.st for all-gather / multimem.ld_reduce for reduce-scatter on multicast-bound buffers; defaults from the p = 8 measurement),
 * "nvls_bcast" [1] (the fused GEMM + all-reduce writes a reduced tile to every member with one multimem.st) */
int bg_set_tunable(const char* name, long long value);
long long bg_get_tunable(const char* name);
/* how many kernels this library has launched since load (bench.py's gpu_launches) */
unsigned long long bg_launch_count(void);

/* ---- context + symmetric arena (replaces ProcessGroupNCCL communicator state) --------------------------- */
int bg_ctx_create(int rank, int world, int device, size_t arena_bytes, bg_ctx_t* out);
/* flags: BG_CTX_VMM allocates the arena with the virtual-memory API (cuMemCreate) instead of cudaMalloc; that is what NVSwitch
 * multicast objects can bind.  Such an arena is shared between processes as a POSIX file descriptor (bg_arena_export_fd /
 * bg_arena_import_fd; the host passes the descriptor over a unix socket) instead of a cudaIpc handle.  OPT-IN. */
#define BG_CTX_VMM 1u
int bg_ctx_create_ex(int rank, int world, int device, size_t arena_bytes, unsigned flags, bg_ctx_t* out);
int bg_ctx_destroy(bg_ctx_t ctx);
int bg_arena_info(bg_ctx_t ctx, void** base, size_t* bytes, size_t* used);
int bg_arena_alloc(bg_ctx_t ctx, size_t bytes, size_t* offset);        /* 256-B aligned bump allocation */
int bg_arena_export(bg_ctx_t ctx, void* handle64);                      /* cudaIpcMemHandle_t, 64 bytes */
int bg_arena_import(bg_ctx_t ctx, int peer_rank, const void* handle64); /* map a peer process's arena */
int bg_arena_attach_local(bg_ctx_t ctx, int peer_rank, bg_ctx_t peer);  /* peer ctx in this process */
int bg_arena_alloc_aligned(bg_ctx_t ctx, size_t bytes, size_t align, size_t* offset);
int bg_arena_mode(bg_ctx_t ctx, int* vmm, int* multicast_supported, size_t* multicast_granularity);
int bg_arena_export_fd(bg_ctx_t ctx, int* fd);                          /* BG_CTX_VMM arenas */
int bg_arena_import_fd(bg_ctx_t ctx, int peer_rank, int fd);
int bg_ctx_error_flag(bg_ctx_t ctx, int* flag);                         /* device-side timeout report */
/* info8[0] = status; [1] = kind (1 signalling a peer, 2 waiting for a peer, 3 fused-GEMM tile reducer);
 * [2] = CTA; [3] = thread or tile; [4] = value last seen; [5], [6] = group index/size or expected count/tiles;
 * [7] = launch site of a barrier timeout (1 all-gather, 2 reduce-scatter, 3 all-reduce, 6 all-to-all, 7 entry barrier of a fused
 * GEMM, 8 exit barrier of the all-reduce tile reducer, 10/11 p2p flags, 12 push kernel of the fused all-gather+GEMM, 13 cp ring
 * K/V push, 14 cp ring wait, 15 cp ring release, 16 cp ring accumulate-and-forward push, 17 in-place pair sum), kind 4 = the
 * gathering GEMM's TMA producer waiting for a block.
 * The reference's analogue is the NCCL watchdog's timeout dump (ProcessGroupNCCL); here a lost peer traps the
 * kernel and leaves this record in mapped host memory. */
int bg_ctx_error_info(bg_ctx_t ctx, int* info8);

/* ---- groups (galvatron/core/runtime/comm_groups.py:7-29 CommGroup / :416 gen_comm_groups) ---------------- */
/* A group is its rank list; creation is O(1), local, and needs no collective (the reference pays one
 * torch.distributed.new_group per group on all ranks, comm_groups.py:14).  Rank lists must be arithmetic
 * progressions (every Galvatron group is). */
int bg_group_create(bg_ctx_t ctx, const int* ranks, int n, int* gid);
int bg_group_info(bg_ctx_t ctx, int gid, int* n, int* my_index, int* ranks_out /* BG_MAX_PEERS */);
/* C mirror of gen_comm_groups for one rank: for each of the n_layers whole-model rows writes the caller's
 * tp/sp/cp/dp/sdp rank lists as (count, ranks[BG_MAX_WORLD]) records; used by the bit-exact mapping test. */
int bg_build_groups(int rank, int world, int pp_size, int n_layers, const int* tp, const int* sp, const int* cp,
                    int* out_counts /* [5][n_layers] */, int* out_ranks /* [5][n_layers][BG_MAX_WORLD] */,
                    int* pp_count, int* pp_ranks /* [BG_MAX_WORLD] */);

/* ---- collectives ----------------------------------------------------------------------------------------- */
/* device-side barrier over the group (replaces torch.distributed.barrier, pipeline.py:370,698,882) */
int bg_barrier(bg_ctx_t ctx, int gid, int lane, void* stream);

/* C1  param all-gather fused with the fp32->bf16 cast.
 * Replaces torch/distributed/fsdp/_flat_param.py:1477 all_gather_into_tensor (+ the MixedPrecision shard cast,
 * galvatron/core/runtime/parallel.py:116-122); also the plain activation all-gathers mappings_group.py:100,
 * layers.py:410-412, redistribute.py:65,110 when src_dtype == dst_dtype.
 * Push: every member casts its shard once and stores it into slot `my_index` of every member's dst.
 *
 * Errors of the plain collectives (this entry, bg_reduce_scatter_acc, bg_all_reduce, bg_pair_sum_inplace, bg_all_to_all_rows),
 * in this order: first the checks that need no context (dtypes, whole 16-B vectors, local pointer alignment, descriptor fields),
 * then a null ctx or a bad lane (BG_EINVAL; a bad gid is BG_EGROUP), then the group's checks, then the symmetric offsets (BG_EINVAL
 * for one that is not 16-B aligned or a buffer that does not lie inside the arena -- compared without overflow, so an element
 * count too large for the arena is refused however large it is).  A call that fails has launched nothing, on this member or for
 * its peers.
 * Here: BG_EUNSUPPORTED for a dtype pair other than fp32->bf16, bf16->bf16 and fp32->fp32 (also when shard_elems is 0);
 * BG_EINVAL for shard_elems not a multiple of 8 (of 4 for fp32->fp32) and for src not 16-B aligned. */
int bg_all_gather_cast(bg_ctx_t ctx, int gid, int lane, const void* src, int src_dtype, const size_t* dst_offs,
                       int dst_dtype, size_t shard_elems, void* stream);

/* C2  gradient reduce-scatter fused with pre/post-divide, cast and accumulate.
 * Replaces torch/distributed/fsdp/_runtime_utils.py:852 (prediv) :858 reduce_scatter_tensor :879 (postdiv)
 * :917-924 (cast to param dtype, += _saved_grad_shard), reached from sp_grad_reduce.py:125-126; with
 * dst_dtype bf16 and accumulate 0 it is the Megatron-SP reduce-scatter (mappings_group.py:120, layers.py:488-494).
 * Pull: member i reads slice i of every member's src, sums in fp32, dst = [dst +] sum * prescale * postscale.  In fp32, in this
 * order: acc = fmaf(x_m, prescale, acc) over the members m (own slice first, then the peers in ring order), acc * postscale, then
 * + the old dst when accumulating, then one rounding to dst's dtype.
 * BG_EUNSUPPORTED for a dst dtype other than bf16 / fp32, a bf16 dst with an fp32 src, or a src dtype other than bf16 / fp32;
 * BG_EINVAL for shard_elems not a multiple of 8 (bf16 src) or 4 (fp32 src) and for dst not 16-B aligned (order and the later
 * checks: see bg_all_gather_cast). */
int bg_reduce_scatter_acc(bg_ctx_t ctx, int gid, int lane, const size_t* src_offs, int src_dtype, void* dst,
                          int dst_dtype, size_t shard_elems, float prescale, float postscale, int accumulate,
                          void* stream);

/* C2 + optimizer (SURVEY 8f-3): the same pull reduce-scatter, but the reduced gradient is consumed in registers by an AdamW
 * step on the caller's fp32 shard (param, exp_avg, exp_avg_sq) -- the fp32 gradient shard is never written.  Update rule of
 * torch.optim.AdamW / apex FusedAdam adam_w_mode (galvatron/core/runtime/utils.py:137-150); `step` >= 1 for bias correction.
 * In fp32, per element, with g = (sum prescale * x) * postscale rounded once (bit for bit bg_reduce_scatter_acc's fp32 output):
 *   m = beta1 * m + (1 - beta1) * g;  v = beta2 * v + (1 - beta2) * g * g
 *   p = p * (1 - lr * weight_decay) - (lr / bias_corr1) * m / (sqrt(v) / bias_corr2_sqrt + eps)
 * (multiply-adds may be contracted).  The hyperparameters are the fp32 values received here, not the caller's doubles: 1 - beta
 * is formed in fp32 from the fp32 beta (at beta2 = 0.999, 1 - 0.999f is 1.3e-5 relative away from 1 - 0.999), and
 * bias_corr1 = 1 - beta1^step and bias_corr2_sqrt = sqrt(1 - beta2^step) are computed in double from the fp32 betas and then
 * rounded to fp32.
 * Errors of the three AdamW entries (this one, _clipped and bg_adamw_clipped), in this order, before the context is looked at and
 * before any launch, all BG_EINVAL: a null param, exp_avg or exp_avg_sq; any of them not 16-B aligned; step < 1; lr, eps or
 * weight_decay negative or not finite; beta1 or beta2 outside [0, 1) or NaN (torch.optim.AdamW's checks, on the fp32 values).
 * Then the errors of bg_reduce_scatter_acc with an fp32 dst. */
int bg_reduce_scatter_adamw(bg_ctx_t ctx, int gid, int lane, const size_t* src_offs, int src_dtype, float* param, float* exp_avg,
                            float* exp_avg_sq, size_t shard_elems, float prescale, float postscale, float lr, float beta1,
                            float beta2, float eps, float weight_decay, long long step, void* stream);

/* Gradient clipping by the global norm with the fused optimizer, in two passes over the same unsharded gradient.
 * Norm pass: the pull reduce-scatter above forms the reduced fp32 value (sum prescale * x) * postscale and writes, per warp of the
 * launch, the fp32 sum of its squares into `partials` (warp order; the entries past the launch's 4 * grid are zeroed; BG_EINVAL
 * when `n_partials` is too small -- 4 x comm_ctas, or 4 x local_ctas for a group of one, always suffice).  The sums accumulate in
 * fp64 in a fixed order: no atomics, run-to-run deterministic.  `skip` holds `n_skip` (<= BG_MAX_SKIP) shard-relative element
 * ranges [lo, hi), multiples of 8, left out of the sum (tensor-parallel duplicates).  `dst` null: nothing else is written; non-null:
 * also the fp32 shard, bit-identical to bg_reduce_scatter_acc's (accumulate 0).  Ranges may touch or overlap (an element in
 * several ranges is left out once); a range with lo = hi is empty.
 * Errors, BG_EINVAL, in this order and before any launch: null `partials` or n_partials < 1; n_skip outside [0, BG_MAX_SKIP]; a
 * range whose bounds are not multiples of 8 or with lo > hi; a range with hi > shard_elems; dst not 16-B aligned; then those of
 * bg_reduce_scatter_acc, then a launch that needs more than n_partials entries. */
#define BG_MAX_SKIP 16
int bg_reduce_scatter_sumsq(bg_ctx_t ctx, int gid, int lane, const size_t* src_offs, int src_dtype, float* dst, size_t shard_elems,
                            float prescale, float postscale, float* partials, int n_partials, const size_t* skip, int n_skip,
                            void* stream);

/* Step pass: bg_reduce_scatter_adamw with the reduced gradient multiplied by the device scalar *clip_coef (null: 1) before the
 * moments are updated: the kernel first forms postscale * *clip_coef in fp32, then g = (sum prescale * x) * that product.  At a
 * coefficient of 1, and with a null one, the result is bit-identical to bg_reduce_scatter_adamw's.  Errors: bg_reduce_scatter_adamw's. */
int bg_reduce_scatter_adamw_clipped(bg_ctx_t ctx, int gid, int lane, const size_t* src_offs, int src_dtype, float* param,
                                    float* exp_avg, float* exp_avg_sq, size_t shard_elems, float prescale, float postscale, float lr,
                                    float beta1, float beta2, float eps, float weight_decay, long long step, const float* clip_coef,
                                    void* stream);

/* The same clipped AdamW rule on a local fp32 gradient `grad` of n elements (a multiple of 4): the step of units whose gradient
 * was reduced into an fp32 shard by the norm pass, with g = grad * *clip_coef (null: grad) rounded once.  Where the norm pass's
 * postscale is a power of two, or the coefficient is 1, this step on its fp32 shard is bit-identical to
 * bg_reduce_scatter_adamw_clipped on the same sources.  Errors, BG_EINVAL: those of bg_reduce_scatter_adamw, then n not a
 * multiple of 4 or grad not 16-B aligned, then a null grad with n > 0. */
int bg_adamw_clipped(float* param, float* exp_avg, float* exp_avg_sq, const float* grad, size_t n, float lr, float beta1,
                     float beta2, float eps, float weight_decay, long long step, const float* clip_coef, void* stream);

/* C3/C5/C6/C13/C14/C16  all-reduce (sum|max): src is a symmetric buffer, dst any local pointer.
 * Replaces _runtime_utils.py:940 (DDP grads), mappings_group.py:19 _reduce (row-parallel fwd, layers.py:1114;
 * column-parallel bwd, mappings_group.py:139), cross_entropy.py:22-30,61-72,78-89, grad_reduce.py:121-124.
 * dst = scale * (sum | max over the members' src), in fp32 in member order, rounded once; every member's dst is bit-identical.
 * One-shot up to the "oneshot_bytes" tunable, and above it whenever the vectors do not split evenly over the members; two-shot
 * (reduce own slice, then gather) otherwise.  src is NOT left as it was in every case: the two-shot kernel writes the reduced,
 * scaled slice `my_index` back into slice `my_index` of the member's own src (its peers gather it from there), and on a
 * multicast-bound src (NVLS) every member's src ends up holding the whole result.  The one-shot kernel leaves src unchanged.
 * BG_EUNSUPPORTED for a dtype other than bf16 / fp32 or an op other than BG_SUM / BG_MAX; BG_EINVAL for elems not a multiple of
 * 8 (bf16) or 4 (fp32) and for dst not 16-B aligned (order and the later checks: see bg_all_gather_cast). */
int bg_all_reduce(bg_ctx_t ctx, int gid, int lane, const size_t* src_offs, void* dst, size_t elems, int dtype,
                  int redop, float scale, void* stream);

/* C14  tied word embeddings across pipeline stages: the first and the last stage hold two copies of one matrix, and after the
 * backward both gradients become their sum (finalize_wte_grads_func, pipeline.py:1031-1050, an all-reduce over the embedding
 * group).  IN PLACE over a group of exactly two members, `offs` the members' arena offsets of `elems` elements (bf16 or fp32, a
 * whole number of 16-B vectors): on return both regions hold scale * (x0 + x1), summed in fp32 in member order and rounded once,
 * bit-identical on both.  Member m reads and writes half of the vectors in both regions; no staging buffer, no copy.
 * BG_EUNSUPPORTED for another dtype and BG_EINVAL for a partial vector (both before the context is looked at), BG_EINVAL for a
 * group of another size; a failed call has launched nothing.  Timeouts are site 17. */
int bg_pair_sum_inplace(bg_ctx_t ctx, int gid, int lane, const size_t* offs, size_t elems, int dtype, float scale, void* stream);

/* C10  Ulysses all-to-all fused with the head/seq transpose (one pass, q/k/v in one launch).
 * Replaces transformer.py:1928-1987 single_all_to_all (permute+contiguous, dist.all_to_all_single :1977,
 * post_all2all :1904-1925).  Pull: for each peer q and tensor t, rows of `row_elems[t]` contiguous elements:
 *   dst_t[b*dst_bs + r*dst_rs + q*dst_peer_off + c] = src_t(peer q)[b*src_bs + r*src_rs + me*src_me_off + c]
 * BG_EINVAL for descs null or n_descs outside 1..4; BG_EUNSUPPORTED for a dtype other than bf16 / fp32; BG_EINVAL for a negative
 * batch, rows, row_elems or stride, a row length or stride that is not a whole number of 16-B vectors, dst not 16-B aligned, and
 * more than 2^32 vectors of one tensor per peer.  Then as bg_all_gather_cast; the source extent checked against the arena is
 * (batch-1)*src_bs + (rows-1)*src_rs + (n-1)*src_me_off + row_elems elements (none for an empty tensor). */
typedef struct bg_a2a_desc {
    const size_t* src_offs; /* symmetric source (arena offsets, group order) */
    void* dst;              /* local destination */
    long long batch, rows, row_elems;
    long long src_bs, src_rs, src_me_off; /* element strides in the peer's source */
    long long dst_bs, dst_rs, dst_peer_off;
} bg_a2a_desc;
int bg_all_to_all_rows(bg_ctx_t ctx, int gid, int lane, const bg_a2a_desc* descs, int n_descs, int dtype,
                       void* stream);

/* C11  pipeline p2p: copy `bytes` into the peer's arena at dst_off on `stream`, then raise flag `flag_id` there;
 * the receiver's bg_p2p_wait orders its stream after the flag (no device-wide sync) and bg_p2p_release hands
 * the slot back (a sender's 2nd..nth use of a flag first waits for that release).
 * Replaces pipeline.py:1095-1127 batch_isend_irecv + :1244 torch.cuda.synchronize(). */
int bg_p2p_send(bg_ctx_t ctx, int peer_rank, size_t dst_off, const void* src, size_t bytes, int flag_id,
                void* stream);
int bg_p2p_wait(bg_ctx_t ctx, int peer_rank, int flag_id, void* stream);
int bg_p2p_release(bg_ctx_t ctx, int peer_rank, int flag_id, void* stream);

/* C15  ring context parallelism: one hop of the zigzag ring (transformer.py:2252-2334 RingComm send_recv / commit / wait, which
 * the forward and backward schedules of :2335-2551 call once per step).  Member i of the cp group sends to member i+1 (mod n).
 * Receive slots are double-buffered by step parity; the flags live in the group's barrier lane BG_LANE_RING, one per CTA channel:
 * a push CTA waits for the receiver's "slot free" flag (skipped with wait_free = 0: the slot's first use), stores 16-B vectors into
 * the receiver's slot and raises its "arrived" flag; bg_cp_ring_wait consumes every channel's "arrived" flag on the receiver's
 * stream, bg_cp_ring_release raises the sender's "slot free" flags once the slot has been read.  The flags reset themselves
 * (CAS 0->1 / 1->0); spin timeouts leave the who/where record of bg_ctx_error_info (sites 13-16).  `elems` (per tensor) fixes the
 * number of channels, so a push and its wait / release must pass the same value.
 * kind 0: K and V, bf16: slot = [k | v] (elems each).  slot_offs: the group's symmetric buffer offsets of the parity's slot. */
#define BG_LANE_RING 5
int bg_cp_ring_push(bg_ctx_t ctx, int gid, int parity, int wait_free, const void* k, const void* v, size_t elems,
                    const size_t* slot_offs, void* stream);
/* kind 1: the backward's dK / dV accumulators, fp32, accumulate-and-forward (transformer.py:2470-2540, where the reference adds the
 * received fp32 buffers and the step's gradients on the compute stream before sending):
 *     next_slot[t] = (acc_in ? acc_in[t] : 0) + (float)contribution_t
 * for t in {dK, dV}; both are [batch][rows][row_elems] with the contribution [batch][c_rows][row_elems] bf16 covering rows
 * c_row0 .. c_row0 + c_rows - 1 only (c_rows 0: none).  The sum happens inside the push, fixed order: results are deterministic. */
int bg_cp_ring_acc_push(bg_ctx_t ctx, int gid, int parity, int wait_free, const float* acc_in, const void* dk, const void* dv,
                        long long batch, long long rows, long long row_elems, long long c_row0, long long c_rows,
                        const size_t* slot_offs, void* stream);
/* kind 0 / 1 as above; elems = per-tensor elements of the push being waited for / released */
int bg_cp_ring_wait(bg_ctx_t ctx, int gid, int kind, int parity, size_t elems, void* stream);
int bg_cp_ring_release(bg_ctx_t ctx, int gid, int kind, int parity, size_t elems, void* stream);

/* ---- local fused elementwise ops adjacent to the collectives (K5/K6/K9/a10 in SURVEY 2.3) ------------------ */
int bg_cast(const void* src, int src_dtype, void* dst, int dst_dtype, size_t elems, float scale, int accumulate,
            void* stream);
int bg_rmsnorm_fwd(const void* x, const void* w, void* y, float* rstd, long long rows, long long cols, float eps,
                   void* stream);
int bg_rmsnorm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw_partial,
                   long long rows, long long cols, int n_partial, void* stream);
/* LayerNorm with bias (GPT / BERT families: gpt_hf/GPTModel_tensor_parallel.py:34,56; fp32 math, one rounding).  backward:
 * dw_partial / db_partial are [n_partial][cols] fp32 per-CTA partial sums (the caller adds them up; a CTA that visits no row writes
 * zeros).  As RMSNorm: BG_EINVAL for rows < 0, cols not a positive multiple of 8 or a pointer not 16-B aligned, BG_EUNSUPPORTED
 * for cols > 8192. */
int bg_layernorm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, long long rows, long long cols,
                     float eps, void* stream);
int bg_layernorm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx, float* dw_partial,
                     float* db_partial, long long rows, long long cols, int n_partial, void* stream);
/* bias + GeLU of the GPT / BERT MLP (transformer.py:150-160 bias_gelu_impl): out = gelu(x + bias) when dy == NULL, else
 * out = dy * gelu'(x + bias).  tanh_form 1 = Megatron's fused / HF gelu_new, 0 = exact erf.  bias may be NULL.  BG_EINVAL for
 * rows < 0, cols not a positive multiple of 8 or a pointer not 16-B aligned. */
int bg_bias_gelu(const void* x, const void* bias, const void* dy, void* out, long long rows, long long cols, int tanh_form, void* stream);
/* bias + dropout + residual add of the GPT / BERT blocks, replacing the reference's F.dropout(x + bias) + residual at
 * GPTModel_tensor_parallel.py:31-39,51-59, BertModel_tensor_parallel.py:29-36,48-55 and the embedding dropouts
 * (GPTModel_sequential.py:55, BertModel_sequential.py:100-102):  y = residual + keep * scale * (x + bias), fp32 math, one rounding
 * per step.  x, residual, y: bf16 [rows][h] rows of a local [s_loc][b_loc][h] tensor; row r is token seq_base + r / b_loc of
 * sample sample_base + r % b_loc.  Element (token t, sample b, column j) is kept iff
 *     Philox4x32-10(counter = {j / 4, t, b, iteration}, key = {seed, site}).word[j % 4] >= floor(p * 2^32)
 * and kept values are scaled by (float)(1 / (1 - p)).  The mask depends on these global coordinates only, so every parallel
 * layout draws the same mask.  bias (bf16 or fp32 [h]) and residual may be NULL.  h % 8 == 0, 0 <= p < 1. */
int bg_dropout_add_fwd(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows, long long h,
                       long long b_loc, long long seq_base, long long sample_base, double p, unsigned seed, unsigned iteration,
                       unsigned site, void* stream);
/* its backward (the residual's gradient is dy itself): dx = bf16(keep * scale * dy) with the mask regenerated from the same
 * arguments; dbias_partial (may be NULL) = [n_partial][h] fp32 per-CTA column sums of keep * scale * dy (the caller adds them). */
int bg_dropout_bwd(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h, long long b_loc,
                   long long seq_base, long long sample_base, double p, unsigned seed, unsigned iteration, unsigned site,
                   void* stream);
/* the same pair at an explicit sample map: row r is sample sample_ids[r % b_loc] (device memory, b_loc uint32 entries) instead of
 * sample_base + r % b_loc; the mask, arithmetic and every other argument as bg_dropout_add_fwd / bg_dropout_bwd.  For the layers
 * whose samples a relocation gathered from several data-parallel ranks' microbatches: not one run of consecutive indices.
 * BG_EINVAL as those entries, and for a null or not 4-B aligned sample_ids. */
int bg_dropout_add_fwd_ids(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows, long long h,
                           long long b_loc, long long seq_base, const uint32_t* sample_ids, double p, unsigned seed, unsigned iteration,
                           unsigned site, void* stream);
int bg_dropout_bwd_ids(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h, long long b_loc,
                       long long seq_base, const uint32_t* sample_ids, double p, unsigned seed, unsigned iteration, unsigned site,
                       void* stream);
/* ViT front end (vit_hf/ViTModel_sequential.py ViTEmbeddings_).  bg_vit_patchify: pixels [batch][channels][height][width] (BG_BF16
 * or BG_F32) -> bf16 patch rows out [rows_pad][patch * patch * channels] in einops' "b c (h p1) (w p2) -> b (h w) (p1 p2 c)" order
 * (fp32 pixels rounded once, RNE); rows batch * P .. rows_pad - 1 are zeros, P = (height / patch) * (width / patch).
 * BG_EUNSUPPORTED for another pixel dtype; BG_EINVAL for an image that does not split into patches, patch * patch * channels not a
 * multiple of 8, rows_pad not a multiple of 8 >= batch * P, pixels not aligned to their element size or out not 16-B aligned. */
int bg_vit_patchify(const void* pixels, int pixel_dtype, void* out, long long batch, long long channels, long long height,
                    long long width, long long patch, long long rows_pad, void* stream);
/* y [s_run][batch][h] bf16 (SBH) from the patch GEMM's output patch_out [>= batch * n_patches][h] (row bi * n_patches + j = patch j
 * of sample bi) and bf16 [h] bias, [h] cls, [n_patches + 1][h] pos:  row 0 = cls + pos[0]; row s in 1..n_patches =
 * patch_out[bi * n_patches + s - 1] + (bias + pos[s]); rows n_patches + 1 .. s_run - 1 (padding tokens) = 0.  fp32 math, one rounding
 * per step.  p > 0: the embedding dropout applied to each sum before its rounding, with exactly bg_dropout_add_fwd's mask at (token s,
 * sample sample_base + bi, seed, iteration, site) and scale.  BG_EINVAL for batch < 1, n_patches < 1, s_run <= n_patches, a null or
 * non-16-B-aligned pointer, and the dropout arguments bg_dropout_add_fwd rejects (h, p, coordinates). */
int bg_vit_embed_fwd(const void* patch_out, const void* bias, const void* cls, const void* pos, void* y, long long batch,
                     long long n_patches, long long s_run, long long h, long long sample_base, double p, unsigned seed, unsigned iteration,
                     unsigned site, void* stream);
/* its backward from dy [s_run][batch][h] (g = dy, or keep * scale * dy regenerated from the same coordinates when p > 0):
 * dpatch [rows_pad][h] bf16 = g of rows 1..n_patches in (sample, patch) order, rows batch * n_patches .. rows_pad - 1 zero;
 * dpos [n_patches + 1][h] fp32 = the sums over the samples, in sample order, of g at each token (row 0 is also the CLS token's
 * gradient); dbias_partial [n_partial][h] fp32 = per-row-group sums of dpos rows 1..n_patches, in row order (the caller adds the
 * n_partial rows).  The sums depend on n_partial only, so the result is deterministic.  Rows of padding tokens are not read.
 * BG_EINVAL as the forward, and for rows_pad not a multiple of 8 >= batch * n_patches and n_partial outside [1, 65535]. */
int bg_vit_embed_bwd(const void* dy, void* dpatch, float* dpos, float* dbias_partial, int n_partial, long long batch,
                     long long n_patches, long long s_run, long long rows_pad, long long h, long long sample_base, double p, unsigned seed,
                     unsigned iteration, unsigned site, void* stream);
/* bias + tanh of the ViT pooler: out = tanh(x + bias) when dy == NULL, else out = dy * (1 - tanh(x + bias)^2), fp32 math, one
 * rounding.  bias may be NULL; the dbias column sums are the caller's, as for bg_bias_gelu.  BG_EINVAL for rows < 0, cols not a
 * positive multiple of 8 or a pointer not 16-B aligned. */
int bg_bias_tanh(const void* x, const void* bias, const void* dy, void* out, long long rows, long long cols, void* stream);
/* Swin (swin/SwinModel_tensor_parallel.py).  Activations are SBH rows (row = token * mb + sample) of tokens_run tokens per sample,
 * the tokens real ones first; a (possibly cyclically shifted) window partition of a layer shape is one int32 token map
 * map[w * window_tokens + i] = the token at position i of window w, and inv its inverse (inv[map[j]] = j); window rows are
 * [mb * n_windows][window_tokens][...], window b * n_windows + w of sample b.  tokens must equal n_windows * window_tokens; the
 * maps must be permutations of 0..tokens-1 (the caller builds them; they are not checked).  bf16 activations, 16-B vectors.
 * bg_swin_window_qkv_fwd: mixed [tokens_run * mb][heads * 3 * head_dim] (per head q | k | v) + bias [heads * 3 * head_dim] -> q, k, v
 * [mb * n_windows][window_tokens][heads][head_dim], one rounding.  bg_swin_window_qkv_bwd: dmixed rows gathered from dq, dk, dv
 * (padding-token rows zero) and dbias_partial [n_partial][heads * 3 * head_dim] fp32 per-row-group column sums in row order (the
 * caller adds the rows; deterministic).  BG_EINVAL for inconsistent counts, head_dim not a multiple of 8, n_partial outside
 * [1, 65535] and null or misaligned pointers. */
int bg_swin_window_qkv_fwd(const void* mixed, const void* bias, const int* map, void* q, void* k, void* v, long long mb,
                           long long tokens, long long tokens_run, long long n_windows, long long window_tokens, long long heads,
                           long long head_dim, void* stream);
int bg_swin_window_qkv_bwd(const void* dq, const void* dk, const void* dv, void* dmixed, float* dbias_partial, int n_partial,
                           const int* inv, long long mb, long long tokens, long long tokens_run, long long n_windows,
                           long long window_tokens, long long heads, long long head_dim, void* stream);
/* Swin's learned relative-position bias (HF SwinSelfAttention.relative_position_bias_table), window w, L = window_tokens = w * w,
 * (2w-1)^2 table entries.  bg_swin_rel_bias_fwd: table [(2w-1)^2][heads] (table_dtype BG_BF16 or BG_F32), index int32 [L * L]
 * (HF's relative_position_index, entries < (2w-1)^2) and shift_mask uint8 [n_windows][L][L] (non-zero where HF's shift mask separates
 * query i and key j; NULL when the block is not shifted) -> bias [mb * n_windows][heads][L][ld] bf16, window b * n_windows + w of
 * sample b: element (n, h, i, j) = table[index[i * L + j]][h] rounded to bf16, or -inf where shift_mask[n % n_windows][i][j] != 0;
 * columns L .. ld - 1 zero.  bg_swin_rel_bias_bwd: the gradient of that bias, same layout, -> dtable_partial [n_partial][(2w-1)^2]
 * [heads] fp32: partial p sums windows p, p + n_partial, ... and, for entry t, the cells c = i * L + j in the order cells[offsets[t]]
 * .. cells[offsets[t + 1] - 1] (the caller lists every cell with index t there, once); the caller adds the rows.  The order of every
 * sum is fixed, so the result is deterministic.  The index, cells and offsets are not checked.  BG_EINVAL for a size < 1,
 * window_tokens != window^2, ld not a multiple of 8 >= window_tokens, n_partial outside [1, 65535] and null or misaligned pointers
 * (bias / dbias 16-B, table its element size, the int32 arrays and dtable_partial 4-B); BG_EUNSUPPORTED for a table dtype other than
 * BG_BF16 / BG_F32, more than 65535 heads or a window above 15 x 15 tokens per side (L * L fp32 > 200 KiB of shared memory). */
int bg_swin_rel_bias_fwd(const void* table, int table_dtype, const int* index, const unsigned char* shift_mask, void* bias, long long mb,
                         long long n_windows, long long heads, long long window, long long window_tokens, long long ld, void* stream);
int bg_swin_rel_bias_bwd(const void* dbias, const int* cells, const int* offsets, float* dtable_partial, int n_partial, long long mb,
                         long long n_windows, long long heads, long long window, long long window_tokens, long long ld, void* stream);
/* T5 cross-attention (t5/T5Model_tensor_parallel.py): the two projections' outputs -> the attention library's layout.
 * bg_cross_attn_qkv_fwd: q_mixed [s_q * batch][heads * head_dim] + q_bias and kv_mixed [s_k * batch][heads * 2 * head_dim] (per head
 * k | v) + kv_bias, SBH rows (row = token * batch + sample) -> q [batch][s_q][heads][head_dim], k, v [batch][s_k][heads][head_dim];
 * the bias added in fp32, one rounding; either bias may be NULL (nothing added).  bg_cross_attn_qkv_bwd: dq, dk, dv -> dq_mixed and
 * dkv_mixed in the inputs' layouts, and dbias_partial [n_partial][heads * 3 * head_dim] fp32 per-row-group column sums in row order,
 * the query's heads * head_dim columns first (the caller adds the rows; deterministic).  bf16, 16-B vectors; s_q * batch and
 * s_k * batch may be odd.  BG_EINVAL for a size < 1, head_dim not a positive multiple of 8, n_partial outside [1, 65535] and null
 * or misaligned pointers. */
int bg_cross_attn_qkv_fwd(const void* q_mixed, const void* q_bias, const void* kv_mixed, const void* kv_bias, void* q, void* k, void* v,
                          long long s_q, long long s_k, long long batch, long long heads, long long head_dim, void* stream);
int bg_cross_attn_qkv_bwd(const void* dq, const void* dk, const void* dv, void* dq_mixed, void* dkv_mixed, float* dbias_partial,
                          int n_partial, long long s_q, long long s_k, long long batch, long long heads, long long head_dim, void* stream);
/* attention output windows [mb * n_windows][window_tokens][cols] -> SBH rows [tokens_run * mb][cols] (padding-token rows zero), and
 * the backward gather; pure copies.  BG_EINVAL as above and for cols not a positive multiple of 8. */
int bg_swin_window_merge_fwd(const void* windows, void* rows, const int* map, const int* inv, long long mb, long long tokens,
                             long long tokens_run, long long n_windows, long long window_tokens, long long cols, void* stream);
int bg_swin_window_merge_bwd(const void* drows, void* dwindows, const int* map, const int* inv, long long mb, long long tokens,
                             long long tokens_run, long long n_windows, long long window_tokens, long long cols, void* stream);
/* Patch merging + LayerNorm.  x holds a height x width token grid of mb samples with cols_in columns: SBH rows (token * mb + b) or,
 * with in_bsh, rows b * height * width + token (the patch GEMM's order); rows_in >= mb * height * width rows.  Output row t' * mb + b
 * of y [tokens_out_run * mb][r * r * cols_in] (t' on the (height / r) x (width / r) grid) is the concatenation over q = 0..r*r-1 of
 * token (r i' + (q & 1), r j' + (q >> 1)) -- HF SwinPatchMerging's x0, x1, x2, x3 -- plus add_bias (may be NULL), normalised as
 * bg_layernorm_fwd does (same arithmetic, so the same rounding) with w, b [r * r * cols_in]; mean / rstd fp32 per output row.
 * Padding-token rows are zero (mean = rstd = 0).  r = 1 with the patch bias is the embedding's bias + norm.  Backward: dx rows
 * scattered to the sources (every input token feeds one output token; input rows mb * height * width .. rows_in - 1 zero) and per-CTA
 * fp32 partials dw = sum dy * xhat, db = sum dy and, iff add_bias != NULL, dbias = sum dx.  BG_EINVAL for r not 1 or 2, a grid that
 * does not split into r x r blocks, cols_in not a positive multiple of 8, too few rows, n_partial outside [1, 65535] and null or
 * misaligned pointers; BG_EUNSUPPORTED for a merged row wider than 10240 columns. */
int bg_swin_merge_ln_fwd(const void* x, const void* add_bias, const void* w, const void* b, void* y, float* mean, float* rstd,
                         long long mb, long long height, long long width, long long r, int in_bsh, long long rows_in, long long cols_in,
                         long long tokens_out_run, float eps, void* stream);
int bg_swin_merge_ln_bwd(const void* dy, const void* x, const void* add_bias, const void* w, const float* mean, const float* rstd,
                         void* dx, float* dw_partial, float* db_partial, float* dbias_partial, int n_partial, long long mb,
                         long long height, long long width, long long r, int in_bsh, long long rows_in, long long cols_in, void* stream);
/* Swin's pooler: x [tokens_run][mb][cols] -> y [rows_out][cols], y[b] = (fp32 sum of x[t][b] over t < tokens, in token order) /
 * tokens, rows mb .. rows_out - 1 zero.  Backward: dx[t][b] = dy[b] / tokens for t < tokens, 0 for the padding tokens.  BG_EINVAL
 * for tokens < 1, tokens_run < tokens, mb < 1, rows_out < mb, cols not a positive multiple of 8 and null or misaligned pointers. */
int bg_swin_mean_pool_fwd(const void* x, void* y, long long tokens, long long tokens_run, long long mb, long long rows_out,
                          long long cols, void* stream);
int bg_swin_mean_pool_bwd(const void* dy, void* dx, long long tokens, long long tokens_run, long long mb, long long cols, void* stream);
/* Per-sample drop path (stochastic depth) of Swin's attention branch on an SBH block [rows][h] whose row r is sample
 * sample_base + r % b_loc:  y = residual + keep * scale * (x + bias), dx = keep * scale * dy with fp32 per-row-group dbias partials
 * (as bg_dropout_bwd).  The sample is kept iff word 0 of Philox4x32-10(counter = (0, 0xffffffff, sample, iteration), key = (seed,
 * site)) >= floor(p * 2^32); scale = 1 / (1 - p); arithmetic and argument checks as bg_dropout_add_fwd / bg_dropout_bwd (bias bf16
 * or fp32, bias and residual may be NULL; dbias_partial may be NULL). */
int bg_drop_path_add_fwd(const void* x, const void* bias, int bias_dtype, const void* residual, void* y, long long rows, long long h,
                         long long b_loc, long long sample_base, double p, unsigned seed, unsigned iteration, unsigned site, void* stream);
int bg_drop_path_add_bwd(const void* dy, void* dx, float* dbias_partial, int n_partial, long long rows, long long h, long long b_loc,
                         long long sample_base, double p, unsigned seed, unsigned iteration, unsigned site, void* stream);
/* host-only: one Philox4x32-10 block (the generator of curand_philox4x32_x.h), so the mask definition can be checked without a
 * GPU.  No CUDA call. */
void bg_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
/* log-sum-exp merge of one ring step's flash-attn block result into the running result (transformer.py:2209-2250
 * update_out_and_lse): for query rows row_off .. row_off + sq_blk - 1 of the running state,
 *     lse = m + log(exp(lse_a - m) + exp(lse_b - m)),  m = max(lse_a, lse_b);   out = out_a exp(lse_a - lse) + out_b exp(lse_b - lse)
 * in fp32.  blk_out [b][sq_blk][n][d] bf16, blk_lse [b][n][sq_blk] fp32 (flash-attn's layout); acc_out [b][s][n][d] fp32 and
 * acc_lse [b][n][s] fp32 are updated in place (init = 1: they are set to the block instead).  final_out (bf16 [b][s][n][d], may be
 * NULL): also write every row of the merged output there, rounded once; acc_lse is then the output's LSE.  d % 8 == 0, d <= 256. */
int bg_lse_merge(const void* blk_out, const float* blk_lse, float* acc_out, float* acc_lse, void* final_out, long long b, long long s,
                 long long sq_blk, long long n, long long d, long long row_off, int init, void* stream);
int bg_swiglu_fwd(const void* gate_up, void* y, long long rows, long long ffn, void* stream);
int bg_swiglu_bwd(const void* dy, const void* gate_up, void* dgate_up, long long rows, long long ffn, void* stream);
/* fused QKV split + RoPE + [s,b,ng,(r+2)*hn] -> q [b,s,ng*r,hn], k/v [b,s,ng,hn] relayout; backward=1 is the exact
 * transpose (reads dq,dk,dv, writes dmixed).  Replaces the split / repeat_interleave / apply_rotary_pos_emb /
 * rearrange(...).contiguous() chain of transformer.py:731-767,842-867 (GQA stays un-expanded: flash-attn is
 * called with ng KV heads).  cos/sin: [s, hn/2] fp32 tables for this rank's positions. */
int bg_qkv_rope(void* mixed, void* q, void* k, void* v, const float* cos_t, const float* sin_t, long long s, long long b,
                long long ng, long long r, long long hn, int backward, void* stream);

/* a10  vocab-parallel cross-entropy (cross_entropy.py:14-152) as three row kernels around the two small
 * all-reduces (MAX of rowmax; SUM of (sum_exp, predicted_logit)).  bg_ce_bwd overwrites logits with dlogits. */
int bg_ce_rowmax(const void* logits, int dtype, float* rowmax, long long rows, long long vocab_local, void* stream);
int bg_ce_sumexp(const void* logits, int dtype, const long long* target, const float* rowmax, float* out2 /* [rows][2] */,
                 long long rows, long long vocab_local, long long vocab_start, void* stream);
int bg_ce_bwd(void* logits, int dtype, const long long* target, const float* rowmax, const float* sum2,
              const float* grad_loss, long long rows, long long vocab_local, long long vocab_start, void* stream);

/* ---- GEMM (K1): bf16 x bf16 -> fp32 accumulate in registers -> bf16, wgmma + TMA -------------------------- */
/* C[M,N] (+)= A op B.  layout: 0 = "TN" C = A[M,K] * B[N,K]^T (forward, layers.py:417);
 * 1 = "NN" C = A[M,K] * B[K,N] (dgrad, layers.py:462); 2 = "NT" C = A[K,M]^T * B[K,N] (wgrad, layers.py:534). */
int bg_gemm_bf16(const void* a, const void* b, void* c, long long m, long long n, long long k, int layout,
                 int accumulate, void* stream);
/* C = A op B + addend ([M][N] bf16): the residual add behind a projection (llama_hf/LlamaModel_tensor_parallel.py:83,100
 * `hidden_states + input_tensor`) in the GEMM epilogue -- one rounding, no separate elementwise pass.  addend may alias c. */
int bg_gemm_bf16_add(const void* a, const void* b, void* c, const void* addend, long long m, long long n, long long k, int layout,
                     void* stream);

/* C5/C8 fused with K1: C = A op B is computed in 128x128 wgmma tiles and REDUCE-SCATTERED along M over the group inside
 * the same operation -- every finished partial tile is TMA-stored into the owning rank's arena (peer HBM over NVLink) and
 * counted there; a tile reducer on the owner -- launched into the same stream as the GEMM's programmatic dependent, so it
 * runs beside the GEMM CTAs once all of them are resident -- sums the p partials as they land and writes out[M/p, N].
 * Replaces layers.py:1061-1109 (row-parallel GEMM then mappings_group.py:120 reduce-scatter) and :462,488-494 (dgrad +
 * reduce-scatter).  partial_offs: symmetric bf16 buffer of M*N elements; flag_offs: symmetric u32[(M/p/128)*ceil(N/128)],
 * zero-initialised.  `out` is complete in stream order.
 * Returns BG_EINVAL, in this order, for: layout outside 0-2; m, n or k not a positive multiple of 8; a, b or out not 16-B
 * aligned; a null ctx or a bad lane (bad gid: BG_EGROUP); a group of fewer than 2 members; M not a multiple of p*128; a symmetric
 * offset that is not 16-B aligned or a buffer outside the arena.  A failed call -- these, or a tensor-map encode that rejects an
 * operand (BG_ECUDA) -- has launched nothing, on this member or for its peers. */
int bg_gemm_reduce_scatter(bg_ctx_t ctx, int gid, int lane, const void* a, const void* b, long long m, long long n, long long k,
                           int layout, const size_t* partial_offs, const size_t* flag_offs, void* out, void* stream);

/* C5/C6 fused with K1: GEMM + ALL-REDUCE (row-parallel forward, layers.py:1110-1114: matmul then reduce_from_tensor_model_parallel
 * _region; column-parallel dgrad, mappings_group.py:139).  Both shots of the two-shot all-reduce happen inside the fused
 * operation: partial tiles are scattered to their owners as in bg_gemm_reduce_scatter; the owner's tile reducer sums a tile when
 * its p partials have landed and immediately broadcasts the rows into EVERY member's out buffer (peer stores, or one multimem.st
 * when out is multicast-bound); the reducers leave through a cross-rank barrier, so out -- a symmetric bf16 [M][N] buffer,
 * out_offs -- is complete on every member in stream order.  Deterministic (fixed summation order), fp32 accumulation.
 * BG_EINVAL as bg_gemm_reduce_scatter (with no `out` pointer to check: out is symmetric); a failed call has launched nothing. */
int bg_gemm_all_reduce(bg_ctx_t ctx, int gid, int lane, const void* a, const void* b, long long m, long long n, long long k, int layout,
                       const size_t* partial_offs, const size_t* flag_offs, const size_t* out_offs, void* stream);

/* C7 fused with K1: ALL-GATHER + GEMM (column-parallel forward under Megatron-SP, layers.py:399-417: _all_gather_base into the
 * global buffer, then matmul; also the row-parallel dgrad, whose dY is gathered, mappings_group.py:243-258).
 * C[M,N] = gather_M(a_local[M/p,K]) op B.  A slim push kernel on comm_stream (resident beside the GEMM) sends the local rows to
 * every member's staging buffer (stage_offs: symmetric bf16 [M][K]) in 128-row blocks and counts each block in on the receiver
 * (flag_offs: symmetric u32[p][M/p/128], zero-initialised); the GEMM's TMA producer reads the rank's own rows from a_local and
 * every remote block from staging as soon as its counter is complete, walking the blocks in arrival order.  layout 0 (TN) or
 * 1 (NN).  C is complete in `stream` order; a_local may be reused after the call in `stream` order.
 * Returns BG_EINVAL, in this order, for: layout outside 0-1; m, n or k not a positive multiple of 8; a_local, b or c not 16-B
 * aligned; a null ctx or a bad lane (bad gid: BG_EGROUP); a group of fewer than 2 members; M not a multiple of p*128; a symmetric
 * offset that is not 16-B aligned or a buffer outside the arena.  A failed call -- these, or a tensor-map encode that rejects an
 * operand (BG_ECUDA) -- has launched nothing: no push, no GEMM, no wait on either stream. */
int bg_all_gather_gemm(bg_ctx_t ctx, int gid, int lane, const void* a_local, const size_t* stage_offs, const size_t* flag_offs,
                       const void* b, void* c, long long m, long long n, long long k, int layout, void* stream, void* comm_stream);

/* ---- NVLS: all-reduce reduced and replicated INSIDE the NVSwitch (multimem.ld_reduce / multimem.st) ---------------------
 * Replaces the tensor-parallel all-reduces (mappings_group.py:19, layers.py:474-480) for large messages, where NCCL itself
 * switches to NVLS: N/p bytes in and N/p out per GPU instead of 2(p-1)/p*N.  One multicast object per group over one
 * symmetric buffer: the group's first rank creates it (-> fd), every other member imports the fd, ALL join (device added),
 * barrier on the host, ALL bind their own arena range (multicast-granularity aligned).  BG_CTX_VMM contexts only.
 * The bound range may be any part of the arena (the host binds the whole region that holds its symmetric buffers): every
 * collective whose buffer lies inside it at the same offset on all members then uses the switch on its own --
 * bg_all_reduce (ld_reduce + st), bg_all_gather_cast and the bg_gemm_all_reduce broadcast (multimem.st), bg_reduce_scatter_acc /
 * _adamw (multimem.ld_reduce) -- above "nvls_min_bytes". */
int bg_group_mc_create(bg_ctx_t ctx, int gid, size_t bytes, int* fd_out);
int bg_group_mc_join(bg_ctx_t ctx, int gid, int fd /* -1 on the creator */, size_t bytes);
int bg_group_mc_bind(bg_ctx_t ctx, int gid, size_t arena_offset);
int bg_group_mc_disable(bg_ctx_t ctx, int gid);   /* setup failed on some member: the group keeps the peer-to-peer kernels */

#ifdef __cplusplus
}
#endif
#endif /* BG_GALVATRON_H */
