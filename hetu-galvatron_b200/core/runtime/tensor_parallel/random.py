"""Dropout randomness of the GPT / BERT families (the role of megatron ``core/tensor_parallel/random.py``).

Hidden-state dropout (embedding output, attention-block output, MLP-block output) draws no state at all: the mask of an element is a
pure function of (seed, iteration, site, global sample index, global token position, hidden column) -- Philox4x32-10, defined in
``include/bg_galvatron.h`` -- so TP, Megatron-SP, Ulysses, ZeRO, pipelining and activation recompute all draw the masks a single
process draws on the global batch, and nothing is stored for backward.  The coordinates come from a per-microbatch *dropout
context*: the iteration is ``forward_backward``'s ``iter``, the sample base is (data-parallel index x local batch + the offset of the
microbatch in the contiguous ``chunk`` split, pipeline/utils.py).  ``GalvatronModel.forward_backward`` and the schedules set it;
``_BiasDropoutAddFn`` copies it into its autograd context and ``_CheckpointFn`` captures it for the recompute.

That sample base is the embedding row's.  A layer whose strategy differs from its predecessor's holds the samples a relocation
gathered or split (sample_layout.py): the context also carries the model's per-row sample layouts, and a row draws at its own
samples -- through the ``sample_base`` kernels when they are one run of consecutive indices (every row that holds the embedding's
samples: the same launches as without a layout), else through the kernels that take a device vector of sample ids.

Site numbering: site = 3 * row + kind, row 0 = the embedding (kind 0), row i + 1 = transformer layer i with kind 1 = attention-block
output and kind 2 = MLP-block output.  The row is the whole-model row (GPT, BERT and ViT: the embedding, then the layers).

Attention-probability dropout stays inside the attention library call (torch SDPA / flash-attn), whose masks come from torch's
generator and cannot be made layout-invariant.  It runs under ``RngTracker.fork``: a generator state per (layer, tensor-parallel
rank, Ulysses rank), seeded like megatron's ``model_parallel_cuda_manual_seed`` (seed + 2718 + ...), so the head slices of
different ranks are not correlated; the checkpoint recompute replays the tracker state.
"""
import collections
import contextlib

import torch

from ..backend import get_backend

DropoutContext = collections.namedtuple("DropoutContext", "seed iteration sample_base batch samples")

_CTX = DropoutContext(seed=0, iteration=0, sample_base=0, batch=None, samples=None)
_STEP = dict(seed=0, iteration=0, sample_base=0, layouts=None, local=0)
_IDS = {}       # (global sample ids, device) -> int32 id vector: one per distinct non-contiguous row / microbatch

SITE_EMBEDDING, SITE_ATTENTION, SITE_MLP = 0, 1, 2
# Swin's per-sample drop path on the attention branch (its blocks have no hidden dropout there; the mask's counter is one no
# dropout element uses, include/bg_galvatron.h bg_drop_path_add_fwd)
SITE_DROP_PATH = SITE_ATTENTION


def check_probability(p, name="dropout"):
    """0 <= p < 1, else ValueError (at construction)."""
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError("%s probability %r must satisfy 0 <= p < 1" % (name, p))
    return p


def site(layer_row, kind):
    return 3 * int(layer_row) + int(kind)


class MicrobatchSamples(collections.namedtuple("MicrobatchSamples", "layouts local offset size")):
    """The rows' sample layouts (sample_layout.derive_sample_layouts) at one microbatch of a ``local``-sample batch."""

    def ids(self, row):
        from ..sample_layout import instantiate
        return instantiate(self.layouts[row], self.local, self.offset, self.size)


def begin_iteration(seed, iteration, sample_base, layouts=None, local=0):
    """One ``forward_backward`` call: the iteration and the global index of this rank's first sample; ``layouts`` ({row: layout} of
    this rank's rows, None = every row holds the embedding's samples) and ``local`` (the data-parallel batch) map each row to the
    samples it holds."""
    _STEP.update(seed=int(seed), iteration=int(iteration), sample_base=int(sample_base), layouts=layouts, local=int(local))
    set_microbatch(0, None)


def set_microbatch(offset, size):
    """Before a microbatch's forward: its first sample is ``offset`` samples into this rank's local batch."""
    global _CTX
    samples = None
    if _STEP["layouts"] is not None and size is not None:
        samples = MicrobatchSamples(_STEP["layouts"], _STEP["local"], int(offset), int(size))
    _CTX = DropoutContext(_STEP["seed"], _STEP["iteration"], _STEP["sample_base"] + int(offset), None if size is None else int(size),
                          samples)


def row_samples(row, ctx=None):
    """Global sample indices held by whole-model row ``row`` in the current (or the given) microbatch context, in local order; None
    when the context carries no layout."""
    ctx = _CTX if ctx is None else ctx
    if ctx.samples is None or row not in ctx.samples.layouts:
        return None
    return ctx.samples.ids(row)


def _row_sample(ctx, row, x):
    """The sample coordinate of row ``row``'s activation x [s_loc, b_loc, h]: an int s (its samples are s, s + 1, ...) or the int32
    device vector of its sample ids."""
    ids = row_samples(row, ctx)
    if ids is None:
        if ctx.batch is not None and x.shape[1] != ctx.batch:
            raise ValueError("dropout: a layer sees %d samples of a %d-sample microbatch and the model has no sample layout for row %d"
                             % (x.shape[1], ctx.batch, row))
        return ctx.sample_base
    if x.shape[1] != len(ids):
        raise ValueError("dropout: row %d holds %d samples, its sample layout %d" % (row, x.shape[1], len(ids)))
    if ids == list(range(ids[0], ids[0] + len(ids))):
        return ids[0]
    key = (tuple(ids), x.device)
    t = _IDS.get(key)
    if t is None:
        t = torch.tensor(ids, dtype=torch.int32)
        # (pinned + non_blocking: the copy is ordered on the stream and the host does not wait for the work queued before it)
        t = _IDS[key] = t.pin_memory().to(x.device, non_blocking=True) if x.device.type == "cuda" else t
    return t


def get_context():
    return _CTX


def set_context(ctx):
    global _CTX
    _CTX = ctx


class _BiasDropoutAddFn(torch.autograd.Function):
    """y = residual + keep * scale * (x + bias): one row kernel forward, one backward that regenerates the mask -- one launch of
    each per run of consecutive tokens in the local rows (a zigzag context-parallel rank holds two runs).  The sample coordinate is
    an int (the row's samples are consecutive) or the row's sample-id vector, which the context keeps for the backward (it may run
    under another microbatch's dropout context)."""

    @staticmethod
    def forward(ctx, x, bias, residual, p, coords, runs):
        ctx.p, ctx.coords, ctx.runs = p, coords, runs     # (seed, iteration, site, sample base or ids), ((row0, rows, token0), ...)
        ctx.has_residual, ctx.bias_dtype = residual is not None, None if bias is None else bias.dtype
        seed, iteration, site_id, sample = coords
        be = get_backend()
        fwd = be.dropout_add_fwd_ids if torch.is_tensor(sample) else be.dropout_add_fwd
        if len(runs) == 1:
            return fwd(x, bias, residual, p, seed, iteration, site_id, runs[0][2], sample)
        return torch.cat([fwd(x[r0:r0 + n], bias, None if residual is None else residual[r0:r0 + n], p, seed, iteration, site_id, t0,
                              sample) for r0, n, t0 in runs])

    @staticmethod
    def backward(ctx, dy):
        seed, iteration, site_id, sample = ctx.coords
        with_bias, be = ctx.bias_dtype is not None, get_backend()
        bwd = be.dropout_bwd_ids if torch.is_tensor(sample) else be.dropout_bwd
        parts = [bwd(dy[r0:r0 + n], ctx.p, seed, iteration, site_id, t0, sample, with_bias=with_bias) for r0, n, t0 in ctx.runs]
        dx = parts[0][0] if len(parts) == 1 else torch.cat([d for d, _ in parts])
        db = None if not with_bias else (parts[0][1] if len(parts) == 1 else sum(b for _, b in parts)).to(ctx.bias_dtype)
        return dx, db, (dy if ctx.has_residual else None), None, None, None


def bias_dropout_add(x, bias, residual, p, site_id, seq_base=0):
    """Dropout of an SBH tensor x [s_loc, b_loc, h] (plus bias, plus residual) with the current microbatch's dropout context.
    ``seq_base``: the local rows are tokens ``seq_base``.. of the microbatch's samples; or the rows' runs of consecutive tokens,
    ((first row, rows, first token), ...) as ``redistribute.token_runs`` gives them, covering the rows in order.  The samples are
    those the site's row (``site_id // 3``) holds."""
    ctx = _CTX
    sample = _row_sample(ctx, int(site_id) // 3, x)
    if isinstance(seq_base, (tuple, list)):
        runs = tuple(tuple(int(v) for v in run) for run in seq_base)
    else:
        runs = ((0, x.shape[0], int(seq_base)),)
    if runs[0][0] != 0 or sum(n for _, n, _ in runs) != x.shape[0] or any(a[0] + a[1] != b[0] for a, b in zip(runs, runs[1:])):
        raise ValueError("dropout: token runs %s do not cover the %d local rows in order" % (runs, x.shape[0]))
    return _BiasDropoutAddFn.apply(x, bias, residual, float(p), (ctx.seed, ctx.iteration, int(site_id), sample), runs)


class RngTracker:
    """Named generator states swapped into torch's default generator of a device (megatron ``CudaRNGStatesTracker``)."""

    def __init__(self):
        self.states = {}

    def get_states(self):
        return {k: v.clone() for k, v in self.states.items()}

    def set_states(self, states):
        self.states = {k: v.clone() for k, v in states.items()}

    @staticmethod
    def _get(device):
        return torch.cuda.get_rng_state(device) if device.type == "cuda" else torch.get_rng_state()

    @staticmethod
    def _set(state, device):
        if device.type == "cuda":
            torch.cuda.set_rng_state(state, device)
        else:
            torch.set_rng_state(state)

    @contextlib.contextmanager
    def fork(self, name, seed, device):
        key = (name, str(device))
        if key not in self.states:
            g = torch.Generator(device=device)
            g.manual_seed(int(seed))
            self.states[key] = g.get_state()
        orig = self._get(device)
        self._set(self.states[key], device)
        try:
            yield
        finally:
            self.states[key] = self._get(device)
            self._set(orig, device)


_TRACKER = RngTracker()


def get_rng_tracker():
    return _TRACKER


def model_parallel_seed(seed, layer_number, tp_rank, sp_rank):
    """megatron's ``seed + 2718 + tp_rank``, extended by the Ulysses rank and the layer (so pipeline stages differ as well)."""
    return int(seed) + 2718 + tp_rank + 64 * sp_rank + 4096 * int(layer_number)
