"""Activation relocation between consecutive layers whose (tp|sp, cp) strategy differs.

Same contract as ``galvatron/core/runtime/redistribute.py`` ``fused_split_allgather`` (:354-426): a float activation
[s/g_old, b_old, h] becomes [s/g_new, b_new, h] by
    1. (sequence parallel only) all-gather the sequence over the OLD sequence group              (:283-289)
    2. undo / apply the zigzag context-parallel token order if the cp degree changes            (:290-296)
    3. SBH -> BSH, then split (fused_split_group) or all-gather (fused_allgather_group) the BATCH (:298-326)
    4. BSH -> SBH, then (sequence parallel only) keep this rank's slice of the NEW sequence group (:327-345)
and integer tensors (tokens / labels / masks, ``is_input=False``) only do the batch split / gather (:231-267).
Backward applies the same function with the split / all-gather roles swapped (:391-416).

The gathers are the pull all-gather kernel over peer memory (C12); splits are local slices.
"""
import torch

from .backend import get_backend


def _size(group):
    return 1 if group is None else group.size


def _zigzag_indices(cp):
    idx = []
    for r in range(cp):
        idx += [r, 2 * cp - r - 1]
    return idx


def _zigzag_transformation(x, cp):
    """Token-chunk order for zigzag ring attention: rank r holds chunks (r, 2cp-1-r) (:8-27)."""
    if cp == 1:
        return x
    assert 2 * cp <= x.shape[0], "sequence length must be larger than 2*cp"
    # chunk views concatenated: an index tensor built on the host would be a copy that synchronises the stream with the host in
    # every context-parallel layer (and, with virtual ranks on one device, would wait on a peer whose work is not issued yet)
    chunks = x.reshape(2 * cp, -1, *x.shape[1:])
    return torch.cat([chunks[i] for i in _zigzag_indices(cp)]).reshape(-1, *x.shape[1:])


def local_positions(seq, cp=1, cp_rank=0, sp=1, sp_rank=0):
    """Global token positions of the rows one rank holds of a ``seq``-token sequence, in row order (LongTensor).

    The reference's layout for zigzag context parallelism composed with Ulysses (``get_pos_emb_on_this_cp_sp_rank_galvatron``,
    megatron/core/models/common/embeddings/rotary_pos_embedding.py:33-56): cp rank r holds chunks (r, 2cp-1-r) of 2cp equal chunks,
    and sp rank j holds the j-th of ``sp`` contiguous slices of those two chunks concatenated (a slice straddles the two chunks when
    ``sp`` is odd).  Tokens, labels, RoPE tables and relocation all follow it: the relocation gathers over tp_sp_cp groups whose
    rank order is sp-minor, which is this order."""
    if cp == 1:
        if seq % sp:
            raise ValueError("sequence length %d is not a multiple of the sequence-parallel degree %d" % (seq, sp))
        idx = torch.arange(seq)
    else:
        half = seq // (2 * cp)
        if seq % (2 * cp * sp):
            raise ValueError("sequence length %d is not a multiple of 2 x cp x sp = %d" % (seq, 2 * cp * sp))
        idx = torch.cat([torch.arange(cp_rank * half, (cp_rank + 1) * half),
                         torch.arange((2 * cp - 1 - cp_rank) * half, (2 * cp - cp_rank) * half)])
    n = idx.numel() // sp
    return idx[sp_rank * n:(sp_rank + 1) * n]


def zigzag_local(x, group, sp_group=None):
    """[b, s] tokens / labels / positions -> the tokens this rank holds [b, s/(c*p)]: the context-parallel rank's two zigzag chunks
    (r, 2c-1-r), and of those the Ulysses rank's contiguous slice (``local_positions``).  The reference's real-data loader does this
    slicing before the model (Megatron ``get_batch_on_this_cp_rank``, models/llama_hf/dataloader.py:151, then the vocab_sp slice
    :45-57); here the first and the last layer do it, so ``forward_backward`` takes the same full-sequence batch in every mode."""
    c, p = _size(group), _size(sp_group)
    if c == 1 and p == 1:
        return x
    idx = local_positions(x.shape[1], c, group.rank_in_group() if c > 1 else 0, p, sp_group.rank_in_group() if p > 1 else 0)
    if c == 1:      # one contiguous slice
        return x[:, int(idx[0]):int(idx[-1]) + 1].contiguous()
    return x[:, idx.to(x.device)].contiguous()


def token_runs(positions):
    """Global token positions of a rank's rows (row order) -> the maximal runs of consecutive tokens, ((first row, rows, first
    token), ...).  A zigzag rank's rows are at most two runs, and so is any contiguous slice of them (Megatron-SP, Ulysses)."""
    pos = [int(t) for t in positions]
    runs, start = [], 0
    for i in range(1, len(pos) + 1):
        if i == len(pos) or pos[i] != pos[i - 1] + 1:
            runs.append((start, i - start, pos[start]))
            start = i
    return tuple(runs)


def _reverse_zigzag_transformation(x, cp):
    if cp == 1:
        return x
    fwd = _zigzag_indices(cp)
    inv = [0] * (2 * cp)
    for pos, src in enumerate(fwd):
        inv[src] = pos
    chunks = x.reshape(2 * cp, -1, *x.shape[1:])
    return torch.cat([chunks[i] for i in inv]).reshape(-1, *x.shape[1:])


def _gather_first_dim(x, group):
    if _size(group) == 1:
        return x
    be = get_backend()
    if x.is_floating_point():
        return be.all_gather_first_dim(x.contiguous(), group)
    # integer payloads (tokens / labels): move the bytes as fp32 words
    flat = x.contiguous()
    words = flat.view(torch.float32) if flat.element_size() % 4 == 0 else None
    if words is None:
        raise TypeError("relocation of %s tensors is not supported" % x.dtype)
    words = words.reshape(x.shape[0], -1)
    out = be.all_gather_first_dim(words, group)
    return out.view(x.dtype).reshape(x.shape[0] * group.size, *x.shape[1:])


def _split_first_dim(x, group):
    n = _size(group)
    if n == 1:
        return x
    assert x.shape[0] % n == 0, "First dimension of the tensor should be divisible by the group size"
    r, loc = group.rank_in_group(), x.shape[0] // n
    return x[r * loc:(r + 1) * loc].contiguous()


def _relocate_plain(x, fused_allgather_group, fused_split_group):
    """is_input=False path (:231-267): batch split or gather only."""
    if fused_split_group is not None:
        return _split_first_dim(x, fused_split_group)
    if fused_allgather_group is not None:
        return _gather_first_dim(x, fused_allgather_group)
    return x


def _relocate_float(x, allgather_cp_group, allgather_sep_group, split_cp_group, split_sep_group, fused_allgather_group,
                    fused_split_group, sequence_parallel, sbh):
    if sequence_parallel and _size(split_sep_group) > 1:
        x = _gather_first_dim(x, split_sep_group)
    # Reference quirk g1: gen_redistributed_group_with_cp returns (tp_old, tp_new, cp_new, cp_old) but is unpacked as
    # (split_tp_sp, allgather_tp_sp, split_cp, allgather_cp) (comm_groups.py:306 vs :483), so ``split_cp_group`` is the NEW layer's
    # context-parallel group and ``allgather_cp_group`` the OLD one.  The mapping is kept bit-exact (goldens); the reference then
    # reads the sizes the other way round (redistribute.py:290-296) and applies the wrong token permutation whenever the cp
    # degree changes between two rows.  Here the sizes are read for what the slots actually hold, which makes mixed-cp
    # strategies numerically correct (tests: cp_mixed_* in tests/test_host_runtime.py).
    old_cp, new_cp = _size(allgather_cp_group), _size(split_cp_group)
    if old_cp != new_cp:
        x = _reverse_zigzag_transformation(x, old_cp)
        x = _zigzag_transformation(x, new_cp)
    if fused_split_group is not None or fused_allgather_group is not None:
        if sbh:
            x = x.transpose(0, 1)           # "s b h -> b s h"
        if fused_split_group is not None:
            x = _split_first_dim(x.contiguous(), fused_split_group)
        if fused_allgather_group is not None:
            x = _gather_first_dim(x.contiguous(), fused_allgather_group)
        if sbh:
            x = x.transpose(0, 1)           # "b s h -> s b h"
    if sequence_parallel and _size(allgather_sep_group) > 1:
        x = _split_first_dim(x, allgather_sep_group)
    return x.contiguous()


class _Fused_split_allgather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input_, is_input, allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group, split_tp_sp_group,
                split_cp_group, split_tp_sp_cp_group, fused_allgather_group, fused_split_group, sequence_parallel, sbh):
        ctx.args = (is_input, allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group, split_tp_sp_group,
                    split_cp_group, split_tp_sp_cp_group, fused_allgather_group, fused_split_group, sequence_parallel, sbh)
        if not is_input:
            return _relocate_plain(input_, fused_allgather_group, fused_split_group)
        return _relocate_float(input_, allgather_cp_group, allgather_tp_sp_cp_group, split_cp_group, split_tp_sp_cp_group,
                               fused_allgather_group, fused_split_group, sequence_parallel, sbh)

    @staticmethod
    def backward(ctx, grad_output):
        (is_input, ag_tp_sp, ag_cp, ag_sep, sp_tp_sp, sp_cp, sp_sep, fused_ag, fused_sp, seqpar, sbh) = ctx.args
        if not is_input:
            g = _relocate_plain(grad_output, fused_sp, fused_ag)
        else:  # roles swapped: what was split is gathered and vice versa (:403-409)
            g = _relocate_float(grad_output, sp_cp, sp_sep, ag_cp, ag_sep, fused_sp, fused_ag, seqpar, sbh)
        return (g,) + (None,) * 11


def fused_split_allgather(input_, is_input, allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group,
                          split_tp_sp_group, split_cp_group, split_tp_sp_cp_group, fused_allgather_group, fused_split_group):
    from .arguments import get_args
    args = get_args()
    return _Fused_split_allgather.apply(input_, is_input, allgather_tp_sp_group, allgather_cp_group, allgather_tp_sp_cp_group,
                                        split_tp_sp_group, split_cp_group, split_tp_sp_cp_group, fused_allgather_group,
                                        fused_split_group, bool(args.sequence_parallel), args.shape_order == "SBH")
