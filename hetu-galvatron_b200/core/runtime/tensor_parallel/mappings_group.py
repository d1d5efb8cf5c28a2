"""Group-explicit autograd collectives -- same names and forward/backward pairing as
``galvatron/site_package/megatron/core/tensor_parallel/mappings_group.py:11-282`` (Galvatron's addition to Megatron).

Every primitive is an identity for a group of one rank (:15,30,49,70,92,109).  The data movement itself is the
peer-memory kernel behind ``backend.all_reduce / all_gather_* / reduce_scatter_*`` (one-shot/two-shot all-reduce,
pull all-gather, pull reduce-scatter over NVLink), not an NCCL call.
"""
import torch

from ..backend import get_backend


def get_tensor_model_parallel_world_size_group(group):
    return 1 if group is None else group.size


def get_tensor_model_parallel_rank_group(group):
    return 0 if group is None else group.rank_in_group()


def _size(group):
    return 1 if group is None else group.size


def _reduce(input_, group):
    """All-reduce the input tensor across the group (:11-21)."""
    if _size(group) == 1:
        return input_
    return get_backend().all_reduce(input_, group)


def _split_along_last_dim(input_, group):
    """Keep this rank's slice of the last dimension (:24-41)."""
    n = _size(group)
    if n == 1:
        return input_
    last = input_.shape[-1]
    assert last % n == 0
    r = group.rank_in_group()
    return input_[..., r * (last // n):(r + 1) * (last // n)].contiguous()


def _split_along_first_dim(input_, group):
    """Keep this rank's slice of the first dimension (:44-60)."""
    n = _size(group)
    if n == 1:
        return input_
    dim = input_.shape[0]
    assert dim % n == 0, "First dimension of the tensor should be divisible by tensor parallel size"
    r = group.rank_in_group()
    return input_[r * (dim // n):(r + 1) * (dim // n)].contiguous()


def _gather_along_last_dim(input_, group):
    if _size(group) == 1:
        return input_
    return get_backend().all_gather_last_dim(input_, group)


def _gather_along_first_dim(input_, group):
    if _size(group) == 1:
        return input_
    return get_backend().all_gather_first_dim(input_, group)


def _reduce_scatter_along_first_dim(input_, group):
    if _size(group) == 1:
        return input_
    return get_backend().reduce_scatter_first_dim(input_, group)


class _CopyToModelParallelRegion(torch.autograd.Function):
    """identity forward, all-reduce backward (:125-139; the column-parallel dgrad all-reduce, C6)."""

    @staticmethod
    def forward(ctx, input_, group):
        ctx.group = group
        return input_

    @staticmethod
    def backward(ctx, grad_output):
        return _reduce(grad_output, ctx.group), None


class _ReduceFromModelParallelRegion(torch.autograd.Function):
    """all-reduce forward, identity backward (:142-156; the row-parallel forward all-reduce, C5)."""

    @staticmethod
    def forward(ctx, input_, group):
        return _reduce(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        return grad_output, None


class _ScatterToModelParallelRegion(torch.autograd.Function):
    """split last dim forward, gather last dim backward (:159-174)."""

    @staticmethod
    def forward(ctx, input_, group):
        ctx.group = group
        return _split_along_last_dim(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        return _gather_along_last_dim(grad_output, ctx.group), None


class _GatherFromModelParallelRegion(torch.autograd.Function):
    """gather last dim forward, split backward (:177-192)."""

    @staticmethod
    def forward(ctx, input_, group):
        ctx.group = group
        return _gather_along_last_dim(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        return _split_along_last_dim(grad_output, ctx.group), None


class _ScatterToSequenceParallelRegion(torch.autograd.Function):
    """split first dim forward, gather first dim backward (:195-210)."""

    @staticmethod
    def forward(ctx, input_, group):
        ctx.group = group
        return _split_along_first_dim(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        return _gather_along_first_dim(grad_output, ctx.group), None


class _GatherFromSequenceParallelRegion(torch.autograd.Function):
    """gather first dim forward; backward reduce-scatters when the consumer computed in tensor parallel, else
    splits (:213-240)."""

    @staticmethod
    def forward(ctx, input_, group, tensor_parallel_output_grad=True):
        ctx.group, ctx.tp_grad = group, tensor_parallel_output_grad
        return _gather_along_first_dim(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        if ctx.tp_grad:
            return _reduce_scatter_along_first_dim(grad_output, ctx.group), None, None
        return _split_along_first_dim(grad_output, ctx.group), None, None


class _ReduceScatterToSequenceParallelRegion(torch.autograd.Function):
    """reduce-scatter forward (C8), gather backward (:243-258)."""

    @staticmethod
    def forward(ctx, input_, group):
        ctx.group = group
        return _reduce_scatter_along_first_dim(input_, group)

    @staticmethod
    def backward(ctx, grad_output):
        return _gather_along_first_dim(grad_output, ctx.group), None


def copy_to_tensor_model_parallel_region_group(input_, group):
    return _CopyToModelParallelRegion.apply(input_, group)


def reduce_from_tensor_model_parallel_region_group(input_, group):
    return _ReduceFromModelParallelRegion.apply(input_, group)


def scatter_to_tensor_model_parallel_region_group(input_, group):
    return _ScatterToModelParallelRegion.apply(input_, group)


def gather_from_tensor_model_parallel_region_group(input_, group):
    return _GatherFromModelParallelRegion.apply(input_, group)


def scatter_to_sequence_parallel_region_group(input_, group):
    return _ScatterToSequenceParallelRegion.apply(input_, group)


def gather_from_sequence_parallel_region_group(input_, group, tensor_parallel_output_grad=True):
    return _GatherFromSequenceParallelRegion.apply(input_, group, tensor_parallel_output_grad)


def reduce_scatter_to_sequence_parallel_region_group(input_, group):
    return _ReduceScatterToSequenceParallelRegion.apply(input_, group)
