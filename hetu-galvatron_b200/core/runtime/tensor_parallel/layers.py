"""Tensor-parallel linear / embedding layers with an explicit ``tp_group`` -- the operator API of
``galvatron/site_package/megatron/core/tensor_parallel/layers.py`` (``VocabParallelEmbedding`` :166,
``LinearWithGradAccumulationAndAsyncCommunication`` :375, ``ColumnParallelLinear`` :651, ``RowParallelLinear`` :927).

What differs from the reference is where the bytes go, not the math:
  * the GEMMs are the wgmma kernel (``backend.gemm``), and a GEMM whose result is about to be reduced writes it
    straight into the TP group's peer-visible staging buffer, so the all-reduce / reduce-scatter kernel pulls it over
    NVLink with no intermediate copy (reference: cuBLAS, then a separate NCCL kernel on the same stream);
  * the Megatron-SP all-gather lands in that staging buffer too and is consumed in place by the GEMM (reference: a
    global scratch buffer, ``megatron/core/utils.py:62-80``);
  * wgrad accumulates directly into the layer's flat bf16 gradient buffer (``weight._bg_grad``) that the sharded
    data-parallel unit reduce-scatters -- Megatron's ``gradient_accumulation_fusion`` idea without apex.
"""
import math

import torch
import torch.nn as nn

from ..backend import get_backend
from .mappings_group import (_reduce, copy_to_tensor_model_parallel_region_group,
                             gather_from_tensor_model_parallel_region_group,
                             reduce_from_tensor_model_parallel_region_group,
                             reduce_scatter_to_sequence_parallel_region_group,
                             scatter_to_tensor_model_parallel_region_group)


def _size(group):
    return 1 if group is None else group.size


def _rank(group):
    return 0 if group is None or group.size == 1 else group.rank_in_group()


class VocabUtility:
    """``megatron/core/tensor_parallel/utils.py`` VocabUtility: contiguous [first, last) slice per rank."""

    @staticmethod
    def vocab_range_from_per_partition_vocab_size(per_partition, rank, world_size):
        return rank * per_partition, (rank + 1) * per_partition

    @staticmethod
    def vocab_range_from_global_vocab_size(global_size, rank, world_size):
        assert global_size % world_size == 0, "{} is not divisible by {}".format(global_size, world_size)
        return VocabUtility.vocab_range_from_per_partition_vocab_size(global_size // world_size, rank, world_size)


def _write_wgrad(weight, dy2d, x2d):
    """dW = dy^T x, accumulated into the flat gradient buffer when the weight belongs to a sharded unit."""
    be = get_backend()
    sink = getattr(weight, "_bg_grad", None)
    if sink is None:
        return be.gemm(dy2d, x2d, "nt")
    unit = weight._bg_unit
    if sink.dtype == dy2d.dtype:
        be.gemm(dy2d, x2d, "nt", out=sink, accumulate=unit.grad_started(weight))
    else:
        # --reduce_in_fp32: the unsharded gradient buffer is fp32 (arguments.py:187); the wgmma GEMM writes bf16, so the wgrad
        # goes through a bf16 tile buffer and the cast kernel accumulates it into the fp32 buffer
        tmp = be.gemm(dy2d, x2d, "nt")
        be.cast(tmp, sink, accumulate=unit.grad_started(weight))
    unit.mark_grad(weight)
    return None


class LinearWithGradAccumulationAndAsyncCommunication(torch.autograd.Function):
    """y = x W^T with the tensor/sequence-parallel communication of layers.py:375-547.

    sequence_parallel: all-gather x along dim 0 before the GEMM (:399-413), re-gather in backward (:449-455) and
        reduce-scatter dgrad (:488-494).
    allreduce_dgrad:   all-reduce dgrad over the TP group (what ``copy_to_tensor_model_parallel_region`` does in
        backward, mappings_group.py:139).
    allreduce_out:     all-reduce y over the TP group (row-parallel forward, :1110-1114; identity in backward).
    reduce_scatter_out: reduce-scatter y along the sequence (row-parallel forward under Megatron-SP, :1109); backward gathers dy.
    recompute:         (opt-in, ``--recompute_activations``) instead of saving ``input`` for the wgrad GEMM, save what it was made
        from -- ("swiglu", gate_up) or ("rmsnorm", x, norm_weight, eps), tensors the producing op keeps anyway -- and redo that
        elementwise pass in backward: one layer then holds 352 MiB less at Llama-3-8B / seq 8192.

    Every GEMM that has a collective next to it is one backend operation, which runs as ONE fused kernel pair when the shapes allow
    (M a multiple of p x 128) and otherwise writes the GEMM into the group's peer-visible staging buffer and runs the stand-alone
    collective kernel after it:
      all-gather -> GEMM        ``backend.all_gather_gemm``      (C7: SP forward; the row-parallel dgrad under SP)
      GEMM -> reduce-scatter    ``backend.gemm_reduce_scatter``  (C8: row-parallel forward under SP; the SP dgrad)
      GEMM -> all-reduce        ``backend.gemm_all_reduce``      (C5: row-parallel forward; C6: column-parallel dgrad)
    """

    @staticmethod
    def forward(ctx, input, weight, sequence_parallel, allreduce_dgrad, allreduce_out, tp_group, reduce_scatter_out=False,
                recompute_kind=None, recompute_eps=0.0, addend=None, *recipe):
        # addend: a tensor of the OUTPUT's shape added to it (the residual of the block: `out + residual`).  When no collective
        # follows the GEMM it rides in the GEMM epilogue (fp32 accumulator + addend, one rounding, no elementwise pass).
        be = get_backend()
        ctx.has_addend = addend is not None
        ctx.recompute = (recompute_kind, recompute_eps, len(recipe)) if recompute_kind else None
        if ctx.recompute:
            ctx.save_for_backward(weight, *recipe)
        else:
            ctx.save_for_backward(input, weight)
        multi = _size(tp_group) > 1
        ctx.tp_group = tp_group
        ctx.reduce_scatter_out = reduce_scatter_out and multi
        n_out = weight.shape[0]
        if ctx.reduce_scatter_out:
            # row-parallel forward under Megatron-SP (layers.py:1061-1109): GEMM + reduce-scatter along the sequence
            ctx.sequence_parallel, ctx.allreduce_dgrad = False, False
            x2d = input.reshape(-1, input.shape[-1])
            out = be.gemm_reduce_scatter(x2d, weight, "tn", tp_group)
            out = out.view(input.shape[0] // tp_group.size, *input.shape[1:-1], n_out)
            return out if addend is None else out + addend
        ctx.sequence_parallel = sequence_parallel and multi
        ctx.allreduce_dgrad = allreduce_dgrad and multi
        if ctx.sequence_parallel:
            x2d = input.reshape(-1, input.shape[-1])
            full_shape = (input.shape[0] * tp_group.size,) + tuple(input.shape[1:-1])
            out, _ = be.all_gather_gemm(x2d.contiguous(), weight, "tn", tp_group)
            out = out.view(*full_shape, n_out)
            return out if addend is None else out + addend
        x2d = input.reshape(-1, input.shape[-1])
        if allreduce_out and multi:
            out = be.gemm_all_reduce(x2d, weight, "tn", tp_group).view(*input.shape[:-1], n_out)
            return out if addend is None else out + addend
        if addend is not None:
            return be.gemm(x2d, weight, "tn", addend=addend.contiguous().reshape(-1, n_out)).view(*input.shape[:-1], n_out)
        return be.gemm(x2d, weight, "tn").view(*input.shape[:-1], n_out)

    @staticmethod
    def backward(ctx, grad_output):
        be = get_backend()
        if ctx.recompute:
            kind, eps, n_recipe = ctx.recompute
            weight, recipe = ctx.saved_tensors[0], ctx.saved_tensors[1:]
            if kind == "swiglu":
                input = be.swiglu_fwd(recipe[0])
            elif kind == "rmsnorm":
                input, _ = be.rmsnorm_fwd(recipe[0], recipe[1], eps)
            else:
                raise ValueError("unknown recompute recipe %r" % (kind,))
        else:
            n_recipe = 0
            input, weight = ctx.saved_tensors
        group = ctx.tp_group
        k = weight.shape[1]
        ctx.saved_grad_output = grad_output if ctx.has_addend else None      # d(out + addend) / d(addend) = identity
        grad_input, dgrad_done, gather_event = None, False, None
        if ctx.reduce_scatter_out:
            # backward of the reduce-scatter is an all-gather along the sequence (mappings_group.py:243-258); the dgrad GEMM
            # consumes the gathered dy block by block while it arrives, and the wgrad GEMM reads it from staging afterwards
            dy_local = grad_output.reshape(-1, grad_output.shape[-1])
            if ctx.needs_input_grad[0] and be.fuses("ag_gemm", dy_local.shape[0] * group.size, k, dy_local.shape[1], group):
                gi, dy2d = be.all_gather_gemm(dy_local.contiguous(), weight, "nn", group)
                grad_input = gi.view(grad_output.shape[0] * group.size, *grad_output.shape[1:-1], k)
                dgrad_done = True
            else:
                grad_output = be.all_gather_first_dim(grad_output.contiguous(), group)
                dy2d = grad_output.reshape(-1, grad_output.shape[-1])
        else:
            dy2d = grad_output.reshape(-1, grad_output.shape[-1])
        if not dy2d.is_contiguous():
            dy2d = dy2d.contiguous()
        total = input
        if weight.requires_grad and ctx.sequence_parallel:
            if ctx.needs_input_grad[0] and be.fuses("gemm_rs", dy2d.shape[0], k, dy2d.shape[1], group):
                # the re-gather of the input (for wgrad) runs on the communication stream WHILE the fused dgrad GEMM +
                # reduce-scatter runs here (layers.py:449-462 overlaps the same pair); wgrad waits for it below
                total, gather_event = be.all_gather_into_staging(input, group, overlap=True)
            else:
                total = be.all_gather_into_staging(input, group)
        grad_weight = None
        if weight.requires_grad and gather_event is None:
            grad_weight = _write_wgrad(weight, dy2d, total.reshape(-1, total.shape[-1]))
        # dgrad_addend (set by _CrossKvFn): a gradient of the input's shape that arrives from elsewhere and is summed into the dgrad --
        # inside the GEMM epilogue when no collective follows it, else once after the collective (never once per rank)
        addend = getattr(ctx, "dgrad_addend", None)
        if ctx.needs_input_grad[0] and not dgrad_done:
            if ctx.sequence_parallel:
                # dgrad GEMM + reduce-scatter along the sequence (layers.py:462,488-494)
                out = be.gemm_reduce_scatter(dy2d, weight, "nn", group)
                grad_input = out.view(grad_output.shape[0] // group.size, *grad_output.shape[1:-1], k)
            elif ctx.allreduce_dgrad:
                grad_input = be.gemm_all_reduce(dy2d, weight, "nn", group).view(*grad_output.shape[:-1], k)
            elif addend is not None:
                grad_input = be.gemm(dy2d, weight, "nn", addend=addend.contiguous().reshape(-1, k)).view(*grad_output.shape[:-1], k)
                addend = None
            else:
                grad_input = be.gemm(dy2d, weight, "nn").view(*grad_output.shape[:-1], k)
        if addend is not None and grad_input is not None:
            grad_input = grad_input + addend
        if gather_event is not None:
            be.wait_event(gather_event)
            grad_weight = _write_wgrad(weight, dy2d, total.reshape(-1, total.shape[-1]))
        grad_addend = ctx.saved_grad_output if ctx.has_addend else None
        return (grad_input, grad_weight, None, None, None, None, None, None, None, grad_addend) + (None,) * n_recipe


def linear_with_grad_accumulation_and_async_allreduce(input, weight, bias=None, gradient_accumulation_fusion=False,
                                                      async_grad_allreduce=False, sequence_parallel=False, tp_group=None,
                                                      allreduce_out=False, reduce_scatter_out=False, recompute=None, addend=None):
    """Same call shape as layers.py:550-648 (``async_grad_allreduce`` here means "all-reduce dgrad over tp_group").
    ``recompute``: None, ("swiglu", gate_up) or ("rmsnorm", x, norm_weight, eps) -- see the Function's docstring."""
    if recompute is None:
        out = LinearWithGradAccumulationAndAsyncCommunication.apply(input, weight, sequence_parallel, async_grad_allreduce,
                                                                    allreduce_out, tp_group, reduce_scatter_out, None, 0.0, addend)
    else:
        kind = recompute[0]
        eps = float(recompute[3]) if kind == "rmsnorm" else 0.0
        recipe = recompute[1:3] if kind == "rmsnorm" else recompute[1:2]
        out = LinearWithGradAccumulationAndAsyncCommunication.apply(input, weight, sequence_parallel, async_grad_allreduce,
                                                                    allreduce_out, tp_group, reduce_scatter_out, kind, eps, addend, *recipe)
    return out if bias is None else out + bias


def mark_tensor_parallel(param):
    """``set_tensor_model_parallel_attributes`` (layers.py:95-105): this parameter is a different slice on every rank of its
    tensor-parallel group.  Parameters WITHOUT the mark (norm weights, the row-parallel bias) are replicas -- the gradient-norm
    of ``clip_grad_norm`` counts them once (clip_grads.py:61-75 ``param_is_not_tensor_parallel_duplicate``)."""
    setattr(param, "tensor_model_parallel", True)
    return param


class _ParallelLinearBase(nn.Module):
    def _make_weight(self, rows, cols, init_std, params_dtype, device):
        self.weight = mark_tensor_parallel(nn.Parameter(torch.empty(rows, cols, dtype=params_dtype, device=device)))
        self.init_std = init_std
        if self.weight.device.type != "meta":
            self.reset_parameters()

    def reset_parameters(self):
        """``colummn_row_reset_parameters`` (tensor_parallel/reset.py:10-17): N(0, init_method_std), zero bias.
        (Parameter attributes are set here as well as at construction: materialising a meta module makes new Parameter objects.)"""
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        mark_tensor_parallel(self.weight)
        if getattr(self, "bias", None) is not None:
            nn.init.zeros_(self.bias)
            if isinstance(self, RowParallelLinear):
                setattr(self.bias, "sequence_parallel", self.sequence_parallel)  # layers.py:1045
            else:
                mark_tensor_parallel(self.bias)


class ColumnParallelLinear(_ParallelLinearBase):
    """Y = XA with A split along its output dimension over ``tp_group`` (layers.py:651-910)."""

    def __init__(self, input_size, output_size, *, config=None, init_method=None, bias=False, gather_output=False,
                 skip_bias_add=False, tp_group=None, sp_group=None, cp_group=None, sequence_parallel=None,
                 init_std=0.02, params_dtype=torch.float32, device=None):
        super().__init__()
        self.input_size, self.output_size, self.gather_output = input_size, output_size, gather_output
        self.tp_group, self.sp_group, self.cp_group = tp_group, sp_group, cp_group
        world = _size(tp_group)
        assert output_size % world == 0, "{} is not divisible by {}".format(output_size, world)
        self.output_size_per_partition = output_size // world
        self.skip_bias_add = skip_bias_add
        sp = getattr(config, "sequence_parallel", False) if sequence_parallel is None else sequence_parallel
        self.sequence_parallel = bool(sp) and world > 1
        if config is not None:
            init_std = getattr(config, "init_method_std", init_std)
        self._make_weight(self.output_size_per_partition, input_size, init_std, params_dtype, device)
        if bias:
            self.bias = mark_tensor_parallel(nn.Parameter(torch.zeros(self.output_size_per_partition, dtype=params_dtype, device=device)))
        else:
            self.register_parameter("bias", None)

    def forward(self, input_, recompute=None):
        bias = self.bias if not self.skip_bias_add else None
        # without SP the input is replicated: dgrad must be all-reduced (copy_to_tensor_model_parallel_region, :875)
        out = linear_with_grad_accumulation_and_async_allreduce(
            input_, self.weight, bias, async_grad_allreduce=not self.sequence_parallel,
            sequence_parallel=self.sequence_parallel, tp_group=self.tp_group, recompute=recompute)
        if self.gather_output:
            assert not self.sequence_parallel
            out = gather_from_tensor_model_parallel_region_group(out, self.tp_group)
        return out, (self.bias if self.skip_bias_add else None)


class RowParallelLinear(_ParallelLinearBase):
    """Y = XA with A split along its input dimension; output all-reduced (or reduce-scattered under SP)
    (layers.py:927-1121)."""

    def __init__(self, input_size, output_size, *, config=None, init_method=None, bias=False, input_is_parallel=True,
                 skip_bias_add=False, tp_group=None, sp_group=None, cp_group=None, sequence_parallel=None,
                 init_std=0.02, params_dtype=torch.float32, device=None):
        super().__init__()
        self.input_size, self.output_size, self.input_is_parallel = input_size, output_size, input_is_parallel
        self.tp_group, self.sp_group, self.cp_group = tp_group, sp_group, cp_group
        world = _size(tp_group)
        assert input_size % world == 0, "{} is not divisible by {}".format(input_size, world)
        self.input_size_per_partition = input_size // world
        self.skip_bias_add = skip_bias_add
        sp = getattr(config, "sequence_parallel", False) if sequence_parallel is None else sequence_parallel
        self.sequence_parallel = bool(sp) and world > 1
        if self.sequence_parallel and not input_is_parallel:
            raise RuntimeError("To enable `sequence_parallel`, `input_is_parallel` must be `True`")
        if config is not None:
            init_std = getattr(config, "output_layer_init_std", getattr(config, "init_method_std", init_std))
        self._make_weight(output_size, self.input_size_per_partition, init_std, params_dtype, device)
        if bias:
            self.bias = nn.Parameter(torch.zeros(output_size, dtype=params_dtype, device=device))
            setattr(self.bias, "sequence_parallel", self.sequence_parallel)  # layers.py:1045
        else:
            self.register_parameter("bias", None)

    def forward(self, input_, recompute=None, residual=None):
        """``residual``: added to the output (after the collective; inside the GEMM epilogue when there is none).  Only honoured
        when this layer adds no bias of its own before it (bias is None or skip_bias_add) -- the callers' contract."""
        if not self.input_is_parallel:
            input_ = scatter_to_tensor_model_parallel_region_group(input_, self.tp_group)
            recompute = None
        if residual is not None and not self.skip_bias_add and self.bias is not None:
            raise ValueError("residual fusion needs skip_bias_add (the bias would be added after the residual)")
        if self.sequence_parallel:
            # GEMM and the sequence reduce-scatter (:1109, C8) are one operation: partial tiles go straight to their owner
            out = linear_with_grad_accumulation_and_async_allreduce(
                input_, self.weight, None, async_grad_allreduce=False, sequence_parallel=False, tp_group=self.tp_group,
                reduce_scatter_out=True, recompute=recompute, addend=residual)
        else:
            # GEMM and the all-reduce of :1110-1114 (C5) are one operation; its backward is the identity, as
            # reduce_from_tensor_model_parallel_region's is (mappings_group.py:142-156)
            out = linear_with_grad_accumulation_and_async_allreduce(
                input_, self.weight, None, async_grad_allreduce=False, sequence_parallel=False, tp_group=self.tp_group,
                allreduce_out=True, recompute=recompute, addend=residual)
        if not self.skip_bias_add and self.bias is not None:
            out = out + self.bias
        return out, (self.bias if self.skip_bias_add else None)


class _VocabEmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, weight, vocab_start, vocab_end, masked):
        if masked:
            oob = (tokens < vocab_start) | (tokens >= vocab_end)
            idx = (tokens - vocab_start).masked_fill(oob, 0)
        else:
            oob, idx = None, tokens
        out = weight.index_select(0, idx.reshape(-1)).view(*tokens.shape, weight.shape[1])
        if masked:
            out.masked_fill_(oob.unsqueeze(-1), 0.0)
        ctx.save_for_backward(idx, oob if masked else torch.empty(0, device=tokens.device), weight)
        ctx.masked = masked
        return out

    @staticmethod
    def backward(ctx, grad_output):
        idx, oob, weight = ctx.saved_tensors
        g = grad_output.reshape(-1, grad_output.shape[-1])
        if ctx.masked:
            g = g.masked_fill(oob.reshape(-1, 1), 0.0)
        sink = getattr(weight, "_bg_grad", None)
        if sink is not None:
            unit = weight._bg_unit
            if not unit.grad_started(weight):
                sink.zero_()
            sink.index_add_(0, idx.reshape(-1), g.to(sink.dtype))
            unit.mark_grad(weight)
            return None, None, None, None, None
        dw = torch.zeros_like(weight)
        dw.index_add_(0, idx.reshape(-1), g.to(dw.dtype))
        return None, dw, None, None, None


class VocabParallelEmbedding(nn.Module):
    """Embedding split along the vocabulary over ``tp_group``; masked lookup + all-reduce (layers.py:166-262)."""

    def __init__(self, num_embeddings, embedding_dim, *, config=None, init_method=None, tp_group=None, sp_group=None,
                 cp_group=None, init_std=0.02, params_dtype=torch.float32, device=None):
        super().__init__()
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        self.tp_group, self.sp_group, self.cp_group = tp_group, sp_group, cp_group
        world = _size(tp_group)
        self.vocab_start_index, self.vocab_end_index = VocabUtility.vocab_range_from_global_vocab_size(
            num_embeddings, _rank(tp_group), world)
        self.num_embeddings_per_partition = self.vocab_end_index - self.vocab_start_index
        if config is not None:
            init_std = getattr(config, "init_method_std", init_std)
        self.init_std = init_std
        self.weight = mark_tensor_parallel(nn.Parameter(torch.empty(self.num_embeddings_per_partition, embedding_dim, dtype=params_dtype,
                                                                    device=device)))
        if self.weight.device.type != "meta":
            self.reset_parameters()

    def reset_parameters(self):
        nn.init.normal_(self.weight, mean=0.0, std=self.init_std)
        mark_tensor_parallel(self.weight)

    def forward(self, input_):
        masked = _size(self.tp_group) > 1
        out_parallel = _VocabEmbeddingFn.apply(input_, self.weight, self.vocab_start_index, self.vocab_end_index, masked)
        return reduce_from_tensor_model_parallel_region_group(out_parallel, self.tp_group)   # :261
