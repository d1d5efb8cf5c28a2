"""Which global samples each row of a hybrid-parallel model holds.

The batch enters the first row (the embedding) split contiguously over the data-parallel ranks of the vocabulary rows
(``vtp_data_group``): data-parallel index d holds samples d * local .. (d + 1) * local - 1, and microbatch (offset, size) of them
samples d * local + offset + 0 .. size - 1.  A relocation between two rows whose tensor / sequence-parallel degrees differ splits or
gathers the BATCH (redistribute.py, step 3), and pipeline stages pass a row's output to the same position of the next stage, so
after a few rows a rank can hold e.g. microbatch 1 of data-parallel ranks 0 and 1: samples that are not one run of consecutive
indices.  Dropout draws its masks at global sample indices, so every row needs to know which ones it holds.

A row's *layout* is an ordered tuple of pieces (d, lo, hi): the samples [lo * size, hi * size) of data-parallel index d's current
microbatch, with lo and hi fractions of the microbatch.  ``derive_sample_layouts`` builds them once, at model construction, by
replaying every relocation's split / gather over the groups' actual rank lists (``gen_comm_groups`` evaluated for every rank) on
the previous row's layouts, across pipeline stage boundaries too; ``instantiate`` turns one into global sample indices.
"""
from fractions import Fraction

from .comm_groups import gen_comm_groups


def _split(layout, n, k):
    """Part k of the concatenated pieces cut into n equal parts (``_split_first_dim``)."""
    total = sum(hi - lo for _, lo, hi in layout)
    a, b = total * k / n, total * (k + 1) / n
    out, pos = [], Fraction(0)
    for d, lo, hi in layout:
        s, e = max(a, pos), min(b, pos + hi - lo)
        if s < e:
            out.append((d, lo + s - pos, lo + e - pos))
        pos += hi - lo
    return _merge(out)


def _merge(layout):
    """Adjacent pieces of one data-parallel index that continue each other become one."""
    out = []
    for d, lo, hi in layout:
        if out and out[-1][0] == d and out[-1][2] == lo:
            out[-1] = (d, out[-1][1], hi)
        else:
            out.append((d, lo, hi))
    return tuple(out)


def derive_sample_layouts(hp_whole, rank, world):
    """{row: layout} for the rows ``rank`` holds (its pipeline stage's rows), from the whole-model strategy ``hp_whole``
    (``hp_config_whole_model``)."""
    tp, sp, cp = hp_whole["tp_sizes_whole"], hp_whole["sp_sizes_whole"], hp_whole["cp_sizes_whole"]
    pp, stages = hp_whole["pp_deg"], hp_whole["pp_ranks_whole"]
    per_stage = world // pp
    groups = {}

    def groups_of(q):       # (fused_allgather groups, fused_split groups, vtp_data_group) of rank q
        if q not in groups:
            g = gen_comm_groups(list(tp), list(sp), list(cp), pp, list(hp_whole["tp_consec_whole"]), rank=q, world_size=world)
            groups[q] = (g[12], g[13], g[15])
        return groups[q]

    memo = {}

    def entering(q, i):     # the layout of the activation that reaches row i on rank q, before row i's relocation
        if i == 0:
            return ((groups_of(q)[2].ranks.index(q), Fraction(0), Fraction(1)),)
        prev = q if stages[i - 1] == stages[i] else q - per_stage * (stages[i] - stages[i - 1])
        return layout(prev, i - 1)

    def layout(q, i):
        if (q, i) not in memo:
            fused_ag, fused_split, _ = groups_of(q)
            x = entering(q, i)
            if fused_split[i] is not None:
                x = _split(x, fused_split[i].size, fused_split[i].ranks.index(q))
            if fused_ag[i] is not None:
                x = _merge(piece for member in fused_ag[i].ranks for piece in entering(member, i))
            memo[(q, i)] = x
        return memo[(q, i)]

    stage = rank // per_stage
    return {i: layout(rank, i) for i in range(len(tp)) if stages[i] == stage}


def instantiate(layout, local, offset, size):
    """Global sample indices of a row, in its local batch order, for the microbatch (``offset``, ``size``) of a ``local``-sample
    data-parallel batch."""
    ids = []
    for d, lo, hi in layout:
        a, b = lo * size, hi * size
        if a.denominator != 1 or b.denominator != 1:
            raise ValueError("a relocation splits a %d-sample microbatch into unequal parts (layout %s)" % (size, layout))
        base = d * local + offset
        ids.extend(range(base + int(a), base + int(b)))
    return ids
