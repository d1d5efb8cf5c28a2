"""GPU checks of tied word embeddings across pipeline stages (C14): the in-place pair sum over peer memory and the CUDA path end to end.

* ``bg_pair_sum_inplace`` for two virtual ranks on one device, on registered regions at different arena offsets: bf16 and fp32,
  scale 1 and 0.5, from one 16-B vector up to half the GPT-3 6.7B embedding (50257 x 4096 / 2 elements).  Both members end
  bit-identical and equal to torch's fp32 sum rounded once; three back-to-back calls on the same lane all land (the barrier flags
  reset themselves); bad arguments come back as status codes; registrations of different sizes are refused at ``exchange()``.
* The GPT family with tied embeddings through the CUDA backend against the HF-pinned oracle (tests/test_families.py's cases, and
  tests/test_tied_embeddings.py's).  Across pipeline stages the report must show the pair-sum kernel ran and no staging
  buffer the size of the matrix was reserved for the embedding group.  Cases skip below the GPU count they need.  (The context-parallel
  ``cp2_tied`` runs in tests/test_gpu_gpt_cp.py.)"""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

GPT3_HALF = 50257 * 4096 // 2
SIZES = [8, 24, 8 * 1000 + 8, 1 << 20, GPT3_HALF]       # elements (multiples of 8: whole vectors in bf16 and fp32)


def _need(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip("needs %d GPU(s)" % n)


@pytest.fixture(scope="module")
def pair():
    """two virtual ranks, a region of the largest fp32 size on each, member 0's 4 KiB further into its arena than member 1's; one
    registered buffer per (dtype, size) over the start of that region"""
    _need(1)
    from hetu_galvatron_b200 import _bg as bg
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    bg.lib()
    bg.set_tunable("timeout_ms", 20000)
    nbytes = GPT3_HALF * 4
    comms = bg.BgComm.local_world(2, device=0, arena_bytes=nbytes + (8 << 20))
    grp = CommGroup([0, 1])
    comms[0].alloc(4096)
    regions = [c.alloc(nbytes) for c in comms]
    bufs = {}
    for dt in (torch.bfloat16, torch.float32):
        for n in SIZES:
            esz = torch.empty((), dtype=dt).element_size()
            bufs[(dt, n)] = [c.sym_register(grp, off, n * esz) for c, (off, _) in zip(comms, regions)]
    for c in comms:
        c.exchange()
    assert bufs[(torch.float32, 8)][0].offs()[0] != bufs[(torch.float32, 8)][0].offs()[1]
    yield bg, comms, grp, bufs
    torch.cuda.synchronize()
    for c in comms:
        c.close()


@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_pair_sum_bit_exact(pair, dt, n, scale):
    bg, comms, grp, bufs = pair
    views = [b.view(dt, n) for b in bufs[(dt, n)]]
    gen = torch.Generator(device="cuda").manual_seed(n)
    xs = [torch.randn(n, device="cuda", generator=gen).to(dt) for _ in range(2)]
    for v, x in zip(views, xs):
        v.copy_(x)
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in comms]
    for _ in range(3):            # back to back on one lane, no host synchronisation in between
        for c, b, s in zip(comms, bufs[(dt, n)], streams):
            c.pair_sum_inplace(grp, b, dt, scale=scale, stream=s)
    torch.cuda.synchronize()
    assert all(c.error_flag() == 0 for c in comms)
    want = xs
    for _ in range(3):
        y = ((want[0].float() + want[1].float()) * scale).to(dt)
        want = [y, y]
    bits = torch.int16 if dt == torch.bfloat16 else torch.int32
    assert torch.equal(views[0].view(bits), views[1].view(bits))
    assert torch.equal(views[0].view(bits), want[0].view(bits))


def test_pair_sum_bad_arguments_are_status_codes(pair):
    bg, comms, grp, bufs = pair
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    b = bufs[(torch.bfloat16, 24)][0]
    with pytest.raises(bg.BgError, match="not a whole number"):
        comms[0].pair_sum_inplace(grp, b, torch.bfloat16, elems=12)
    rc = bg.lib().bg_pair_sum_inplace(comms[0]._ctx, comms[0].group_id(grp), bg.LANE_REDUCE, b.offs(), 8, 7, 1.0, None)
    assert rc == -7                                      # BG_EUNSUPPORTED: an unknown dtype
    solo = CommGroup([0])
    s = comms[0].sym_register(solo, b.offset, 64)
    with pytest.raises(bg.BgError, match="exactly 2"):
        comms[0].pair_sum_inplace(solo, s, torch.bfloat16)
    with pytest.raises(bg.BgError, match="16-B aligned"):
        comms[0].sym_register(grp, b.offset + 8, 64)


def test_registered_sizes_must_match_at_exchange():
    _need(1)
    from hetu_galvatron_b200 import _bg as bg
    from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup
    comms = bg.BgComm.local_world(2, device=0, arena_bytes=4 << 20)
    try:
        grp = CommGroup([0, 1])
        for c, nbytes in zip(comms, (4096, 8192)):      # e.g. the embedding row and the head row sharded differently
            off, _ = c.alloc(8192)
            c.sym_register(grp, off, nbytes)
        with pytest.raises(bg.BgError, match="same size"):
            comms[0].exchange()
    finally:
        for c in comms:
            c.close()


# ---- the GPT family through the CUDA backend -------------------------------------------------------------------------------------
def _cases():
    from test_families import CASES as FAMILY
    from test_tied_embeddings import CASES as TIED
    cases = {k: v for k, v in FAMILY.items() if k.startswith("gpt_tied_")}
    cases.update(TIED)
    return cases


CASES = _cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_gpt_tied_cuda(name):
    world, cfg = CASES[name]
    _need(world)
    from test_tied_embeddings import launch
    rep = launch(world, dict(cfg), backend="cuda")
    assert rep["tied"] and rep["launches"] > 0
    assert rep["max_grad_err"] < cfg.get("_tol", 3e-2)
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])
    if cfg.get("pp_deg", 1) > 1:
        # rank 0 is on the first stage: it registered its tied gradient range over the embedding group and ran the pair sum
        (ranks, nbytes), = rep["tied_registered"]
        assert rep["fused_calls"].get("tied_pair_sum", 0) > 0
        assert rep["staging"].get(",".join(str(r) for r in ranks), 0) < nbytes, rep["staging"]
    else:
        assert rep["tied_registered"] == [] and "tied_pair_sum" not in rep["fused_calls"]
