"""The dropout pair at an explicit sample map (bg_dropout_add_fwd_ids / bg_dropout_bwd_ids through CudaBackend) on the GPU, against the
numpy Philox restatement of tests/_dropout_ref.py at GPT-2.7B (h 2560) and BERT-large (h 1024) row shapes: masks, forward output and
dx bit-identical, dbias within fp32 summation error, and bit-identical to the sample_base entries when the ids are one run.  The
entries' status codes, with and without a device.  And the relocated-layer cases of tests/test_dropout_relocation.py end to end on
CudaBackend (they skip below the GPU count they need)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _dropout_ref as dref  # noqa: E402
from test_dropout_relocation import CASES, VIT_CASE, launch  # noqa: E402

BF = torch.bfloat16


def _need(n):
    if not torch.cuda.is_available() or torch.cuda.device_count() < n:
        pytest.skip("needs %d GPU(s)" % n)


@pytest.fixture(scope="module")
def be():
    _need(1)
    from hetu_galvatron_b200.core.runtime import world
    from hetu_galvatron_b200.core.runtime.backend import CudaBackend
    world.get_rank()
    b = CudaBackend(arena_bytes=1 << 24)
    yield b
    b.close()


# (name, s, b, h): a gathered microbatch of the GPT-2.7B strategy (two ranks' 4 samples) and of a BERT-large one (two ranks' 8)
SHAPES = [("gpt_2.7b", 48, 8, 2560), ("bert_large", 40, 16, 1024)]


def _ids(kind, b):
    if kind == "two_runs":          # microbatch 1 of 2 of data-parallel ranks 0 and 1, local batch b
        return [b // 2 + i for i in range(b // 2)] + [b + b // 2 + i for i in range(b // 2)]
    if kind == "strided":
        return [3 + 5 * i for i in range(b)]
    if kind == "reversed":
        return [1000 + b - 1 - i for i in range(b)]
    raise ValueError(kind)


def _keep(seed, it, site, s, ids, h, p, seq_base):
    return dref.keep_mask(seed, it, site, seq_base + np.arange(s), np.asarray(ids, dtype=np.uint32), h, p)


def _dev_ids(ids):
    return torch.tensor(ids, dtype=torch.int32, device="cuda")


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize("kind", ["two_runs", "strided", "reversed"])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_mapped_forward_and_backward_bit_identical(be, shape, kind, p):
    _, s, b, h = shape
    seed, it, site, seq_base = 1234, 3, 7, 96
    ids = _ids(kind, b)
    g = torch.Generator().manual_seed(h + b)
    x, r, dy = (torch.randn(s, b, h, generator=g).to(BF) for _ in range(3))
    keep = _keep(seed, it, site, s, ids, h, p, seq_base)
    dids = _dev_ids(ids)
    ones = torch.ones(s, b, h, dtype=BF, device="cuda")
    assert torch.equal(be.dropout_add_fwd_ids(ones, None, None, p, seed, it, site, seq_base, dids).cpu() != 0, keep)
    for bias in (None, torch.randn(h, generator=g), torch.randn(h, generator=g).to(BF)):
        for res in (None, r):
            got = be.dropout_add_fwd_ids(x.cuda(), None if bias is None else bias.cuda(), None if res is None else res.cuda(), p, seed, it,
                                         site, seq_base, dids).cpu()
            want = dref.dropout_add_ref(x, bias, res, keep, p)
            assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    dx, db = be.dropout_bwd_ids(dy.cuda(), p, seed, it, site, seq_base, dids, with_bias=True)
    want_dx, want_db = dref.dropout_bwd_ref(dy, keep, p)
    assert torch.equal(dx.cpu().view(torch.int16), want_dx.view(torch.int16))
    tol = 1e-5 * (dy.float().abs().reshape(-1, h).sum(0) / (1 - p)) + 1e-6
    assert ((db.cpu() - want_db).abs() <= tol).all()
    dx2, none = be.dropout_bwd_ids(dy.cuda(), p, seed, it, site, seq_base, dids, with_bias=False)
    assert none is None and torch.equal(dx2, dx)


@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_contiguous_ids_equal_the_sample_base_entries(be, shape):
    _, s, b, h = shape
    seed, it, site, seq_base, base, p = 77, 1, 4, 0, 40, 0.1
    g = torch.Generator().manual_seed(3)
    x, r, dy = (torch.randn(s, b, h, generator=g).to(BF).cuda() for _ in range(3))
    bias = torch.randn(h, generator=g).cuda()
    dids = _dev_ids(list(range(base, base + b)))
    assert torch.equal(be.dropout_add_fwd_ids(x, bias, r, p, seed, it, site, seq_base, dids),
                       be.dropout_add_fwd(x, bias, r, p, seed, it, site, seq_base, base))
    dx_i, db_i = be.dropout_bwd_ids(dy, p, seed, it, site, seq_base, dids, with_bias=True)
    dx_b, db_b = be.dropout_bwd(dy, p, seed, it, site, seq_base, base, with_bias=True)
    assert torch.equal(dx_i, dx_b) and torch.equal(db_i, db_b)       # same grid, same per-CTA sums


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_mapped_entries_reject_bad_ids_on_the_device(be):
    L, s, b, h = be.bg.lib(), 4, 2, 64
    x, y = torch.zeros(s, b, h, dtype=BF, device="cuda"), torch.empty(s, b, h, dtype=BF, device="cuda")
    ids = torch.zeros(4, dtype=torch.int32, device="cuda")
    for ptr in (None, ids.data_ptr() + 2):
        assert L.bg_dropout_add_fwd_ids(x.data_ptr(), None, 0, None, y.data_ptr(), s * b, h, b, 0, ptr, 0.1, 1, 0, 0, None) == -1
        assert b"sample_ids must be non-null and 4-B aligned" in L.bg_last_error()
        assert L.bg_dropout_bwd_ids(x.data_ptr(), y.data_ptr(), None, 1, s * b, h, b, 0, ptr, 0.1, 1, 0, 0, None) == -1
    with pytest.raises(AssertionError, match="sample_ids"):        # the backend checks the vector against the batch
        be.dropout_add_fwd_ids(x, None, None, 0.1, 1, 0, 0, 0, ids)


# Bad-argument calls of the two entries in a child process that sees no device, so a call that slipped past validation would fail at
# its launch (and be counted) instead of launching a kernel on a bad pointer.
_BAD_IDS_CALLS = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M, I4 = 0x10000, 0x10002, 0x10004       # 16-B aligned, 2-B aligned, 4-B aligned; never dereferenced
EINVAL = -1
out = []
def call(want_msg, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_last_error().decode(), L.bg_launch_count() - before],
                    want=[EINVAL, want_msg, 0]))
DF, DB = "bg_dropout_add_fwd_ids", "bg_dropout_bwd_ids"
def fwd(x=A, y=A, rows=8, h=768, b_loc=2, seq_base=0, ids=I4, p=0.1):
    return (x, None, 0, None, y, rows, h, b_loc, seq_base, ids, p, 1, 0, 0, None)
def bwd(dy=A, dx=A, n_partial=1, rows=8, h=768, b_loc=2, seq_base=0, ids=I4, p=0.1):
    return (dy, dx, None, n_partial, rows, h, b_loc, seq_base, ids, p, 1, 0, 0, None)
for ids in (None, M):
    call(DF + ": sample_ids must be non-null and 4-B aligned", DF, *fwd(ids=ids))
    call(DB + ": sample_ids must be non-null and 4-B aligned", DB, *bwd(ids=ids))
call(DF + ": x and y must be non-null; 16-B alignment", DF, *fwd(x=None))
call(DF + ": x and y must be non-null; 16-B alignment", DF, *fwd(y=M))
call(DB + ": dy and dx must be non-null; 16-B alignment", DB, *bwd(dx=None))
call(DB + ": n_partial 0 must be in [1, 65535]", DB, *bwd(n_partial=0))
for name, f in ((DF, fwd), (DB, bwd)):
    call(name + ": hidden 12 must be a positive multiple of 8", name, *f(h=12))
    call(name + ": rows 9 must be a multiple of b_loc 2", name, *f(rows=9))
    call(name + ": token / sample coordinates must fit 32 bits", name, *f(seq_base=-1))
    call(name + ": dropout probability 1 must be in [0, 1)", name, *f(p=1.0))
print(json.dumps(out))
"""


def test_mapped_entries_reject_bad_arguments_without_a_device():
    """The existing dropout checks (shape, coordinates, probability, pointers, partials) and a null or not 4-B aligned sample map,
    all before any launch."""
    import __graft_entry__ as ge
    from hetu_galvatron_b200 import _bg
    if not os.path.exists(_bg.LIB_PATH):
        ge.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_IDS_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(calls) == 4 + 4 + 2 * 4
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("name", sorted(CASES))
def test_relocated_dropout_matches_the_oracle_on_gpus(name):
    world, cfg = CASES[name]
    _need(world)
    rep = launch(world, dict(cfg), backend="cuda")
    assert rep["max_grad_err"] < 3e-2 and rep["launches"] > 0
    assert abs(rep["loss_step1"] - rep["ref_loss_step1"]) <= 5e-3 * abs(rep["ref_loss_step1"])


@pytest.mark.gpu
@pytest.mark.timeout(1800)
def test_vit_relocated_dropout_matches_the_oracle_on_gpus():
    world, cfg = VIT_CASE
    _need(world)
    rep = launch(world, dict(cfg), backend="cuda")
    assert rep["max_grad_err"] < 3e-2
