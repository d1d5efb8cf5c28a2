"""CPU checks of the C-ABI boundary: the library loads (no GPU calls), exports every symbol include/bg_galvatron.h
declares, reports errors through return codes, and its C mirror of the group builder is bit-exact with the goldens."""
import ctypes
import json
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bg():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    from hetu_galvatron_b200 import _bg
    if not os.path.exists(_bg.LIB_PATH):
        ge.build()
    _bg.lib()
    return _bg


def _declared_symbols():
    text = open(os.path.join(ROOT, "include", "bg_galvatron.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bg_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree(bg):
    declared = _declared_symbols()
    assert len(declared) >= 30
    assert sorted(bg.SIGNATURES) == declared
    handle = bg.lib()
    for name in declared:
        assert hasattr(handle, name), name


def test_exports_match_nm(bg):
    out = subprocess.run(["nm", "-D", "--defined-only", bg.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r"\bT (bg_[a-z0-9_]+)", out))
    assert set(_declared_symbols()) <= exported


def test_kernels_are_hopper_native(bg):
    """SASS evidence: wgmma.mma_async -> HGMMA, TMA -> UTMALDG/UTMASTG, all for sm_90a."""
    sass = subprocess.run(["cuobjdump", "-sass", bg.LIB_PATH], capture_output=True, text=True).stdout
    if not sass:
        pytest.skip("cuobjdump unavailable")
    for mnemonic in ("HGMMA", "UTMALDG", "UTMASTG"):
        assert mnemonic in sass, mnemonic
    assert "sm_90a" in sass


def test_errors_are_return_codes(bg):
    L = bg.lib()
    assert L.bg_set_tunable(b"no_such_tunable", 1) == -1
    assert b"unknown tunable" in L.bg_last_error()
    assert L.bg_set_tunable(b"comm_ctas", 100000) == -1
    assert L.bg_group_create(None, None, 0, None) == -1
    with pytest.raises(bg.BgError):
        bg.check(L.bg_arena_alloc(None, 16, None))
    assert bg.get_tunable("comm_ctas") == 132      # one slim CTA per SM


# Bad-argument calls of the LayerNorm, bias-GeLU and dropout entries, each with the status and message it must return.  They run in a child
# process that sees no device (CUDA_VISIBLE_DEVICES=""), so a call that slips past validation fails with BG_ECUDA at its launch
# instead of launching a kernel on a bad pointer.
_BAD_ROW_CALLS = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M = 0x10000, 0x10002            # a 16-B aligned and a misaligned address; neither is ever dereferenced
EINVAL, EUNSUPPORTED = -1, -7
out = []
def call(want_rc, want_msg, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_last_error().decode(), L.bg_launch_count() - before],
                    want=[want_rc, want_msg, 0]))
FWD, BWD, GELU = "bg_layernorm_fwd", "bg_layernorm_bwd", "bg_bias_gelu"
for i in range(4):                 # x, w, b, y
    p = [A] * 4; p[i] = M
    call(EINVAL, FWD + ": 16-B alignment", FWD, *p, A, A, 4, 768, 1e-5, None)
for i in (0, 1, 2, 5, 6, 7):       # dy, x, w, dx, dw_partial, db_partial (mean and rstd are read as scalars)
    p = [A] * 8; p[i] = M
    call(EINVAL, BWD + ": 16-B alignment", BWD, *p, 4, 768, 7, None)
for rows, cols, rc, why in ((4, 0, EINVAL, "cols 0 must be a positive multiple of 8"),
                            (4, -8, EINVAL, "cols -8 must be a positive multiple of 8"),
                            (4, 12, EINVAL, "cols 12 must be a positive multiple of 8"),
                            (-1, 768, EINVAL, "rows -1 must be >= 0"),
                            (4, 8200, EUNSUPPORTED, "cols 8200 > 8192")):
    call(rc, FWD + ": " + why, FWD, A, A, A, A, A, A, rows, cols, 1e-5, None)
    call(rc, BWD + ": " + why, BWD, A, A, A, A, A, A, A, A, rows, cols, 7, None)
call(EINVAL, BWD + ": n_partial must be >= 1", BWD, A, A, A, A, A, A, A, A, 4, 768, 0, None)
for i in range(4):                 # x, bias, dy, out
    p = [A] * 4; p[i] = M
    call(EINVAL, GELU + ": 16-B alignment", GELU, *p, 4, 768, 1, None)
call(EINVAL, GELU + ": 16-B alignment", GELU, M, None, None, A, 4, 768, 0, None)
for cols in (0, 12):
    call(EINVAL, GELU + ": cols %d must be a positive multiple of 8" % cols, GELU, A, None, None, A, 4, cols, 1, None)
call(EINVAL, GELU + ": rows -1 must be >= 0", GELU, A, None, None, A, -1, 768, 1, None)
DF, DB = "bg_dropout_add_fwd", "bg_dropout_bwd"
DROP = (8, 768, 2, 0, 0, 0.1, 1, 0, 0, None)   # rows, h, b_loc, seq_base, sample_base, p, seed, iteration, site, stream
for i in (0, 4):                   # x, y (bias and residual may be null)
    p = [A, None, 0, None, A]; p[i] = None
    call(EINVAL, DF + ": x and y must be non-null; 16-B alignment", DF, *p, *DROP)
for i in range(2):                 # dy, dx (dbias_partial may be null)
    p = [A, A]; p[i] = None
    call(EINVAL, DB + ": dy and dx must be non-null; 16-B alignment", DB, *p, None, 1, *DROP)
print(json.dumps(out))
"""


def test_row_ops_reject_bad_arguments(bg):
    """LayerNorm and bias-GeLU validate their arguments as RMSNorm does, before any launch: BG_EINVAL for a negative row count,
    a width that is not a positive multiple of 8, a pointer that is not 16-B aligned (their 16-B vector accesses would fault)
    and no backward partials; BG_EUNSUPPORTED for a row wider than the register-resident 8192 columns.  The dropout entries reject
    a null x, y, dy or dx with BG_EINVAL, as the drop-path entries do."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_ROW_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(calls) == 4 + 6 + 10 + 1 + 5 + 2 + 1 + 2 + 2
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


# Bad-argument calls of the plain GEMM entries, and the context-free bad arguments of the fused GEMM + collective entries (called
# with a null context: every check that needs no context comes first).  Same child process as above, with no device.
_BAD_GEMM_CALLS = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M = 0x10000, 0x10008            # a 16-B aligned and an 8-B aligned address; neither is ever dereferenced
EINVAL = -1
out = []
def call(want_msg, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_last_error().decode(), L.bg_launch_count() - before],
                    want=[EINVAL, want_msg, 0]))
GEMM, ADD = "bg_gemm_bf16", "bg_gemm_bf16_add"
BAD_DIMS = ((0, 64, 64), (64, 0, 64), (64, 64, 0), (-8, 64, 64), (64, -8, 64), (64, 64, -8), (12, 64, 64), (64, 12, 64),
            (64, 64, 12))
for layout in (-1, 3):
    call(GEMM + ": layout %d" % layout, GEMM, A, A, A, 64, 64, 64, layout, 0, None)
    call(GEMM + ": layout %d" % layout, ADD, A, A, A, A, 64, 64, 64, layout, None)
for m, n, k in BAD_DIMS:
    why = GEMM + ": m,n,k (%d,%d,%d) must be positive multiples of 8" % (m, n, k)
    call(why, GEMM, A, A, A, m, n, k, 0, 1, None)
    call(why, ADD, A, A, A, A, m, n, k, 1, None)
for i in range(3):                 # a, b, c
    p = [A] * 3; p[i] = M
    call(GEMM + ": pointers must be 16-B aligned", GEMM, *p, 64, 64, 64, 2, 0, None)
    call(GEMM + ": pointers must be 16-B aligned", ADD, *p, A, 64, 64, 64, 2, None)
for addend in (None, M):
    call(ADD + ": addend must be a 16-B aligned [M][N] bf16 tensor", ADD, A, A, A, addend, 64, 64, 64, 0, None)
RS, AR, AG = "bg_gemm_reduce_scatter", "bg_gemm_all_reduce", "bg_all_gather_gemm"
def rs(layout=0, m=256, n=64, k=64, a=A, b=A, o=A):
    return (None, 0, 2, a, b, m, n, k, layout, None, None, o, None)
def ar(layout=0, m=256, n=64, k=64, a=A, b=A):
    return (None, 0, 2, a, b, m, n, k, layout, None, None, None, None)
def ag(layout=0, m=256, n=64, k=64, a=A, b=A, c=A):
    return (None, 0, 4, a, None, None, b, c, m, n, k, layout, None, None)
for name, make, layouts, ptrs in ((RS, rs, (-1, 3), ("a", "b", "o")), (AR, ar, (-1, 3), ("a", "b")), (AG, ag, (-1, 2), ("a", "b", "c"))):
    names = {RS: "a, b and out", AR: "a and b", AG: "a_local, b and c"}[name]
    for layout in layouts:
        call(name + ": layout %d" % layout, name, *make(layout=layout))
    for m, n, k in BAD_DIMS:
        call(name + ": m,n,k (%d,%d,%d) must be positive multiples of 8" % (m, n, k), name, *make(m=m, n=n, k=k))
    for ptr in ptrs:
        call(name + ": %s must be 16-B aligned" % names, name, *make(**{ptr: M}))
    call("null ctx", name, *make())             # every context-free argument valid: the context is checked next
print(json.dumps(out))
"""


def test_gemm_entries_reject_bad_arguments(bg):
    """The plain GEMM entries, and the fused GEMM + reduce-scatter / all-reduce / all-gather entries, reject a bad layout, a
    dimension that is not a positive multiple of 8 and an operand that is not 16-B aligned (TMA bases and strides; the tile
    reducer's 16-B stores into `out`) with BG_EINVAL before any launch.  The fused entries make these checks before they look
    at the context, so a call that fails them can never have launched an entry barrier or a push that its peers then wait on."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_GEMM_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(calls) == 2 * (2 + 9 + 3) + 2 + (2 + 9 + 3 + 1) + (2 + 9 + 2 + 1) + (2 + 9 + 3 + 1)
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


# Bad-argument calls of the plain collective entries, with a null context: each must fail on its own context-free check, which comes
# before the context is looked at.  The last call of each entry has every such argument valid and fails on the null context.  Same
# child process as above, with no device.
_BAD_COLL_CALLS = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M = 0x10000, 0x10008            # a 16-B aligned and an 8-B aligned address; neither is ever dereferenced
EINVAL, EUNSUPPORTED = -1, -7
BF, F32 = 0, 1
out = []
def call(want_rc, want_msg, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_last_error().decode(), L.bg_launch_count() - before],
                    want=[want_rc, want_msg, 0]))
AG, RS, AR, PS, A2A = "bg_all_gather_cast", "bg_reduce_scatter_acc", "bg_all_reduce", "bg_pair_sum_inplace", "bg_all_to_all_rows"
def ag(src=A, sd=F32, dd=BF, n=64):
    return (None, 0, 0, src, sd, None, dd, n, None)
for sd, dd in ((BF, F32), (2, BF), (F32, 2), (-1, -1)):
    call(EUNSUPPORTED, "all_gather_cast %d->%d" % (sd, dd), AG, *ag(sd=sd, dd=dd))
    call(EUNSUPPORTED, "all_gather_cast %d->%d" % (sd, dd), AG, *ag(sd=sd, dd=dd, n=0))    # checked before the empty return
for sd, dd, n, per in ((F32, BF, 4, 8), (BF, BF, 12, 8), (F32, F32, 6, 4)):
    call(EINVAL, "shard_elems %d must be a multiple of %d (pad the flat buffer)" % (n, per), AG, *ag(sd=sd, dd=dd, n=n))
call(EINVAL, "src not 16-B aligned", AG, *ag(src=M))
call(EINVAL, "null ctx", AG, *ag())
def rs(sd=BF, dst=A, dd=F32, n=64, acc=0):
    return (None, 0, 1, None, sd, dst, dd, n, 0.5, 0.25, acc, None)
for dd in (2, -1):
    call(EUNSUPPORTED, "reduce_scatter dst dtype %d" % dd, RS, *rs(dd=dd))
call(EUNSUPPORTED, "reduce_scatter 1->0", RS, *rs(sd=F32, dd=BF))
for sd in (2, -1):
    call(EUNSUPPORTED, "reduce_scatter src dtype %d" % sd, RS, *rs(sd=sd))
for sd, dd, n, per in ((BF, F32, 4, 8), (BF, BF, 12, 8), (F32, F32, 6, 4)):
    call(EINVAL, "shard_elems %d must be a multiple of %d" % (n, per), RS, *rs(sd=sd, dd=dd, n=n))
for dd in (F32, BF):
    call(EINVAL, "dst not 16-B aligned", RS, *rs(dd=dd, dst=M, acc=1))
call(EINVAL, "null ctx", RS, *rs())
def ar(dst=A, n=64, dt=BF, op=0):
    return (None, 0, 2, None, dst, n, dt, op, 1.0 / 3.0, None)
for dt in (2, -1):
    call(EUNSUPPORTED, "all_reduce dtype %d" % dt, AR, *ar(dt=dt))
for op in (2, -1):
    call(EUNSUPPORTED, "all_reduce op %d" % op, AR, *ar(op=op))
for dt, n, per in ((BF, 4, 8), (F32, 6, 4)):
    call(EINVAL, "all_reduce elems %d must be a multiple of %d (pad)" % (n, per), AR, *ar(dt=dt, n=n))
call(EINVAL, "dst not 16-B aligned", AR, *ar(dst=M))
call(EINVAL, "null ctx", AR, *ar())
def ps(n=64, dt=BF):
    return (None, 0, 1, None, n, dt, 0.5, None)
call(EUNSUPPORTED, "bg_pair_sum_inplace dtype 2", PS, *ps(dt=2))
for dt, n, per in ((BF, 12, 8), (F32, 6, 4)):
    call(EINVAL, "bg_pair_sum_inplace: elems %d is not a whole number of 16-B vectors (%d elements)" % (n, per), PS, *ps(n=n, dt=dt))
call(EINVAL, "null ctx", PS, *ps())
GOOD = dict(batch=2, rows=4, row_elems=64, src_bs=512, src_rs=128, src_me_off=64, dst_bs=512, dst_rs=64, dst_peer_off=256)
def a2a(dt=BF, count=None, **kw):
    ds = (_bg.bg_a2a_desc * 2)()
    for d in ds:
        d.dst = A
        for k, v in dict(GOOD, **kw).items():
            setattr(d, k, v)
    return (None, 0, 2, ds, 2 if count is None else count, dt, None)
call(EINVAL, "1..4 tensors per all_to_all launch", A2A, None, 0, 2, None, 1, BF, None)
for count in (0, 5):
    call(EINVAL, "1..4 tensors per all_to_all launch", A2A, *a2a(count=count))
for dt in (2, -1):
    call(EUNSUPPORTED, "all_to_all dtype %d" % dt, A2A, *a2a(dt=dt))
for k in GOOD:
    call(EINVAL, "all_to_all: negative extent or stride", A2A, *a2a(**{k: -GOOD[k]}))
for k in GOOD:
    if k not in ("batch", "rows"):
        call(EINVAL, "all_to_all: strides/row length must be multiples of 8 elements", A2A, *a2a(**{k: GOOD[k] + 4}))
call(EINVAL, "all_to_all: strides/row length must be multiples of 4 elements", A2A, *a2a(dt=F32, row_elems=66))
call(EINVAL, "all_to_all dst not 16-B aligned", A2A, *a2a(dst=M))
for b, r, e in ((1 << 16, 1 << 16, 8), (1, 1 << 20, 1 << 15), (1 << 32, 1, 8), (1 << 40, 1 << 40, 8)):
    call(EINVAL, "all_to_all: more than 2^32 16-B vectors per peer", A2A, *a2a(batch=b, rows=r, row_elems=e))
call(EINVAL, "null ctx", A2A, *a2a(batch=0))      # an empty tensor is valid
call(EINVAL, "null ctx", A2A, *a2a(dt=F32))
call(EINVAL, "null ctx", A2A, *a2a())
print(json.dumps(out))
"""


def test_collectives_reject_bad_arguments(bg):
    """The all-gather, reduce-scatter, all-reduce, pair-sum and all-to-all entries reject an unsupported dtype or dtype pair
    (BG_EUNSUPPORTED), and an element count that is not a whole number of 16-B vectors, a misaligned local pointer, a negative
    all-to-all extent or stride and an all-to-all of more than 2^32 vectors per peer (BG_EINVAL), with zero launches and before they
    look at the context: a call that fails them can never have left its peers waiting."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_COLL_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    assert len(calls) == (8 + 3 + 1 + 1) + (2 + 1 + 2 + 3 + 2 + 1) + (2 + 2 + 2 + 1 + 1) + (1 + 2 + 1) + \
        (1 + 2 + 2 + 9 + 7 + 1 + 1 + 4 + 3)
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


# Bad-argument calls of the optimizer entries (the AdamW reduce-scatter, its clipped form, the local clipped step and the norm
# pass), with a null context.  Every hyperparameter is an exact fp32 value, so the message formats it as Python does.  Same child
# process as above, with no device.
_BAD_OPT_CALLS = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from hetu_galvatron_b200 import _bg
L = _bg.lib()
A, M = 0x10000, 0x10008            # a 16-B aligned and an 8-B aligned address; neither is ever dereferenced
EINVAL = -1
BF, F32 = 0, 1
INF, NAN = float("inf"), float("nan")
out = []
def call(want_msg, name, *args):
    before = L.bg_launch_count()
    rc = getattr(L, name)(*args)
    out.append(dict(call="%s%r" % (name, args), got=[rc, L.bg_last_error().decode(), L.bg_launch_count() - before],
                    want=[EINVAL, want_msg, 0]))
RSA, RSC, LOC, SSQ = "bg_reduce_scatter_adamw", "bg_reduce_scatter_adamw_clipped", "bg_adamw_clipped", "bg_reduce_scatter_sumsq"
HYPER = dict(lr=1e-4, b1=0.5, b2=0.75, eps=1e-8, wd=0.0625, step=1)
def rsa(p=A, m=A, v=A, **kw):
    h = dict(HYPER, **kw)
    return (None, 0, 1, None, BF, p, m, v, 64, 0.5, 0.25, h["lr"], h["b1"], h["b2"], h["eps"], h["wd"], h["step"], None)
def rsc(p=A, m=A, v=A, **kw):
    return rsa(p, m, v, **kw)[:-1] + (A, None)
def loc(p=A, m=A, v=A, g=A, n=64, **kw):
    h = dict(HYPER, **kw)
    return (p, m, v, g, n, h["lr"], h["b1"], h["b2"], h["eps"], h["wd"], h["step"], A, None)
STATE = "adamw: param, exp_avg and exp_avg_sq must be non-null"
BAD = [(dict(lr=x), "adamw: lr %g must be finite and >= 0" % x) for x in (-1.0, INF, -INF, NAN)] + \
      [(dict(eps=x), "adamw: eps %g must be finite and >= 0" % x) for x in (-0.5, INF, NAN)] + \
      [(dict(wd=x), "adamw: weight_decay %g must be finite and >= 0" % x) for x in (-0.5, INF, NAN)] + \
      [(dict(b1=x), "adamw: beta1 %g outside [0, 1)" % x) for x in (1.0, -0.5, 2.0, INF, NAN)] + \
      [(dict(b2=x), "adamw: beta2 %g outside [0, 1)" % x) for x in (1.0, -0.5, 2.0, INF, NAN)] + \
      [(dict(b1=0.99999999), "adamw: beta1 1 outside [0, 1)"),        # rounds to 1 in fp32
       (dict(step=0), "adam step must be >= 1"), (dict(step=-(1 << 40)), "adam step must be >= 1")]
for make in (rsa, rsc, loc):
    name = {rsa: RSA, rsc: RSC, loc: LOC}[make]
    for i in range(3):             # param, exp_avg, exp_avg_sq
        p = [A] * 3; p[i] = None
        call(STATE, name, *make(*p))
        p = [A] * 3; p[i] = M
        call("optimizer state not 16-B aligned", name, *make(*p))
    for kw, msg in BAD:
        call(msg, name, *make(**kw))
    if make is loc:
        call("adamw: 6 elements / gradient alignment (need multiples of 4, 16 B)", name, *make(n=6))
        call("adamw: 64 elements / gradient alignment (need multiples of 4, 16 B)", name, *make(g=M))
        call("adamw: null grad", name, *make(g=None))
    else:                          # every hyperparameter edge that is valid, in turn: the context is checked next
        for kw in (dict(lr=0.0, wd=0.0, b1=0.0, b2=0.0, eps=0.0), dict(b1=0.99999994, b2=0.99999994), dict(step=(1 << 31) + 5)):
            call("null ctx", name, *make(**kw))
def ssq(skip=(), dst=A, n=64, parts=A, n_parts=64):
    flat = [x for r in skip for x in r]
    arr = (ctypes.c_size_t * max(1, len(flat)))(*flat)
    return (None, 0, 1, None, BF, dst, n, 0.5, 0.25, parts, n_parts, arr, len(skip), None)
call("sum-of-squares partials missing", SSQ, *ssq(parts=None))
call("sum-of-squares partials missing", SSQ, *ssq(n_parts=0))
call("-1 skip ranges (at most 16)", SSQ, *ssq(skip=[(0, 8)] * 17)[:-2] + (-1, None))
call("17 skip ranges (at most 16)", SSQ, *ssq(skip=[(0, 8)] * 17))
for lo, hi in ((4, 8), (0, 12), (16, 8)):
    call("skip range [%d, %d) is not 8-element aligned" % (lo, hi), SSQ, *ssq(skip=[(lo, hi)]))
for lo, hi in ((0, 72), (64, 72), (72, 80)):
    call("skip range [%d, %d) ends past the shard of 64 elements" % (lo, hi), SSQ, *ssq(skip=[(0, 8), (lo, hi)]))
call("dst not 16-B aligned", SSQ, *ssq(dst=M))
for skip in ([], [(0, 0)], [(0, 64)], [(56, 64), (0, 8), (0, 64)], [(8, 16)] * 16):
    call("null ctx", SSQ, *ssq(skip=skip))
call("null ctx", SSQ, *ssq(dst=None))
print(json.dumps(out))
"""


def test_optimizer_rejects_bad_arguments(bg):
    """The AdamW entries (the reduce-scatter, its clipped form and the local clipped step) reject, with BG_EINVAL and zero launches
    and before they look at the context: a null or misaligned optimizer state, step < 1, lr, eps or weight_decay negative or not
    finite, and beta1 or beta2 outside [0, 1) or NaN -- as fp32 values, so a beta that rounds to 1 is refused (beta1 = 1 would
    turn every parameter into inf or NaN); the local step also a null gradient.  The norm pass rejects a skip range that ends
    past the shard, as well as missing partials, too many ranges and misaligned or inverted ranges.  Valid edges (lr, wd, eps
    and the betas 0; the largest fp32 beta below 1; a step past 2^31; empty, whole-shard, overlapping and BG_MAX_SKIP ranges)
    pass every check and fail on the null context."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, "-c", _BAD_OPT_CALLS, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stderr
    calls = json.loads(res.stdout.strip().splitlines()[-1])
    n_bad = 4 + 3 + 3 + 5 + 5 + 3
    assert len(calls) == 2 * (6 + n_bad + 3) + (6 + n_bad + 3) + (2 + 2 + 3 + 3 + 1 + 5 + 1)
    bad = [c for c in calls if c["got"] != c["want"]]
    assert not bad, bad


def test_c_mirror_of_group_builder_matches_goldens(bg):
    L = bg.lib()
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "comm_groups.json")))
    kinds = ["tp_groups", "sp_groups", "cp_groups", "dp_groups", "seq_data_groups"]
    for case in gold["cases"]:
        hpw, W = case["hp_configs_whole"], case["world"]
        n = len(hpw["tp_sizes_whole"])
        arr = lambda v: (ctypes.c_int * n)(*v)  # noqa: E731
        for rank in range(W):
            cnt = (ctypes.c_int * (5 * n))()
            rk = (ctypes.c_int * (5 * n * 64))()
            pc, pr = ctypes.c_int(), (ctypes.c_int * 64)()
            bg.check(L.bg_build_groups(rank, W, hpw["pp_deg"], n, arr(hpw["tp_sizes_whole"]), arr(hpw["sp_sizes_whole"]),
                                       arr(hpw["cp_sizes_whole"]), cnt, rk, ctypes.byref(pc), pr))
            want = case["groups_per_rank"][rank]
            assert [pr[j] for j in range(pc.value)] == want["pp_group"]
            for kind, key in enumerate(kinds):
                got = [[rk[(kind * n + i) * 64 + j] for j in range(cnt[kind * n + i])] for i in range(n)]
                assert got == want[key], (case["name"], rank, key)


def test_product_never_imports_the_oracle():
    """oracle/ is test infrastructure: only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline / reference arm may use it.
    No module of the package (nor the C sources) may name it in an import; the CUDA backend must be what get_backend() builds."""
    import ast
    pkg = os.path.join(ROOT, "hetu-galvatron_b200")
    offenders = []
    for dp, _, files in os.walk(pkg):
        for f in files:
            path = os.path.join(dp, f)
            if f.endswith(".py"):
                tree = ast.parse(open(path).read())
                for node in ast.walk(tree):
                    names = []
                    if isinstance(node, ast.Import):
                        names = [a.name for a in node.names]
                    elif isinstance(node, ast.ImportFrom) and node.module:
                        names = [node.module]
                    offenders += [(os.path.relpath(path, ROOT), n) for n in names if n == "oracle" or n.startswith("oracle.")]
            elif f.endswith((".cu", ".cuh", ".h")):
                if "oracle/" in open(path, errors="replace").read():
                    offenders.append((os.path.relpath(path, ROOT), "oracle/ path"))
    assert not offenders, offenders
    src = open(os.path.join(pkg, "core", "runtime", "backend.py")).read()
    assert "class CudaBackend" in src and "OracleBackend" not in src.replace("``oracle/gloo_backend.py``", "")
