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
