"""CPU checks of the backend's peer-visible buffer bookkeeping and of its choice between a fused GEMM + collective and the GEMM
followed by the stand-alone collective:
  * ``fusion_allowed`` selects exactly what the rule below selects, on a grid through every boundary of that rule;
  * ``StagingLayout`` places the regions and counter blocks of a staging buffer where the fused kernels are told they are;
  * the reservations make the same ``sym_alloc`` calls (group, size, order) for growing, repeated and shrinking requests -- the
    arena layout, and the multicast regions derived from it, depend on that sequence -- and refuse to grow after ``exchange()``."""
import itertools

import pytest
import torch

from hetu_galvatron_b200 import _bg
from hetu_galvatron_b200.core.runtime import backend
from hetu_galvatron_b200.core.runtime.comm_groups import CommGroup

F = 1 << 16     # counter bytes at the end of every staging buffer


def _rule(kind, m, n, k, p, data_bytes, env):
    """The selection rule, written out: ``env`` is the kind's HGB_FUSE_* value (None = unset)."""
    on, force = env != "0", env == "force"
    if kind == "ag_gemm":
        return (on and p >= 2 and m % (p * 128) == 0 and k % 8 == 0 and data_bytes is not None and data_bytes >= 2 * m * k
                and 4 * (m // 128) <= F // 2)
    min_k, counter_bytes = (3072, F // 2) if kind == "gemm_rs" else (2048, F // 4)
    if not on or p < 2 or m % (p * 128) or n % 8:
        return False
    if k is not None and k < min_k and not force:
        return False
    tiles = (m // p // 128) * ((n + 127) // 128)
    return data_bytes is not None and data_bytes >= 2 * m * n and 4 * tiles <= counter_bytes


def test_fusion_rule_grid():
    checked = selected = 0
    for p in (1, 2, 4, 8):
        # whole 128-row tiles per rank and 8 rows off them; 8192 // p tiles per rank reach the gather counter block's edge,
        # (64 tiles) x (64 / 128 column tiles) the all-reduce / reduce-scatter edges
        ms = sorted({p * 128 * a + d for a in (1, 3, 64, 8192 // p, 8192 // p + 1) for d in (-8, 0, 8)})
        ns = (128, 136, 1004, 8192, 8200, 16384, 16392)
        for kind, m, n, k, env in itertools.product(("gemm_rs", "gemm_ar", "ag_gemm"), ms, ns,
                                                    (None, 2040, 2048, 2056, 3064, 3072, 3080, 4100), (None, "0", "force")):
            if kind == "ag_gemm" and k is None:
                continue
            need = 2 * m * (k if kind == "ag_gemm" else n)
            for data_bytes in (None, need - 256, need, need + 256):
                want = _rule(kind, m, n, k, p, data_bytes, env)
                got = backend.fusion_allowed(kind, m, n, k, p, data_bytes, env != "0", env == "force")
                assert got == want, (kind, m, n, k, p, data_bytes, env)
                checked += 1
                selected += want
    assert selected > 1000 and checked - selected > 1000


@pytest.mark.parametrize("n", [256, 4096, 3 << 20])
def test_staging_layout(n):
    lay = backend.StagingLayout(n)
    assert (lay.n, lay.partials, lay.result, lay.scatter_counters, lay.gather_counters, lay.total) == (
        n, n, 2 * n, 3 * n, 3 * n + F // 2, 3 * n + F)


class _FakeComm:
    """Records sym_alloc calls; exchange() gives every buffer its offsets."""

    def __init__(self):
        self.calls, self.bufs = [], []

    def sym_alloc(self, group, nbytes):
        self.calls.append((tuple(group.ranks), nbytes))
        buf = type("Buf", (), {})()
        buf.offsets, buf.u8 = None, torch.ones(nbytes, dtype=torch.uint8)
        self.bufs.append(buf)
        return buf

    def exchange(self):
        for b in self.bufs:
            b.offsets = [0]


def _backend(comm):
    be = backend.CudaBackend.__new__(backend.CudaBackend)     # the reservations need no device
    be.bg, be.comm, be._bufs, be._cp_rings = _bg, comm, backend._SymBuffers(comm), {}
    return be


def test_reservations_allocate_like_before():
    comm = _FakeComm()
    be = _backend(comm)
    g, h, one = CommGroup([0, 1]), CommGroup([0, 2]), CommGroup([3])
    assert be.reserve_staging(one, 1 << 20) is None and be.reserve_staging(None, 1 << 20) is None
    s1 = be.reserve_staging(g, 1000)                 # rounded up to 1024 data bytes
    assert int(s1.u8[3 * 1024:].sum()) == 0 and int(s1.u8[:3 * 1024].min()) == 1      # only the counters are zeroed
    assert be.reserve_staging(g, 1024) is s1         # repeat: no call
    s2 = be.reserve_staging(g, 5000)                 # grow: a new buffer; the first stays allocated
    assert be.reserve_staging(g, 4000) is s2         # shrink: no call
    be.reserve_staging(h, 256)
    be.reserve_cp_ring(g, 10)                        # rounded up to 16 elements, 24 B each
    be.reserve_cp_ring(g, 16)
    be.reserve_cp_ring(g, 17)
    be.reserve_cp_ring(one, 1 << 20)
    be.reserve_checkpoint_gather(g, 1000)            # sym_alloc rounds to 1024: 1020 fits, 1030 does not
    be.reserve_checkpoint_gather(g, 1020)
    be.reserve_checkpoint_gather(g, 1030)
    be.reserve_checkpoint_gather(None, 1 << 20)
    assert comm.calls == [((0, 1), 3 * 1024 + F), ((0, 1), 3 * 5120 + F), ((0, 2), 3 * 256 + F), ((0, 1), 16 * 24),
                          ((0, 1), 24 * 24), ((0, 1), 1000), ((0, 1), 1030)]
    assert be.staging(g, 5120) is s2
    with pytest.raises(_bg.BgError):
        be.staging(g, 5121)
    with pytest.raises(_bg.BgError):
        be.staging(CommGroup([1, 2]), 16)
    comm.exchange()
    n_calls = len(comm.calls)
    assert be.reserve_staging(g, 5120) is s2         # after exchange(): repeat and shrink still fine ...
    be.reserve_cp_ring(g, 8)
    be.reserve_checkpoint_gather(g, 1280)
    for grow in (lambda: be.reserve_staging(g, 5121), lambda: be.reserve_cp_ring(g, 25),
                 lambda: be.reserve_checkpoint_gather(g, 1281)):
        with pytest.raises(_bg.BgError):             # ... growing raises
            grow()
    assert len(comm.calls) == n_calls


def test_fuses_reads_the_reservation_and_force(monkeypatch):
    monkeypatch.delenv("HGB_FUSE_GEMM_RS", raising=False)
    be = _backend(_FakeComm())
    be.fuse = dict.fromkeys(backend.FUSE_ENV, True)
    g = CommGroup([0, 1])
    assert not be.fuses("ag_gemm", 256, 64, 64, g)              # no staging reserved
    be.reserve_staging(g, 2 * 256 * 64)
    assert be.fuses("ag_gemm", 256, 64, 64, g) and not be.fuses("ag_gemm", 256, 64, 72, g)
    assert not be.fuses("gemm_rs", 256, 64, 64, g)              # K below the threshold ...
    monkeypatch.setenv("HGB_FUSE_GEMM_RS", "force")             # ... unless forced, read at every call
    assert be.fuses("gemm_rs", 256, 64, 64, g) and not be.fuses("gemm_rs", 256, 64, 64, None)
