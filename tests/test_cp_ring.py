"""Ring context parallelism (``cp_comm="ring"``) on the CPU: every context-parallel strategy of tests/test_host_runtime.py, run with the
ring schedule over gloo (tests/_cp_ring_ref.py supplies the transport and the block attention), reproduces the single-process oracle
under the same criteria; the ring keeps only the local s/c rows of K/V for backward where the all-gather path keeps the whole
sequence; an unknown ``cp_comm`` is refused when the model is built."""
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_host_runtime import WORLD2, WORLD4, WORLD8  # noqa: E402

_PORT = [30900]

CP_STRATEGIES = {2: ["cp2", "cp_mixed_vcp1_layers_cp2"],
                 4: ["cp2_dp2_zero3_ckpt", "cp_mixed_tp2_to_cp2", "cp_mixed_cp4_to_tp2cp2", "cp2_pp2_1f1b", "cp2_tp2_megatron_sp"],
                 8: ["tp2_cp2_dp2_zero3"]}
_CORPUS = {2: WORLD2, 4: WORLD4, 8: WORLD8}
CASES = [(w, name) for w, names in CP_STRATEGIES.items() for name in names]


def launch(world, config, timeout=900, backend="oracle"):
    from _launch import launch_ranks
    _PORT[0] += 1
    extra_env = config.pop("_env", {})
    return launch_ranks("_cp_ring_worker", world, config, _PORT[0] + os.getpid() % 500, timeout=timeout, backend=backend,
                        extra_env=extra_env)


@pytest.mark.parametrize("world,name", CASES, ids=["%s" % n for _, n in CASES])
def test_ring_strategy_matches_oracle(world, name):
    rep = launch(world, dict(_CORPUS[world][name]))
    assert rep["max_grad_err"] < 3e-2
    assert abs(rep["loss"] - rep["ref_loss"]) <= 5e-3 * abs(rep["ref_loss"])
    assert rep["ring_pushes"] > 0


@pytest.mark.parametrize("c", [2, 4])
def test_ring_saves_only_local_kv(c):
    rep = launch(c, {"_mode": "saved", "seq": 64})
    assert rep["ring"]["max_dim"] <= rep["s_loc"], rep          # nothing kept for backward spans more than s/c rows
    assert rep["allgather"]["max_dim"] >= rep["s_full"], rep    # the gather path keeps whole-sequence K/V


def test_unknown_cp_comm_is_refused():
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import smoke_model as sm
    from hetu_galvatron_b200.core.runtime.arguments import DEFAULTS
    assert DEFAULTS["cp_comm"] == "allgather"
    args = sm.tiny_args(cp_comm="ring_of_fire")
    with pytest.raises(ValueError, match="cp_comm"):
        sm.build(args)
