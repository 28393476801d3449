"""The C-ABI shared library (rl_markets_b200/librlm.so): loads, exports every symbol include/rlm.h
declares, structure layouts agree with the ctypes mirror, and -- without a GPU -- fails loudly
instead of falling back to a CPU path.  No compute calls here."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import pytest

from rl_markets_b200 import abi, config, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "rlm.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rlm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = lib.load()
    names = _declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(L, n), "librlm.so does not export %s" % n
    assert set(names) == set(lib.EXPORTS)
    header = open(os.path.join(ROOT, "include", "rlm.h")).read()
    assert L.rlm_abi_version() == int(re.search(r"#define RLM_ABI_VERSION (\d+)", header).group(1))


def test_struct_layouts_match_the_c_headers():
    prog = r'''
#include <stdio.h>
#include <stddef.h>
#include "rlm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu %zu %zu %zu %zu\n", sizeof(rlm_config), sizeof(rlm_step_record), sizeof(rlm_tick_msg),
         sizeof(rlm_flow_params), sizeof(rlm_counters), sizeof(rlm_env_stats), offsetof(rlm_config, flow),
         offsetof(rlm_step_record, trace_hash), offsetof(rlm_config, band_px), offsetof(rlm_config, random_seed),
         offsetof(rlm_step_record, delta));
  return 0;
}'''
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "s.c")
        open(src, "w").write(prog)
        exe = os.path.join(d, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    exp = [C.sizeof(abi.Config), C.sizeof(abi.StepRecord), C.sizeof(abi.TickMsg), C.sizeof(abi.FlowParams),
           C.sizeof(abi.Counters), C.sizeof(abi.EnvStats), abi.Config.flow.offset, abi.StepRecord.trace_hash.offset,
           abi.Config.band_px.offset, abi.Config.random_seed.offset, abi.StepRecord.delta.offset]
    assert got == exp


def test_config_default_is_example_yaml():
    L = lib.load()
    c = abi.Config()
    assert L.rlm_config_default(C.byref(c)) == 0
    assert (c.memory_size, c.n_tilings, c.n_actions) == (20000000, 32, 9)
    assert c.algorithm == abi.ALGO["double_q_learn"] and c.policy_type == abi.POLICY["epsilon_greedy"]
    assert [c.state_vars[i] for i in range(c.n_state_vars)] == [abi.VAR[v] for v in
                                                                ["pos", "a_dist", "b_dist", "mpm", "spd", "vol", "imb", "svl"]]
    y = config.example_dict(**{"learning.memory_size": 20000000, "learning.algorithm": "double_q_learn"})
    c2 = config.from_dict(y, flow_seed=1)
    for f in ("memory_size", "n_tilings", "n_actions", "algorithm", "gamma", "lambda_", "alpha_start", "eps_init", "eps_T",
              "spread_lookback", "reward_measure", "damping_factor", "lb_mpm", "lb_vlt", "lb_svl", "pos_lb", "pos_ub",
              "order_size", "target_price_type", "tp_lookback", "n_bands", "open_ms", "close_ms", "random_seed"):
        assert getattr(c, f) == getattr(c2, f), f
    assert list(c.band_px)[:10] == list(c2.band_px)[:10] and list(c.band_ts)[:10] == list(c2.band_ts)[:10]
    assert bytes(c.flow) == bytes(c2.flow)


def test_config_quirks_of_the_reference():
    # inverted target-price selector (base.cpp:101-112) is applied in the library; yaml strings are kept as written
    y = config.example_dict(**{"market.target_price.type": "microprice"})
    assert config.from_dict(y).target_price_type == abi.TP_YAML["microprice"]
    y = config.example_dict(**{"market.target_price.type": "something_else"})
    assert config.from_dict(y).target_price_type == abi.TP_YAML["microprice"]  # any other string -> tp::MidPrice
    with pytest.raises(ValueError):
        config.from_dict(config.example_dict(**{"learning.algorithm": "nope"}))
    with pytest.raises(ValueError):
        config.from_dict(config.example_dict(**{"state.variables": ["pos", "bogus", "spd", "vol"]}))
    with pytest.raises(ValueError):
        config.from_dict(config.example_dict(), ticker="AAL.XX")
    # market.latency (base.cpp:77-99, latency.cpp:9-14): the three types are accepted (the sample is dead upstream:
    # intraday.cpp:178 writes ref_time, nothing reads it), the constructor checks are mirrored
    for lat in ({"market.latency.type": "normal", "market.latency.sigma": 1.0, "market.latency.mu": 2.0},
                {"market.latency.type": "lognormal", "market.latency.beta": 0.5}, {"market.latency.floor": 3.0}):
        config.from_dict(config.example_dict(**lat))
    for bad in ({"market.latency.type": "uniform"}, {"market.latency.floor": -1.0}, {"market.latency.type": "lognormal"}):
        with pytest.raises(ValueError):
            config.from_dict(config.example_dict(**bad))


def test_no_cpu_fallback():
    """Without a CUDA device rlm_create must fail with RLM_ERR_NO_DEVICE (never run on the CPU)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    cfg = config.from_dict(config.example_dict(**{"learning.memory_size": 4096}), n_envs=4)
    with pytest.raises(lib.RlmError) as ei:
        lib.BatchedMarket(cfg)
    assert ei.value.code == abi.RLM_ERR_NO_DEVICE
    px = (C.c_double * 1)(2750.0)
    out = (C.c_int32 * 1)()
    assert lib.load().rlm_test_to_ticks(C.byref(cfg), px, 1, out) == abi.RLM_ERR_NO_DEVICE


def test_set_flow_binding_and_argument_checks():
    """rlm_set_flow (LoadData of another synthetic day on the same env objects) is bound with the header's types and
    refuses a missing handle or flow before it touches a device; the ABI version is unchanged by the addition."""
    L = lib.load()
    assert L.rlm_set_flow.argtypes == [C.c_void_p, C.POINTER(abi.FlowParams)]
    assert L.rlm_abi_version() == 4
    flow = config.from_dict(config.example_dict(), flow_seed=5).flow
    assert L.rlm_set_flow(None, C.byref(flow)) == abi.RLM_ERR_INVALID_ARGUMENT
    assert "rlm_set_flow" in L.rlm_last_error().decode()
    assert L.rlm_set_flow(None, None) == abi.RLM_ERR_INVALID_ARGUMENT
    assert hasattr(lib.BatchedMarket, "set_flow")


def test_product_does_not_import_the_oracle():
    for root, _dirs, files in os.walk(os.path.join(ROOT, "rl_markets_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(root, f), errors="ignore").read()
                assert "lob_oracle" not in txt and "oracle_lib" not in txt and "liblob" not in txt, f
