"""The learner kernels across the configurations rlm_create accepts, against the CPU oracle, bitwise.

The reference itself pins the oracle at every configuration point used here (tools/make_golden.py CONFIG_CASES,
test_oracle_golden.py); this module holds every learner / engine that can take a point to the oracle: 1..9 actions, 4..13
state variables, trace lists from none (lambda = 0) to ~13 000 entries, tables of 1 weight to 2^27 + 1, and the trace
capacity's error path.
"""
import ctypes as C
import os

import numpy as np
import pytest

import golden_util as G
from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu

N_ENVS, N_TICKS = 5, 1500
CONFIG_NAMES = ["act1_q", "act2_random", "act5_double_q", "act7_r_learn", "vars4_sarsa", "vars11_q", "long_traces_sarsa",
                "long_traces_q", "lambda0_q", "m6000_staged", "m8190_staged_sarsa", "m8194_gather", "m2_staged", "m1_gather",
                "m3_gather", "m97_gather"]
# (id, environment, run calls): short calls stay tick-synchronous, a long one is round-paced for Q-learning / SARSA /
# Double-Q (rlm_run_ticks); every switch below is read by rlm_create
VARIANTS = [
    ("default", {}, [100] * 15),
    ("staged0", {"RLM_STAGED": "0"}, [N_TICKS]),
    ("agent3", {"RLM_AGENT_VARIANT": "3"}, [N_TICKS]),
    ("agent1", {"RLM_AGENT_VARIANT": "1"}, [N_TICKS]),
    ("engineF", {"RLM_ENGINE": "F"}, [N_TICKS]),
    ("rounds1", {"RLM_ROUNDS": "1"}, [N_TICKS]),
]


def _case(name):
    return [c for c in G.manifest() if c["name"] == name][0]


def _staged(case):
    """rlm_create stages the whole table in shared memory for single-table agents with an even M <= 8192."""
    return case["algo"] not in ("double_q_learn", "double_r_learn") and case["M"] % 2 == 0 and case["M"] <= 8192


def _rerouted(case, variant):
    """Why rlm_create runs the same kernels as another variant for this combination, or None."""
    r_learning = case["algo"].endswith("r_learn")
    if variant == "staged0" and not _staged(case):
        return "no staged learner at this table size or agent"
    if variant == "engineF" and r_learning:
        return "the fused engine leaves R-learning to the tick-synchronous engine"
    return None


def _params():
    out = []
    for name in CONFIG_NAMES:
        case = _case(name)
        for vid, env, calls in VARIANTS:
            why = _rerouted(case, vid)
            if why:
                out.append(pytest.param(name, env, calls, id="%s-%s-rerouted" % (name, vid), marks=pytest.mark.skip(reason=why)))
            else:
                out.append(pytest.param(name, env, calls, id="%s-%s" % (name, vid)))
    return out


_PORT = {}


def _port(oracle, cfg, name, b):
    """Oracle run of env b of a case (shared by the variants of the case)."""
    if (name, b) not in _PORT:
        _PORT[(name, b)] = oracle.run_port(cfg, b, oracle.generate_ticks(cfg, b, N_TICKS))
    return _PORT[(name, b)]


def _compare(recs, port, label):
    assert len(recs) == port["steps"] > 100, (label, len(recs), port["steps"])
    for i, r in enumerate(recs):
        bad = abi.record_fields_equal(r, port["records"][i])
        assert not bad, "%s step %d (cuda, oracle): %r" % (label, i, G.describe_diff(r, port["records"][i], bad))


def _config(case, **kw):
    cfg = config.from_dict(case["yaml"], n_envs=kw.pop("n_envs", N_ENVS), flow_seed=case["flow_seed"])
    cfg.record_envs = cfg.n_envs
    cfg.record_cap = kw.pop("record_cap", 1200)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("name,env_vars,calls", _params())
def test_config_point_matches_oracle(rlm, oracle, monkeypatch, name, env_vars, calls):
    """Every record, the weights and the trace counter of 5 envs x 1500 ticks, bitwise."""
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    case = _case(name)
    cfg = _config(case)
    m = rlm.BatchedMarket(cfg)
    for n in calls:
        m.run_ticks(n)
    m.sync()
    cnt = m.counters()
    sum_traces = 0
    for b in range(N_ENVS):
        port = _port(oracle, cfg, name, b)
        recs, _keep = m.records(b)
        _compare(recs, port, "%s %r env %d" % (name, env_vars, b))
        assert bytes(m.theta(b, 0)) == bytes((C.c_double * cfg.memory_size)(*port["theta"])), (name, env_vars, b)
        sum_traces += port["sum_traces"]
    assert cnt.steps == sum(_port(oracle, cfg, name, b)["steps"] for b in range(N_ENVS))
    assert cnt.sum_traces == sum_traces, (name, env_vars, cnt.sum_traces, sum_traces)
    m.close()


def test_long_traces_flush_the_update_table_within_a_step(oracle):
    """The long-trace cases are what they are meant to be: lists far longer than one 512-entry batch of the one-warp
    learner's update table, so that a single step drains it several times."""
    case = _case("long_traces_sarsa")
    cfg = _config(case)
    port = _port(oracle, cfg, "long_traces_sarsa", 0)
    assert cfg.trace_cap == 0
    assert max(r.n_traces for r in port["records"]) > 4 * 512


# ---- trace capacity

def _run(rlm, cfg, calls=(N_TICKS,)):
    m = rlm.BatchedMarket(cfg)
    for n in calls:
        m.run_ticks(n)
    m.sync()
    out = ([m.records(b)[0] for b in range(cfg.n_envs)], [bytes(m.theta(b)) for b in range(cfg.n_envs)], m.counters().sum_traces)
    m.close()
    return out


@pytest.mark.parametrize("algo,M", [("sarsa", 8192), ("q_learn", 16384)])
def test_explicit_trace_cap_at_or_above_the_derived_one_changes_nothing(rlm, algo, M):
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
    res = []
    for cap in (0, 864, 2000):  # 0: derived, 32 * (life + 1) = 864 at the default gamma * lambda
        cfg = config.from_dict(y, n_envs=3, flow_seed=41)
        cfg.record_envs, cfg.record_cap, cfg.trace_cap = 3, 1000, cap
        res.append(_run(rlm, cfg))
    recs0, th0, st0 = res[0]
    assert st0 > 0
    for recs, th, st in res[1:]:
        assert th == th0 and st == st0
        for b in range(3):
            assert len(recs[b]) == len(recs0[b]) > 100
            for i in range(len(recs[b])):
                assert not abi.record_fields_equal(recs[b][i], recs0[b][i]), (algo, b, i)


@pytest.mark.parametrize("env_vars,M", [({}, 8192), ({}, 16384), ({"RLM_AGENT_VARIANT": "3"}, 16384),
                                        ({"RLM_ENGINE": "F"}, 16384)],
                         ids=["staged", "one_warp", "three_warp", "fused_F"])
def test_too_small_trace_cap_is_an_error(rlm, monkeypatch, env_vars, M):
    """SARSA keeps ~800 traces at the default gamma * lambda: a capacity of 64 must end in RLM_ERR_RUNTIME at rlm_sync,
    never in a run that finishes with truncated traces."""
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": "sarsa"})
    cfg = config.from_dict(y, n_envs=3, flow_seed=43)
    cfg.trace_cap = 64
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(600)
    with pytest.raises(rlm.RlmError) as ei:
        m.sync()
    assert ei.value.code == abi.RLM_ERR_RUNTIME and "trace list overflow" in str(ei.value)
    m.close()


# ---- table sizes at full scale

def _device_theta(m, M, b):
    out = np.empty(M, dtype=np.float64)
    m.L.rlm_read_theta(m.h, b, 0, out.ctypes.data_as(C.POINTER(C.c_double)), M)
    return out


def _full_scale(rlm, oracle, M, n_envs):
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=n_envs, flow_seed=47)
    cfg.record_envs, cfg.record_cap = n_envs, 1000
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(N_TICKS)
    m.sync()
    sample = np.random.default_rng(M).integers(0, M, 4096)
    for b in range(n_envs):
        port = oracle.run_port(cfg, b, oracle.generate_ticks(cfg, b, N_TICKS), theta_at=sample)
        recs, _keep = m.records(b)
        _compare(recs, port, "M=%d env %d" % (M, b))  # trace_hash covers theta at every traced feature
        th = _device_theta(m, M, b)
        nz, vals = port["theta_nz"]
        assert len(nz) > 1000
        assert np.array_equal(th[nz].view(np.uint64), vals.view(np.uint64)), (M, b)
        assert np.array_equal(th[sample].view(np.uint64), port["theta_at"].view(np.uint64)), (M, b)
        assert np.count_nonzero(th) == len(nz), (M, b)
        del th
    m.close()


@pytest.mark.parametrize("M", [1 << 27, (1 << 27) + 1], ids=["one_warp_limit", "three_warp"])
def test_table_size_boundary_of_the_packed_tile_table(rlm, oracle, M):
    """2^27 is the last size the one-warp learner (packed (feature << 4 | action) tile table) takes; 2^27 + 1 is rerouted
    to the three-warp kernel.  About 1 GB of weights per env on the device, 2 GB per env for the oracle."""
    _full_scale(rlm, oracle, M, 2)


def _host_available_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


@pytest.mark.skipif(os.environ.get("RLM_TEST_HUGE_TABLES") != "1", reason="opt-in (RLM_TEST_HUGE_TABLES=1): 13 GB on the "
                    "device, ~26 GB on the host")
def test_table_above_2_to_the_30(rlm, oracle):
    """M = 1.5 * 2^30: group-0 tiles rebuilt from a stored base add two indices below M, whose sum passes INT_MAX."""
    import torch
    M = 3 << 29
    free, _total = torch.cuda.mem_get_info()
    if free < M * 8 + (2 << 30):
        pytest.skip("%.1f GB free on the device" % (free / 1e9))
    if _host_available_bytes() < M * 16 + (8 << 30):
        pytest.skip("%.1f GB available on the host" % (_host_available_bytes() / 1e9))
    _full_scale(rlm, oracle, M, 1)
