"""Agent::getQ / DoubleAgent::getQb on any state, without a GPU: oracle_get_q (the reference's sum over the oracle's tile
coding) against the reference's own values (tests/golden/q_values.json, tools/ref_q_values.cpp), and the C binding of
rlm_eval_q with its argument checks."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import oracle_lib
from rl_markets_b200 import abi, config, lib

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ALL_VARS = ["pos", "spd", "mpm", "imb", "svl", "vol", "rsi", "vwap", "a_dist", "a_queue", "b_dist", "b_queue", "last_action"]


def fixture_cases():
    with open(os.path.join(GOLD, "q_values.json")) as f:
        return json.load(f)["cases"]


def case_config(case, n_envs=1, seed=None, **kw):
    """The handle configuration of one fixture case: random_init tables drawn from random_seed (+ env_index0 + b)."""
    y = config.example_dict(**{"learning.memory_size": case["memory_size"], "learning.algorithm": case["algorithm"],
                               "learning.n_actions": case["n_actions"], "learning.random_init": True,
                               "debug.random_seed": case["random_seed"] if seed is None else seed,
                               "state.variables": ALL_VARS[:case["n_vars"]]})
    cfg = config.from_dict(y, n_envs=n_envs, **kw)
    assert list(cfg.group_weights) == case["group_weights"]
    return cfg


def case_queries(case):
    """(vars float32 [n][n_vars], expected float64 [n][n_tables][n_actions]) of one fixture case, bit for bit."""
    qs = case["queries"]
    vars_ = np.array([q["vars"] for q in qs], dtype=np.uint32).view(np.float32)
    tabs = ["q", "qb"] if case["algorithm"] == "double_q_learn" else ["q"]
    exp = np.array([[[int(h, 16) for h in q[t]] for t in tabs] for q in qs], dtype=np.uint64).view(np.float64)
    return vars_, exp


def tile_features(cfg, vars_):
    """State::newState(vars, .)'s feature indices of every query (the oracle's tiles(), lobo_tiles): int [n][A][96]."""
    L = oracle_lib.lib()
    vars_ = np.ascontiguousarray(vars_, dtype=np.float32)
    A, nv = cfg.n_actions, cfg.n_state_vars
    assert vars_.ndim == 2 and vars_.shape[1] == nv
    out = np.empty((len(vars_), A, 3 * abi.RLM_N_TILINGS), dtype=np.int32)
    for k in range(len(vars_)):
        L.lobo_tiles(C.byref(cfg), vars_[k].ctypes.data_as(C.POINTER(C.c_float)), out[k].ctypes.data_as(C.POINTER(C.c_int32)))
    return out


def oracle_get_q(cfg, theta_a, theta_b, vars_):
    """Agent::getQ / DoubleAgent::getQb (agent.cpp:117-135, 211-230) on caller tables (float64 [M]; theta_b None: one
    table) -> [n][1 or 2][n_actions], the layout of rlm_eval_q.  Features from the oracle's tiles(); the sum is the
    reference's, term by term in its order -- Q += w0*th (tilings 0..31), w1*th (32..63), w2*th (32..95: the third loop
    starts at T, SURVEY Appendix A8) -- one IEEE multiply and one add per term, vectorised over queries and actions only."""
    T = abi.RLM_N_TILINGS
    f = tile_features(cfg, vars_)
    w0, w1, w2 = (float(x) for x in cfg.group_weights)
    out = []
    for th in [theta_a] if theta_b is None else [theta_a, theta_b]:
        g = np.asarray(th, dtype=np.float64)[f]
        q = np.zeros(f.shape[:2])
        for i in range(T):
            q = q + w0 * g[:, :, i]
        for i in range(T, 2 * T):
            q = q + w1 * g[:, :, i]
        for i in range(T, 3 * T):
            q = q + w2 * g[:, :, i]
        out.append(q)
    return np.stack(out, axis=1)


def oracle_tables(cfg):
    """The oracle agent's random_init tables of env 0 (agent.cpp:37-39,190-192)."""
    L = oracle_lib.lib()
    h = L.lobo_create(C.byref(cfg), 0)
    try:
        M = cfg.memory_size
        a = np.ctypeslib.as_array(L.lobo_theta(h, 0), shape=(M,)).copy()
        dbl = cfg.algorithm in (abi.ALGO["double_q_learn"], abi.ALGO["double_r_learn"])
        b = np.ctypeslib.as_array(L.lobo_theta(h, 1), shape=(M,)).copy() if dbl else None
    finally:
        L.lobo_destroy(h)
    return a, b


def test_fixture_covers_the_configurations():
    cases = fixture_cases()
    assert {c["memory_size"] for c in cases} == {4096, 5003}
    assert {c["n_vars"] for c in cases} == {4, 8, 13}
    assert {c["algorithm"] for c in cases} == {"q_learn", "double_q_learn"}
    assert 9 in {c["n_actions"] for c in cases} and min(c["n_actions"] for c in cases) < 9
    for c in cases:
        v, _ = case_queries(c)
        assert np.isnan(v).any() and np.isinf(v).any() and (v < 0).any() and (np.abs(v) * 32 >= 2.0 ** 31).any()
        assert (v == 1.0 / 32).all(axis=1).any()  # a state on exact tile boundaries


@pytest.mark.parametrize("k", range(len(fixture_cases())))
def test_oracle_get_q_is_the_reference(k):
    case = fixture_cases()[k]
    cfg = case_config(case)
    vars_, exp = case_queries(case)
    ta, tb = oracle_tables(cfg)
    got = oracle_get_q(cfg, ta, tb, vars_)
    assert got.shape == exp.shape
    assert got.view(np.uint64).tolist() == exp.view(np.uint64).tolist()


def test_eval_q_binding_and_argument_checks():
    """rlm_eval_q is bound with the header's types, refuses a missing handle before it touches a device and leaves q_out
    as it was; the ABI version is unchanged by the addition."""
    L = lib.load()
    P = C.POINTER
    assert L.rlm_eval_q.argtypes == [C.c_void_p, P(C.c_float), P(C.c_int32), C.c_int64, P(C.c_double)]
    assert L.rlm_abi_version() == 4
    assert abi.RLM_EVAL_Q_CHUNK == 1 << 17
    header = open(os.path.join(os.path.dirname(GOLD), "..", "include", "rlm.h")).read()
    assert "#define RLM_EVAL_Q_CHUNK (1 << 17)" in header
    vars_ = (C.c_float * 8)()
    out = (C.c_double * 9)(*([7.0] * 9))
    assert L.rlm_eval_q(None, vars_, None, 1, out) == abi.RLM_ERR_INVALID_ARGUMENT
    assert "rlm_eval_q" in L.rlm_last_error().decode()
    assert L.rlm_eval_q(None, None, None, 0, out) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_eval_q(None, vars_, None, -1, None) == abi.RLM_ERR_INVALID_ARGUMENT
    assert list(out) == [7.0] * 9


def test_no_device_means_no_q_values():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    case = fixture_cases()[0]
    with pytest.raises(lib.RlmError) as ei:
        lib.BatchedMarket(case_config(case))
    assert ei.value.code == abi.RLM_ERR_NO_DEVICE


def test_q_values_checks_dtype_and_shape_first():
    """BatchedMarket.q_values refuses the wrong dtype or shape before calling the library (here: a handle-less object)."""
    cfg = case_config(fixture_cases()[0], n_envs=3)
    m = lib.BatchedMarket.__new__(lib.BatchedMarket)
    m.L, m.cfg, m.h = lib.load(), cfg, C.c_void_p()
    nv = cfg.n_state_vars
    with pytest.raises(TypeError):
        m.q_values(np.zeros((2, nv), dtype=np.float64))
    with pytest.raises(ValueError):
        m.q_values(np.zeros((2, nv + 1), dtype=np.float32))
    with pytest.raises(ValueError):
        m.q_values(np.zeros(nv, dtype=np.float32))
    with pytest.raises(TypeError):
        m.q_values(np.zeros((2, nv), dtype=np.float32), policy=np.zeros(2, dtype=np.int64))
    with pytest.raises(ValueError):
        m.q_values(np.zeros((2, nv), dtype=np.float32), policy=np.zeros(3, dtype=np.int32))
    with pytest.raises(ValueError):
        m.q_values(None, policy=np.zeros(3, dtype=np.int32))
    with pytest.raises(lib.RlmError) as ei:  # well-formed: the library refuses the null handle
        m.q_values(np.zeros((2, nv), dtype=np.float32))
    assert ei.value.code == abi.RLM_ERR_INVALID_ARGUMENT
    assert m.n_tables == 1
