"""rlm_eval_q / BatchedMarket.q_values on the device: Agent::getQ / DoubleAgent::getQb (agent.cpp:117-135, 211-230) of
any state (State::newState(vars, .), state.cpp:45-51) and of every env's current decision state.

- the reference's own values on random_init tables (tests/golden/q_values.json), bit for bit, both tables of Double-Q;
- trained tables of every learner, power-of-two and other memory_size, both tick kernels: 10 000 random states with
  per-query policies against oracle_get_q (the reference's sum over the oracle's tile coding) on the read-back theta;
- the live form: under a greedy policy its argmax is the action rlm_act takes (train and backtest, independent and
  shared), and in backtest mode the action the next record carries;
- the call only reads: theta, records, rlm_env_stats and counters are those of the same run without queries;
- chunks, rejections, and the facade's Agent::getQ / getQb."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_q_values import case_config, case_queries, fixture_cases, oracle_get_q
from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOUBLE = (abi.ALGO["double_q_learn"], abi.ALGO["double_r_learn"])


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def tables(m, p):
    T = 2 if m.cfg.algorithm in DOUBLE else 1
    return [np.ctypeslib.as_array(m.theta(p, t)).copy() for t in range(T)]


def random_states(rng, n, nv):
    v = rng.uniform(-40.0, 40.0, size=(n, nv)).astype(np.float32)
    v[rng.random((n, nv)) < 0.1] = rng.integers(-64, 64, size=1)[0] / 32.0  # exact tile boundaries
    v[rng.random((n, nv)) < 0.01] = np.nan
    v[rng.random((n, nv)) < 0.01] = 3.0e9
    return v


def oracle_q(m, vars_, pol):
    """oracle_get_q on the handle's read-back tables, query by query under policy pol[i]."""
    T = 2 if m.cfg.algorithm in DOUBLE else 1
    out = np.empty((len(vars_), T, m.cfg.n_actions))
    for p in np.unique(pol):
        sel = np.nonzero(pol == p)[0]
        th = tables(m, int(p))
        out[sel] = oracle_get_q(m.cfg, th[0], th[1] if T == 2 else None, vars_[sel])
    return out


# ---------------------------------------------------------------- the reference's values
@pytest.mark.parametrize("k", range(len(fixture_cases())))
def test_reference_fixture(rlm, k):
    """Env 0 of a handle seeded S and env 2 of one seeded S - 2 both hold the reference's random_init tables of seed S
    (rlm_random_init_kernel draws env b's from random_seed + env_index0 + b)."""
    case = fixture_cases()[k]
    vars_, exp = case_queries(case)
    m = rlm.BatchedMarket(case_config(case))
    got = m.q_values(vars_)
    assert got.shape == exp.shape
    assert bits(got).tolist() == bits(exp).tolist()
    assert bits(m.q_values(vars_, np.zeros(len(vars_), dtype=np.int32))).tolist() == bits(exp).tolist()
    m.close()
    m3 = rlm.BatchedMarket(case_config(case, n_envs=3, seed=case["random_seed"] - 2))
    got = m3.q_values(vars_, np.full(len(vars_), 2, dtype=np.int32))
    assert bits(got).tolist() == bits(exp).tolist()
    m3.close()


# ---------------------------------------------------------------- trained tables
@pytest.mark.parametrize("variant", [0, 1], ids=["warp", "thread"])
@pytest.mark.parametrize("M", [4096, 5003])
@pytest.mark.parametrize("algo", ["q_learn", "sarsa", "double_q_learn", "r_learn"])
def test_trained_tables(rlm, monkeypatch, algo, M, variant):
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo, "policy.eps_init": 0.3,
                               "learning.alpha_start": 0.05})
    B = 4
    m = rlm.BatchedMarket(config.from_dict(y, n_envs=B, flow_seed=5))
    m.run_ticks(600)
    m.sync()
    assert m.counters().steps > 20 * B
    rng = np.random.default_rng(M + variant)
    n = 10000
    vars_ = random_states(rng, n, m.cfg.n_state_vars)
    pol = rng.integers(0, B, size=n).astype(np.int32)
    got = m.q_values(vars_, pol)
    exp = oracle_q(m, vars_, pol)
    assert bits(got).tolist() == bits(exp).tolist()
    m.close()


# ---------------------------------------------------------------- the live form
def _strict_argmax(row):
    if np.isnan(row).any():
        return None
    mx = row.max()
    return int(np.argmax(row)) if (row == mx).sum() == 1 else None


def _sampled(q):
    """the vector Agent::action samples: Q_A, or (Q_A + Q_B) / 2.0 for double agents (agent.cpp:60-74, 202-209)"""
    return q[:, 0] if q.shape[1] == 1 else (q[:, 0] + q[:, 1]) / 2.0


def _drive(m, steps, query):
    """the split surface for `steps` decisions; with `query`, the live form is checked before every rlm_act.  Returns the
    actions taken per env and the number of strict-maximum rows checked."""
    B = m.cfg.n_envs
    m.env_step(None)
    m.agent_update()
    taken, checked = [[] for _ in range(B)], 0
    for i in range(steps):
        if query:
            q = m.q_values()
            assert q.shape == (B, 2 if m.cfg.algorithm in DOUBLE else 1, m.cfg.n_actions)
            if i > 0:  # (the first decision of a learner's first episode is made in the never-populated State)
                # the live form is the explicit form on rlm_get_state's vectors under each env's policy
                pol = np.zeros(B, np.int32) if m.cfg.shared_policy else np.arange(B, dtype=np.int32)
                st = np.ctypeslib.as_array(m.state()).reshape(B, m.cfg.n_state_vars).copy()
                assert bits(m.q_values(st, pol)).tolist() == bits(q).tolist()
            s = _sampled(q)
        a = list(m.act())
        for b in range(B):
            if a[b] >= 0:
                taken[b].append(a[b])
                if query:
                    k = _strict_argmax(s[b])
                    if k is not None:
                        assert k == a[b], (b, s[b], a[b])
                        checked += 1
        if all(x < 0 for x in a):
            break
        m.env_step((C.c_int32 * B)(*a))
        m.agent_update()
    return taken, checked


def _snapshot(m):
    B = m.cfg.n_envs
    th = [bits(t).tobytes() for p in range(1 if m.cfg.shared_policy else B) for t in tables(m, p)]
    recs = [[bytes(r) for r in m.records(b)[0]] for b in range(m.cfg.record_envs)]
    st = bytes(m.stats())
    c = m.counters()
    return th, recs, st, (c.ticks, c.steps, c.sum_traces, c.terminal_envs)


@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_live_form_train(rlm, algo):
    """Train mode on the split surface, greedy policy: every strict maximum of the live rows is rlm_act's action, and the
    same run without the queries ends in the same theta, records, stats and counters."""
    y = config.example_dict(**{"learning.memory_size": 8192, "learning.algorithm": algo, "policy.type": "greedy",
                               "learning.random_init": True})
    cfg = config.from_dict(y, n_envs=6, flow_seed=9)
    cfg.record_envs, cfg.record_cap = 6, 600
    runs = []
    for query in (True, False):
        m = rlm.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
        taken, checked = _drive(m, 150, query)
        if query:
            assert checked > 300
        runs.append((taken, _snapshot(m)))
        m.close()
    assert runs[0] == runs[1]


@pytest.mark.parametrize("shared", [False, True], ids=["independent", "shared"])
@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_live_form_backtest(rlm, algo, shared):
    """Backtest mode (Backtester::_step): the strict maximum of the live rows is rlm_act's action and the action of the
    step's record."""
    # (a shared table's memory_size is even: 5002; independent tables take any: 5003)
    y = config.example_dict(**{"learning.memory_size": 5002 if shared else 5003, "learning.algorithm": algo, "policy.type": "greedy"})
    B = 5
    cfg = config.from_dict(y, n_envs=B, flow_seed=13, shared_policy=shared)
    cfg.record_envs, cfg.record_cap = B, 800
    m = rlm.BatchedMarket(cfg)
    rng = np.random.default_rng(3)
    for p in range(1 if shared else B):
        for t in range(2 if algo == "double_q_learn" else 1):
            m.write_theta((C.c_double * cfg.memory_size)(*rng.uniform(-1, 1, cfg.memory_size)), policy=p, table=t)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    taken, checked = _drive(m, 400, True)
    assert checked > 200
    for b in range(B):
        recs = [r.action for r in m.records(b)[0]]
        assert len(recs) > 50 and recs == taken[b][:len(recs)], b
    m.close()


# ---------------------------------------------------------------- read-only
@pytest.mark.parametrize("engine", [{"RLM_ROUNDS": "1"}, {"RLM_ROUNDS": "0"}], ids=["rounds", "ticksync"])
def test_queries_change_nothing(rlm, monkeypatch, engine):
    for k, v in engine.items():
        monkeypatch.setenv(k, v)
    y = config.example_dict(**{"learning.memory_size": 16384, "learning.algorithm": "double_q_learn"})
    cfg = config.from_dict(y, n_envs=40, flow_seed=21)
    cfg.record_envs, cfg.record_cap = 4, 400
    rng = np.random.default_rng(7)
    vars_ = random_states(rng, 3000, cfg.n_state_vars)
    pol = rng.integers(0, 40, size=3000).astype(np.int32)
    snaps = []
    for query in (True, False):
        m = rlm.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
        for _ in range(5):
            m.run_ticks(200)
            if query:
                m.q_values()
                m.q_values(vars_, pol)
        m.sync()
        snaps.append(_snapshot(m))
        m.close()
    assert snaps[0] == snaps[1]


def test_queries_change_nothing_shared(rlm):
    """A shared handle queried between rlm_apply_dtheta and the next accumulate, and between accumulate and apply."""
    y = config.example_dict(**{"learning.memory_size": 65536, "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=32, flow_seed=23, shared_policy=True)
    cfg.record_envs, cfg.record_cap = 4, 400
    vars_ = random_states(np.random.default_rng(9), 2000, cfg.n_state_vars)
    snaps, dth = [], []
    for query in (True, False):
        m = rlm.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
        for t in range(400):
            m.shared_tick_accumulate()
            if query and t % 50 == 7:
                m.q_values(vars_)
                m.q_values()
            m.apply_dtheta()
            if query and t % 50 == 3:
                m.q_values(vars_)
        m.sync()
        snaps.append(_snapshot(m))
        dth.append(m.dtheta_tensor().cpu().numpy().tobytes())
        m.close()
    assert snaps[0] == snaps[1] and dth[0] == dth[1]


# ---------------------------------------------------------------- chunks and rejections
def test_chunks(rlm):
    n0 = abi.RLM_EVAL_Q_CHUNK
    y = config.example_dict(**{"learning.memory_size": 4096, "learning.algorithm": "double_q_learn", "learning.random_init": True})
    m = rlm.BatchedMarket(config.from_dict(y, n_envs=4))
    rng = np.random.default_rng(11)
    vars_ = random_states(rng, n0 + 3, m.cfg.n_state_vars)
    pol = rng.integers(0, 4, size=n0 + 3).astype(np.int32)
    whole = m.q_values(vars_, pol)
    parts = np.concatenate([m.q_values(vars_[:n0], pol[:n0]), m.q_values(vars_[n0:], pol[n0:])])
    assert bits(whole).tolist() == bits(parts).tolist()
    sel = rng.choice(n0 + 3, 2000, replace=False)
    sel[:3] = [n0, n0 + 1, n0 + 2]
    assert bits(whole[sel]).tolist() == bits(oracle_q(m, vars_[sel], pol[sel])).tolist()
    m.close()


def test_rejections(rlm):
    y = config.example_dict(**{"learning.memory_size": 4096, "learning.algorithm": "q_learn"})
    B, A = 3, 9
    L = rlm.load()
    P = C.POINTER
    for shared in (False, True):
        m = rlm.BatchedMarket(config.from_dict(y, n_envs=B, shared_policy=shared))
        nv = m.cfg.n_state_vars
        vars_ = (C.c_float * (4 * nv))()
        out = (C.c_double * (8 * A))(*([42.0] * (8 * A)))
        fv = C.cast(vars_, P(C.c_float))
        hi = 1 if shared else B
        cases = [
            (m.h, fv, (C.c_int32 * 4)(0, 0, -1, 0), 4, out),
            (m.h, fv, (C.c_int32 * 4)(0, hi, 0, 0), 4, out),
            (m.h, fv, None, -1, out),
            (m.h, fv, None, 4, None),
            (None, fv, None, 4, out),
            (m.h, None, None, B + 1, out),
            (m.h, None, None, B - 1, out),
            (m.h, None, (C.c_int32 * B)(), B, out),
        ]
        for args in cases:
            assert L.rlm_eval_q(*args) == abi.RLM_ERR_INVALID_ARGUMENT, (shared, args)
            assert list(out) == [42.0] * (8 * A)
        assert L.rlm_eval_q(m.h, fv, None, 0, out) == abi.RLM_OK and list(out) == [42.0] * (8 * A)
        assert L.rlm_eval_q(m.h, fv, (C.c_int32 * 4)(0, hi - 1, 0, 0), 4, out) == abi.RLM_OK
        m.close()


# ---------------------------------------------------------------- the class surface
FACADE_SRC = r'''
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "rlm_facade.hpp"
int main(int argc, char** argv) {  // argv: config file (raw rlm_config), then the state's variables as float bit patterns
  rlm_config cfg;
  FILE* f = fopen(argv[1], "rb");
  if (!f || fread(&cfg, sizeof(cfg), 1, f) != 1) return 2;
  fclose(f);
  rlm::Session s(cfg);
  rlm::rl::Agent m(s);
  std::vector<float> v;
  for (int i = 2; i < argc; ++i) { unsigned u = (unsigned)strtoul(argv[i], nullptr, 10); float x; memcpy(&x, &u, 4); v.push_back(x); }
  const bool dbl = cfg.algorithm == RLM_ALGO_DOUBLE_Q_LEARN || cfg.algorithm == RLM_ALGO_DOUBLE_R_LEARN;
  for (int t = 0; t < (dbl ? 2 : 1); ++t)
    for (int a = 0; a < cfg.n_actions; ++a) {
      const double q = t ? m.getQb(v, a) : m.getQ(v, a);
      unsigned long long u; memcpy(&u, &q, 8); printf("%llu\n", u);
    }
  if (!dbl) { try { m.getQb(v, 0); return 3; } catch (const std::invalid_argument&) {} }
  return 0;
}
'''


@pytest.mark.parametrize("k", [0, 2])
def test_facade_getq(rlm, k):
    case = fixture_cases()[k]
    cfg = case_config(case)
    vars_, exp = case_queries(case)
    with tempfile.TemporaryDirectory() as d:
        src, exe, cf = os.path.join(d, "q.cpp"), os.path.join(d, "q"), os.path.join(d, "cfg.bin")
        open(src, "w").write(FACADE_SRC)
        open(cf, "wb").write(bytes(cfg))
        libdir = os.path.join(ROOT, "rl_markets_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), src, "-L" + libdir, "-lrlm",
                               "-Wl,-rpath," + libdir, "-o", exe])
        m = rlm.BatchedMarket(cfg)
        for i in (0, 8, 11, 20):
            out = subprocess.check_output([exe, cf] + [str(u) for u in vars_[i].view(np.uint32)]).split()
            got = np.array([int(x) for x in out], dtype=np.uint64)
            assert got.tolist() == bits(m.q_values(vars_[i:i + 1])).ravel().tolist() == bits(exp[i]).ravel().tolist()
        m.close()
