"""The training logs on the GPU (rlm_set_model_log / rlm_read_model_log / rlm_get_policy_descr and
rl_markets_b200.train_logs) against the reference's own files (tests/golden/training_logs.json and
tl_<case>_{model_log,training_log}.csv, tools/make_golden.py --training-logs) and the CPU oracle, bitwise.

* Every learner path the accumulation pass follows: the round-paced engine with and without CUDA graphs, the tick-
  synchronous engine with and without graphs, 100-tick calls, the staged, one-warp, three-warp (both EXTRAS: the R-learning
  agents take the other one) and round-1 learners, the thread-per-env tick kernel, the tape source, the split surface
  (act / env_step / agent_update) and a shared handle of one env (the reference).  Env 0's files equal the fixtures byte for byte; env 1, another reference
  process, equals the oracle.
* Shared handles of many envs: env b's values are the sequential sum of its own recorded deltas.
* The count runs on across handle_terminal / reset / new_env and a backtest interlude, which adds no value -- through
  rlm_run_ticks and through the split surface.
* More values than cap_rows between two reads: the read reports the loss.
* With the log off (never on, or on and off again), records, statistics, theta and kernel_launches are those of a handle
  that never had it; with it on, everything but kernel_launches is."""
import ctypes as C
import os

import pytest

import test_training_logs as TL
from rl_markets_b200 import abi, train_logs

pytestmark = pytest.mark.gpu

PATHS = {
    "rounds": {},
    "rounds_nograph": {"RLM_GRAPHS": "0"},
    "ticksync": {"RLM_ROUNDS": "0"},
    "ticksync_nograph": {"RLM_ROUNDS": "0", "RLM_GRAPHS": "0"},
    "one_warp": {"RLM_STAGED": "0"},
    "three_warp": {"RLM_AGENT_VARIANT": "3"},
    "round1": {"RLM_AGENT_VARIANT": "1"},
    "thread_tick": {"RLM_ENV_VARIANT": "1"},
}
SHARED_ALGOS = ("q_learn", "sarsa", "double_q_learn")


def _source(c):
    return abi.SOURCE_TAPE if any("venue" in d for d in c["days"]) else abi.SOURCE_GENERATOR


class Training:
    """One handle through a case's episodes as main.cpp's train() runs them (rlm_run_ticks in whole-day calls, or
    `chunk`-tick calls, or split=True: Learner::_step as rlm_act / rlm_env_step / rlm_agent_update), with TrainingLogs
    for every env."""

    def __init__(self, rlm, c, out_dir, n_envs=1, chunk=None, shared=False, records=False, log=True, split=False):
        self.c = c
        cfg = TL.base_config(c, n_envs=n_envs, source=_source(c), shared_policy=shared)
        if records:
            cfg.record_envs, cfg.record_cap = n_envs, TL.CAP * c["episodes"]
        self.m = m = rlm.BatchedMarket(cfg)
        self.logs = [train_logs.TrainingLogs(m, os.path.join(out_dir, "env%d" % b), env=b) for b in range(n_envs)] if log else []
        if cfg.source == abi.SOURCE_TAPE:
            self._lib, n = TL.day_messages(c["name"], 0)
            m.load_days(self._lib, [0, n])
            m.reset()
        for e in range(c["episodes"]):
            self.episode(e, chunk, split)

    def episode(self, e, chunk, split=False):
        c, m = self.c, self.m
        k = e % len(c["days"])
        if e:
            if len(c["days"]) > 1:
                m.set_flow(TL.day_flow(c, k))
            m.reset()
        T = TL.day_messages(c["name"], k)[1]
        if split:
            split_episode(m)
        else:
            step = chunk or T
            for t0 in range(0, T, step):
                m.run_ticks(min(step, T - t0))
        m.sync()
        assert all(s.terminal for s in m.stats()), (c["name"], e)
        m.handle_terminal(e)
        for b, lg in enumerate(self.logs):
            lg.episode_end(e, c["episode_ids"][e])

    def files(self, b):
        return tuple(open(self.logs[b].paths[k]).read() for k in ("model_log", "training_log"))


def split_episode(m):
    """Runner::RunEpisode on the split surface, as include/rlm_facade.hpp drives it: Initialise and the first from-state,
    then act / performAction / HandleTransition until act reports the end of the episode (-1) for every env.  In
    backtest mode the same calls are Backtester::_step."""
    m.env_step(None)
    m.agent_update()
    while True:
        a = m.act()
        if all(x < 0 for x in a):
            return
        m.env_step(a)
        m.agent_update()


def _check_env(c, tr, b):
    got = tr.files(b)
    if b == 0:
        want = (TL.fixture(c, "model_log"), TL.fixture(c, "training_log"))
    else:
        ml, tl, _v = TL.expected_files(c, TL.oracle_run(c["name"], b))
        want = (ml, tl)
    assert got[0] == want[0], (c["name"], b, "model_log")
    assert got[1] == want[1], (c["name"], b, "training_log")


@pytest.mark.parametrize("name", [c["name"] for c in TL.CASES])
@pytest.mark.parametrize("path", ["rounds", "ticksync", "ticksync_nograph"])
def test_every_case_against_the_reference(rlm, monkeypatch, tmp_path, name, path):
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    c = TL.case(name)
    tr = Training(rlm, c, str(tmp_path), n_envs=2)
    for b in range(2):
        _check_env(c, tr, b)
    tr.m.close()


@pytest.mark.parametrize("path", ["rounds_nograph", "one_warp", "three_warp", "round1", "thread_tick"])
@pytest.mark.parametrize("name", ["tl_q_learn_eps", "tl_double_q_greedy", "tl_r_learn"])
def test_learner_and_tick_kernels(rlm, monkeypatch, tmp_path, name, path):
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    c = TL.case(name)
    tr = Training(rlm, c, str(tmp_path), n_envs=2)
    for b in range(2):
        _check_env(c, tr, b)
    tr.m.close()


@pytest.mark.parametrize("name", ["tl_q_learn_two_days", "tl_venue_aal", "tl_sarsa_boltzmann"])
def test_short_calls(rlm, tmp_path, name):
    c = TL.case(name)
    tr = Training(rlm, c, str(tmp_path), n_envs=2, chunk=100)
    for b in range(2):
        _check_env(c, tr, b)
    tr.m.close()


@pytest.mark.parametrize("name", ["tl_q_learn_eps", "tl_double_r_learn", "tl_venue_aal", "tl_q_learn_two_days"])
def test_split_surface(rlm, tmp_path, name):
    c = TL.case(name)
    tr = Training(rlm, c, str(tmp_path), n_envs=2, split=True)
    for b in range(2):
        _check_env(c, tr, b)
    tr.m.close()


def test_split_surface_across_a_backtest_interlude(rlm):
    """split-surface training, a test day evaluated on the split surface (new_env, backtest mode), split-surface training
    on fresh env objects: the evaluation adds no value, and every env's values are the sequential sum of its recorded
    training deltas"""
    c = TL.case("tl_q_learn_eps")
    n_envs = 3
    cfg = TL.base_config(c, n_envs=n_envs)
    cfg.record_envs, cfg.record_cap = n_envs, TL.CAP * 4
    m = rlm.BatchedMarket(cfg)
    m.set_model_log(64)
    deltas = [[] for _ in range(n_envs)]
    got = [[] for _ in range(n_envs)]

    def drain():
        for b, v in enumerate(m.model_log()):
            got[b] += v

    def train(e0, e1):
        for e in range(e0, e1):
            if e != e0:
                m.reset()
            split_episode(m)
            m.handle_terminal(e)
            drain()
        for b in range(n_envs):
            deltas[b] += _record_deltas(m, b)

    train(0, 3)
    m.set_mode(abi.MODE_BACKTEST)
    m.new_env()
    split_episode(m)
    m.sync()
    before = [len(g) for g in got]
    drain()
    assert [len(g) for g in got] == before, "evaluation logs nothing"
    assert all(len(_record_deltas(m, b)) > 100 for b in range(n_envs)), "the test day ran"
    m.set_mode(abi.MODE_TRAIN)
    m.new_env()                            # (new env objects: the records start again)
    train(3, 6)
    m.sync()
    for b in range(n_envs):
        vals, _a, _n = train_logs.model_log_values(deltas[b])
        assert len(vals) >= 2 and got[b] == vals, b
    m.close()


@pytest.mark.parametrize("name", [c["name"] for c in TL.CASES if c["algo"] in SHARED_ALGOS and c["M"] % 2 == 0])
def test_shared_handle_of_one_env_is_the_reference(rlm, tmp_path, name):
    c = TL.case(name)
    tr = Training(rlm, c, str(tmp_path), n_envs=1, shared=True)
    _check_env(c, tr, 0)
    tr.m.close()


def _record_deltas(m, b):
    recs, _k = m.records(b)
    return [r.delta for r in recs]


@pytest.mark.parametrize("name", ["tl_q_learn_eps", "tl_double_q_greedy", "tl_venue_aal"])
def test_shared_handle_of_many_envs(rlm, tmp_path, name):
    c = TL.case(name)
    n_envs = 5
    tr = Training(rlm, c, str(tmp_path), n_envs=n_envs, shared=True, records=True)
    for b in range(n_envs):
        vals, _a, _n = train_logs.model_log_values(_record_deltas(tr.m, b))
        assert len(vals) >= 2
        assert tr.files(b)[0] == "".join(v + "\n" for v in train_logs.model_log_lines(vals)), (name, b)
    tr.m.close()


@pytest.mark.parametrize("path", ["rounds", "ticksync"])
def test_count_runs_across_resets_new_env_and_backtest(rlm, monkeypatch, path):
    """train, evaluate a day (new_env, backtest mode), back to training on fresh env objects: only training updates count,
    and the 1000-update windows run on through all of it"""
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    c = TL.case("tl_q_learn_eps")
    n_envs = 3
    cfg = TL.base_config(c, n_envs=n_envs)
    cfg.record_envs, cfg.record_cap = n_envs, TL.CAP * 4
    m = rlm.BatchedMarket(cfg)
    m.set_model_log(64)
    T = c["days"][0]["ticks"]
    deltas = [[] for _ in range(n_envs)]
    got = [[] for _ in range(n_envs)]

    def take_records():
        for b in range(n_envs):
            deltas[b] += _record_deltas(m, b)

    def drain():
        for b, v in enumerate(m.model_log()):
            got[b] += v

    for e in range(3):
        if e:
            m.reset()
        m.run_ticks(T)
        m.handle_terminal(e)
        drain()
    take_records()
    m.set_mode(abi.MODE_BACKTEST)          # a test day: Backtester steps move n_steps, HandleTransition never runs
    m.new_env()
    m.run_ticks(T)
    m.sync()
    assert m.counters().steps > 0
    before = [len(g) for g in got]
    drain()
    assert [len(g) for g in got] == before, "evaluation logs nothing"
    m.set_mode(abi.MODE_TRAIN)
    m.new_env()                            # (new env objects: the records start again)
    for e in range(3, 6):
        if e > 3:
            m.reset()
        m.run_ticks(T)
        m.handle_terminal(e)
    take_records()
    drain()
    m.sync()
    for b in range(n_envs):
        vals, _a, _n = train_logs.model_log_values(deltas[b])
        assert len(vals) >= 2 and got[b] == vals, b
    m.close()


def test_overflow_is_reported(rlm):
    c = TL.case("tl_q_learn_eps")
    m = rlm.BatchedMarket(TL.base_config(c, n_envs=2))
    m.set_model_log(1)
    T = c["days"][0]["ticks"]
    for e in range(c["episodes"]):
        if e:
            m.reset()
        m.run_ticks(T)
        m.handle_terminal(e)
    with pytest.raises(rlm.RlmError) as ei:
        m.model_log()
    assert "lost" in str(ei.value) and ei.value.code == abi.RLM_ERR_RUNTIME
    assert m.model_log() == [[], []]       # the read drained every env
    m.sync()                               # no device error
    m.close()


def test_arguments_and_policy_descr(rlm, monkeypatch):
    c = TL.case("tl_sarsa_boltzmann")
    cfg = TL.base_config(c, n_envs=2)
    m = rlm.BatchedMarket(cfg)
    L, h = m.L, m.h
    rows, n = (C.c_double * 8)(), (C.c_int32 * 2)()
    assert L.rlm_read_model_log(h, 0, 2, rows, n) == abi.RLM_ERR_INVALID_ARGUMENT   # off
    assert L.rlm_set_model_log(h, -1) == abi.RLM_ERR_INVALID_ARGUMENT
    m.set_model_log(4)
    n[0] = n[1] = 77
    assert L.rlm_read_model_log(h, 1, 2, rows, n) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_read_model_log(h, -1, 1, rows, n) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_read_model_log(h, 0, 1, None, n) == abi.RLM_ERR_INVALID_ARGUMENT
    assert list(n) == [77, 77]
    assert L.rlm_get_policy_descr(h, None) == abi.RLM_ERR_INVALID_ARGUMENT
    assert m.policy_descr() == float(cfg.tau_init)
    for e in range(3):
        m.handle_terminal(e)
        assert m.policy_descr() == TL.policy_descr(cfg, e)
    m.go_greedy()
    assert m.policy_descr() == 0.0
    m.close()
    monkeypatch.setenv("RLM_ENGINE", "F")
    m2 = rlm.BatchedMarket(TL.base_config(TL.case("tl_q_learn_eps")))
    with pytest.raises(rlm.RlmError) as ei:
        m2.set_model_log(16)
    assert ei.value.code == abi.RLM_ERR_UNSUPPORTED
    m2.close()


@pytest.mark.parametrize("path", ["rounds", "ticksync"])
def test_log_off_changes_nothing(rlm, monkeypatch, path):
    for k, v in PATHS[path].items():
        monkeypatch.setenv(k, v)
    c = TL.case("tl_double_q_greedy")
    T = c["days"][0]["ticks"]

    def run(setup):
        cfg = TL.base_config(c, n_envs=4)
        cfg.record_envs, cfg.record_cap = 4, TL.CAP * 3
        m = rlm.BatchedMarket(cfg)
        setup(m)
        for e in range(3):
            if e:
                m.reset()
            m.run_ticks(T)
            m.run_ticks(60)
            m.handle_terminal(e)
        m.sync()
        out = dict(recs=[bytes(r) for b in range(4) for r in m.records(b)[0]], stats=[bytes(s) for s in m.stats()],
                   theta=[bytes(m.theta(b, t)) for b in range(4) for t in range(2)], launches=m.counters().kernel_launches,
                   steps=m.counters().steps)
        m.close()
        return out

    never = run(lambda m: None)
    off_again = run(lambda m: (m.set_model_log(8), m.set_model_log(0)))
    on = run(lambda m: m.set_model_log(8))
    assert off_again == never
    assert on["launches"] > never["launches"]
    on.pop("launches"), never.pop("launches")
    assert on == never
