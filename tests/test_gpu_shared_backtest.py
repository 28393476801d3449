"""Evaluation of a shared policy (main.cpp:216-242 for one theta across every env): backtest mode on a shared_policy
handle.  Backtester::_step (serial.cpp:121-137) never writes theta or the traces, so every env is exactly one reference
process that loaded that table: records and stats are compared bitwise with the CPU oracle, env by env
(lobo_create -> oracle_policy.set_theta -> lobo_go_greedy -> lobo_set_backtest -> lobo_run), unlike shared-policy training."""
import copy
import ctypes as C
import os

import numpy as np
import pytest

import golden_util as G
import oracle_policy
from rl_markets_b200 import abi, backtest, config, lib

pytestmark = pytest.mark.gpu
MSG = C.sizeof(abi.TickMsg)
T0_MS, DAY_TICKS = 57425000, 1000  # 250 ms ticks from 15:57:05: the close (16:00) and the closing ClearInventory are inside
CARRIED = ("n_traces", "trace_hash")  # see test_oracle_policy.py


def _yaml(algo, M):
    y = copy.deepcopy(G.backtest_manifest()[0]["yaml"])
    y["learning"]["algorithm"] = algo
    y["learning"]["memory_size"] = M
    return y


def _tables(m):
    """policy 0: Q_A, and Q_B of a Double-Q agent"""
    return [m.theta(0, k) for k in range(2 if m.cfg.algorithm == abi.ALGO["double_q_learn"] else 1)]


def _policy_bytes(m):
    """every byte evaluation must leave alone: the table(s) and the update accumulator"""
    return [bytes(t) for t in _tables(m)] + [m.dtheta_tensor().cpu().numpy().tobytes()]


def _train_shared(rlm, y, n_envs=16, n_ticks=300):
    """a shared policy trained for a few hundred ticks -> its table(s)"""
    m = rlm.BatchedMarket(config.from_dict(y, n_envs=n_envs, shared_policy=True, flow_seed=33))
    m.run_ticks(n_ticks)
    m.sync()
    th = _tables(m)
    assert np.count_nonzero(np.frombuffer(th[0], dtype=np.float64)) > 100
    m.close()
    return th


def _test_flow(y, seed=34):
    flow = config.from_dict(y, flow_seed=seed).flow
    flow.t0_ms = T0_MS
    return flow


def _evaluator(rlm, cfg, theta, flow=None):
    """fresh handle + loaded table(s) + GoGreedy + Backtester + (generator source) the new Intraday of main.cpp:219"""
    m = rlm.BatchedMarket(cfg)
    for p in range(1 if cfg.shared_policy else cfg.n_envs):
        for k, th in enumerate(theta):
            m.write_theta(th, p, k)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    if flow is not None:
        m.new_env(flow)
    return m


def _oracle_eval(oracle, cfg, b, theta, msgs, n):
    """env b of the handle as ONE reference process that loaded theta"""
    L = oracle.lib()
    c = abi.Config.from_buffer_copy(bytes(cfg))
    c.shared_policy = 0
    h = L.lobo_create(C.byref(c), cfg.env_index0 + b)
    for k, th in enumerate(theta):
        oracle_policy.set_theta(L, h, k, th, cfg.memory_size)
    L.lobo_go_greedy(h)
    L.lobo_set_backtest(h, 1)
    recs = (abi.StepRecord * n)()
    used = C.c_int64()
    steps = L.lobo_run(h, msgs, n, -1, recs, n, C.byref(used))
    st = abi.EnvStats()
    L.lobo_stats(h, C.byref(st))
    L.lobo_destroy(h)
    return [recs[i] for i in range(steps)], st, recs


def _assert_records(got, want, tag, skip=()):
    assert len(got) == len(want), (tag, len(got), len(want))
    for i in range(len(got)):
        bad = abi.record_fields_equal(got[i], want[i], skip=skip)
        assert not bad, (tag, i, G.describe_diff(got[i], want[i], bad))


@pytest.mark.parametrize("M", [4096, 2 * 2053])  # (a shared table has an even size: twice a prime takes the modulo path)
@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_shared_evaluation_matches_the_oracle(rlm, oracle, algo, M):
    B = 16
    y = _yaml(algo, M)
    theta = _train_shared(rlm, y)
    cfg = config.from_dict(y, n_envs=B, env_index0=7, shared_policy=True, flow_seed=33)
    cfg.record_envs, cfg.record_cap = B, 600
    flow = _test_flow(y)
    m = _evaluator(rlm, cfg, theta, flow)
    before = _policy_bytes(m)
    m.run_ticks(DAY_TICKS // 3)
    m.run_ticks(DAY_TICKS - DAY_TICKS // 3)
    m.sync()
    assert _policy_bytes(m) == before, "evaluation must not touch theta or dtheta"
    stats = m.stats()
    total = 0
    for b in range(B):
        day = rlm.flow_generate(flow, cfg.env_index0 + b, 0, DAY_TICKS)
        want, st, _k = _oracle_eval(oracle, m.cfg, b, theta, day, DAY_TICKS)
        got, _k2 = m.records(b)
        assert len(got) > 100, (b, len(got))
        _assert_records(got, want, (algo, M, b))
        assert stats[b].terminal == 1 and bytes(stats[b]) == bytes(st), (algo, M, b)
        total += len(got)
    assert m.counters().steps == total
    m.close()


def test_shared_evaluation_of_a_golden_policy(rlm):
    """The table an independent handle trained on a golden case, loaded into a shared handle whose env_index0 is the case's
    env: env 0 reproduces the reference's own evaluation records.  The reference evaluates with the Agent that trained
    (its trace list and generator positions travel along); a handle that loaded the table holds no traces, so n_traces
    and trace_hash -- which Backtester::_step never reads -- are the two fields left out."""
    for case in G.backtest_manifest():
        cfg = G.case_config(case, n_envs=1, env_index0=case["env"])
        cfg.flow.t0_ms = case["t0_ms"]
        tr = rlm.BatchedMarket(cfg)
        tr.run_ticks(case["ticks"])
        tr.sync()
        tr.handle_terminal(0)
        theta = _tables(tr)
        tr.close()
        t = case["test"]
        ecfg = config.from_dict(case["yaml"], n_envs=3, env_index0=t["env"], shared_policy=True, flow_seed=t["flow_seed"])
        ecfg.record_envs, ecfg.record_cap = 1, 600
        flow = config.from_dict(case["yaml"], flow_seed=t["flow_seed"]).flow
        flow.t0_ms = t["t0_ms"]
        m = _evaluator(rlm, ecfg, theta, flow)
        m.run_ticks(t["ticks"])
        m.sync()
        gold, _k = G.records(case["name"] + "_test")
        got, _k2 = m.records(0)
        assert len(gold) > 100
        _assert_records(got, gold, case["name"], skip=CARRIED)
        st, s = m.stats()[0], case["summary"]
        assert (st.terminal, st.position, st.episode_pnl, st.episode_reward, st.ask_transactions, st.bid_transactions,
                st.market_buys, st.market_sells) == (1, s["test_position"], s["test_ep_pnl"], s["test_ep_reward"],
                                                     s["test_ask_tx"], s["test_bid_tx"], s["test_market_buys"],
                                                     s["test_market_sells"])
        m.close()


@pytest.mark.parametrize("variant", [0, 1])  # warp-per-env and thread-per-env tick kernels
@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_shared_equals_independent(rlm, monkeypatch, algo, variant):
    """One table as policy 0 of a shared handle and as the policy of every env of an independent handle."""
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    B = 8
    y = _yaml(algo, 4096)
    theta = _train_shared(rlm, y)
    flow = _test_flow(y)
    ms = []
    for shared in (True, False):
        cfg = config.from_dict(y, n_envs=B, env_index0=3, shared_policy=shared, flow_seed=33)
        cfg.record_envs, cfg.record_cap = B, 600
        m = _evaluator(rlm, cfg, theta, flow)
        m.run_ticks(DAY_TICKS)
        m.sync()
        ms.append(m)
    for b in range(B):
        got, _k = ms[0].records(b)
        assert len(got) > 100
        _assert_records(got, ms[1].records(b)[0], (algo, variant, b))
    assert bytes(ms[0].stats()) == bytes(ms[1].stats())
    assert ms[0].counters().steps == ms[1].counters().steps
    for m in ms:
        m.close()


def _ingested():
    out = []
    for case in G.ingest_manifest():
        msgs, n, _ticks = lib.ingest_csv(*G.ingest_paths(case))
        out.append((case, msgs, n))
    return out


def test_shared_evaluation_on_a_day_library(rlm, oracle):
    """Tape source: the two ingested golden days as a library, envs alternating days under one table; then the days swapped."""
    ing = _ingested()
    case = ing[0][0]
    B, n_days = 4, len(ing)
    theta = _train_shared(rlm, case["yaml"])
    cfg = config.from_dict(case["yaml"], n_envs=B, env_index0=11, shared_policy=True, flow_seed=case["flow_seed"],
                           source=abi.SOURCE_TAPE)
    cfg.record_envs, cfg.record_cap = B, 1000
    offs = [0]
    for _c, _a, n in ing:
        offs.append(offs[-1] + n)
    buf = (abi.TickMsg * offs[-1])()
    for (_c, a, n), o in zip(ing, offs):
        C.memmove(C.addressof(buf) + o * MSG, a, n * MSG)
    m = _evaluator(rlm, cfg, theta)
    m.load_days(buf, offs)
    longest = max(n for _c, _a, n in ing)
    want = {}
    for b in range(B):
        for d in range(n_days):
            day = (abi.TickMsg * ing[d][2]).from_buffer_copy((C.c_char * (ing[d][2] * MSG)).from_address(C.addressof(ing[d][1])))
            want[b, d] = _oracle_eval(oracle, cfg, b, theta, day, ing[d][2])[0]
    before = _policy_bytes(m)
    for swap in (0, 1):
        days = [(b + swap) % n_days for b in range(B)]
        if swap:
            m.assign_days(days)
            m.new_env(None)
        m.run_ticks(longest // 3)
        m.run_ticks(longest)  # more than any day holds: envs stop at the end of theirs
        m.sync()
        assert m.tape_pos() == [ing[d][2] for d in days]
        for b in range(B):
            got, _k = m.records(b)
            assert len(got) > 20
            _assert_records(got, want[b, days[b]], ("tape", swap, b))
    assert [bytes(r) for r in want[0, 0]] != [bytes(r) for r in want[0, 1]], "the two days must tell the passes apart"
    assert _policy_bytes(m) == before
    m.close()


def test_train_evaluate_train_on_one_handle(rlm):
    y = _yaml("q_learn", 4096)
    cfg = config.from_dict(y, n_envs=16, shared_policy=True, flow_seed=33)
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(300)
    m.sync()
    trained = _policy_bytes(m)
    steps0 = m.counters().steps
    m.set_mode(abi.MODE_BACKTEST)
    m.new_env(_test_flow(y))
    m.run_ticks(DAY_TICKS)
    m.sync()
    assert m.counters().steps > steps0 + 16 * 100
    assert _policy_bytes(m) == trained
    m.set_mode(abi.MODE_TRAIN)
    m.reset()
    m.run_ticks(300)
    m.sync()
    assert _policy_bytes(m)[0] != trained[0], "training after the evaluation moves theta again"
    m.close()


def test_evaluation_needs_no_collective(rlm):
    cfg = config.from_dict(_yaml("q_learn", 4096), n_envs=4, shared_policy=True)
    m = rlm.BatchedMarket(cfg)
    m.set_mode(abi.MODE_BACKTEST)
    for call in (m.shared_tick_accumulate, m.apply_dtheta):
        with pytest.raises(rlm.RlmError) as ei:
            call()
        assert ei.value.code == abi.RLM_ERR_INVALID_ARGUMENT and "rlm_run_ticks" in str(ei.value)
    m.set_mode(abi.MODE_TRAIN)
    m.shared_tick_accumulate()
    m.apply_dtheta()
    m.sync()
    m.close()


def test_shared_backtest_needs_the_synchronous_engine(rlm, monkeypatch):
    monkeypatch.setenv("RLM_ENGINE", "f")
    m = rlm.BatchedMarket(config.from_dict(_yaml("q_learn", 4096), n_envs=2, shared_policy=True))
    with pytest.raises(rlm.RlmError) as ei:
        m.set_mode(abi.MODE_BACKTEST)
    assert ei.value.code == abi.RLM_ERR_UNSUPPORTED
    m.close()


def test_logs_of_a_shared_evaluation(rlm, tmp_path):
    y = _yaml("q_learn", 4096)
    theta = _train_shared(rlm, y)
    cfg = config.from_dict(y, n_envs=6, shared_policy=True, flow_seed=33)
    cfg.record_envs, cfg.record_cap = 6, 600
    m = _evaluator(rlm, cfg, theta, _test_flow(y))
    m.run_ticks(DAY_TICKS)
    m.sync()
    out = backtest.write_logs(m, str(tmp_path), env=3)
    rows = open(out["profit_log"]).read().splitlines()
    recs, _k = m.records(3)
    assert rows[0] == backtest.HEADER and len(rows) == 1 + len(recs) > 100
    assert int(rows[1].split(",")[2]) == recs[0].action and float(rows[-1].split(",")[4]) == recs[-1].midprice
    assert len(open(out["test_stats"]).read().splitlines()) == 8
    assert os.path.getsize(out["theta"]) == 8 * cfg.memory_size
    assert open(out["theta"], "rb").read() == bytes(m.theta(0, 0)) == bytes(theta[0])
    m.close()
