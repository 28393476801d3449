"""oracle_policy.set_theta, the test side's checkpoint loader for the oracle (the reference has none, SURVEY section 5):
evaluating env b of a shared policy is lobo_create(b) -> set_theta -> lobo_go_greedy -> lobo_set_backtest(1) -> lobo_run
on b's day.  Pinned here without a GPU against the oracle's own train-then-evaluate sequence and against the reference's
evaluation records."""
import ctypes as C

import golden_util as G
import oracle_lib as oracle
import oracle_policy
from rl_markets_b200 import abi, config

# A freshly created env holds no traces, and its generators stand at their seeds; the agent that trained the table carries
# both into its evaluation (main.cpp:216-222 keeps the Agent).  Backtester::_step never reads the traces, so the records
# differ in these two diagnostics only.
CARRIED = ("n_traces", "trace_hash")


def _run(L, h, ticks, n):
    recs = (abi.StepRecord * n)()
    used = C.c_int64()
    steps = L.lobo_run(h, ticks, n, -1, recs, n, C.byref(used))
    assert steps >= 0
    return [recs[i] for i in range(steps)], recs


def _stats(L, h):
    st = abi.EnvStats()
    L.lobo_stats(h, C.byref(st))
    return bytes(st)


def test_set_theta_round_trips():
    L = oracle.lib()
    for algo, tables in (("q_learn", 1), ("double_q_learn", 2)):
        M = 4099
        cfg = config.from_dict(config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo}))
        h = L.lobo_create(C.byref(cfg), 5)
        vals = [(C.c_double * M)(*[(t + 1) * 0.25 * i - 3.0 for i in range(M)]) for t in range(tables)]
        for t in range(tables):
            oracle_policy.set_theta(L, h, t, vals[t], M)
        for t in range(tables):
            assert bytes(oracle_policy.theta_view(L, h, t, M)) == bytes(vals[t]), (algo, t)
        assert (oracle_policy.theta_view(L, h, 1, M) is None) == (tables == 1)
        L.lobo_destroy(h)


def test_evaluating_a_loaded_table_equals_train_then_evaluate():
    """The oracle trains a golden case, evaluates it the way main.cpp does (same Agent, new Intraday) -- which reproduces
    the reference's evaluation records -- and the same table loaded into a fresh env gives the same evaluation."""
    L = oracle.lib()
    for case in G.backtest_manifest():
        cfg = G.case_config(case)
        cfg.flow.t0_ms = case["t0_ms"]
        M = cfg.memory_size
        trained = L.lobo_create(C.byref(cfg), case["env"])
        _run(L, trained, oracle.lib_generate(cfg, case["env"], case["ticks"]), case["ticks"])
        assert L.lobo_is_terminal(trained) == 1
        L.lobo_handle_terminal(trained, 0)
        tables = 1 if oracle_policy.theta_view(L, trained, 1, M) is None else 2  # (Double-Q: Q_B as well)
        theta = [oracle_policy.theta_view(L, trained, k, M) for k in range(tables)]
        theta_bytes = [bytes(th) for th in theta]
        t = case["test"]
        cfg2 = config.from_dict(case["yaml"], flow_seed=t["flow_seed"])
        cfg2.flow.t0_ms = t["t0_ms"]
        day = oracle.lib_generate(cfg2, t["env"], t["ticks"])
        fresh = L.lobo_create(C.byref(cfg2), t["env"])
        for k in range(tables):
            oracle_policy.set_theta(L, fresh, k, theta[k], M)
        L.lobo_go_greedy(fresh)
        L.lobo_set_backtest(fresh, 1)
        got, _k1 = _run(L, fresh, day, t["ticks"])
        L.lobo_go_greedy(trained)
        L.lobo_set_backtest(trained, 1)
        L.lobo_new_env(trained)
        own, _k2 = _run(L, trained, day, t["ticks"])
        gold, _k3 = G.records(case["name"] + "_test")
        assert len(got) == len(own) == len(gold) > 100, (case["name"], len(got), len(own), len(gold))
        for i in range(len(got)):
            assert not abi.record_fields_equal(own[i], gold[i]), (case["name"], i)
            bad = abi.record_fields_equal(got[i], gold[i], skip=CARRIED)
            assert not bad, (case["name"], i, G.describe_diff(got[i], gold[i], bad))
            assert got[i].n_traces == 0
        assert L.lobo_is_terminal(fresh) == 1 and _stats(L, fresh) == _stats(L, trained)
        for h in (fresh, trained):  # evaluation leaves the table alone
            for k in range(tables):
                assert bytes(oracle_policy.theta_view(L, h, k, M)) == theta_bytes[k]
        L.lobo_destroy(fresh)
        L.lobo_destroy(trained)
