"""The batch oracle of shared-policy training (lobo_batch_*) against the reference, and the dtheta checker of
tests/shared_lockstep.py against the oracle's own sums.  No GPU needed.

With one env a shared tick is theta_{t+1} = theta_t + that env's update, and dtheta = 0 + c is exact (the trace list
holds each feature once): the batch is the reference's Learner.  Only trace_hash differs by definition -- a shared
record hashes theta_t, before the apply; an independent one hashes theta after its own update."""
import ctypes as C

import numpy as np
import pytest

import golden_util as G
import shared_lockstep as S
from rl_markets_b200 import abi, config


def _batch(oracle, cfg):
    from test_shared_policy_cpu import _oracle_batch
    L, b = _oracle_batch(cfg)
    return S.bind(L), b


def shared_cases():
    """The golden training cases shared mode accepts: Q-learning / SARSA / Double-Q, an even table, no random_init."""
    return [c for c in G.manifest() if c["algo"] in ("q_learn", "sarsa", "double_q_learn") and c["M"] % 2 == 0
            and not c["yaml"]["learning"].get("random_init")]


def run_batch_one(oracle, case):
    """The case's env as a shared batch of one, fed the case's ticks -> (records, theta tables, stats, steps, traces)"""
    cfg = G.case_config(case, n_envs=1, env_index0=case["env"])
    cfg.shared_policy = 1
    L, b = _batch(oracle, cfg)
    ticks = oracle.lib_generate(cfg, case["env"], case["ticks"])
    cap = case["ticks"]
    recs = (abi.StepRecord * cap)()
    cnt = (C.c_int32 * 1)()
    for t in range(case["ticks"]):
        L.lobo_batch_accumulate(b, C.byref(ticks[t]), C.addressof(recs), C.addressof(cnt), cap)
        L.lobo_batch_apply(b)
    M = cfg.memory_size
    th = [np.ctypeslib.as_array(L.lobo_batch_theta(b, t), shape=(M,)).copy() for t in range(2 if case["algo"] == "double_q_learn" else 1)]
    st = abi.EnvStats()
    L.lobo_batch_stats(b, 0, C.byref(st))
    out = ([recs[i] for i in range(cnt[0])], th, st, L.lobo_batch_steps(b), L.lobo_batch_sum_traces(b), recs)
    L.lobo_batch_destroy(b)
    return out


def test_shared_cases_cover_the_issue_list():
    names = {c["name"] for c in shared_cases()}
    assert {"m2_staged", "m8194_gather", "m8190_staged_sarsa", "lambda0_q", "long_traces_sarsa", "sarsa_boltzmann_m8192",
            "double_q_m65536", "rew_mm_exp"} <= names
    assert not names & {"m1_gather", "m3_gather", "m97_gather", "q_learn_m5003_greedy", "q_learn_m4096_random_init"}


@pytest.mark.parametrize("name", [c["name"] for c in shared_cases()])
def test_batch_of_one_is_the_reference_learner(oracle, name):
    """lobo_batch with one env against lobo_run (θ, statistics, counters, every record field) and against the golden
    records of the reference (every field but trace_hash)."""
    case = [c for c in shared_cases() if c["name"] == name][0]
    recs, th, st, steps, traces, _keep = run_batch_one(oracle, case)
    cfg = G.case_config(case)
    L = oracle.lib()
    h = L.lobo_create(C.byref(cfg), case["env"])
    ticks = oracle.lib_generate(cfg, case["env"], case["ticks"])
    port = (abi.StepRecord * case["ticks"])()
    used = C.c_int64()
    n = L.lobo_run(h, ticks, case["ticks"], -1, port, case["ticks"], C.byref(used))
    assert len(recs) == n == steps > 100, (name, len(recs), n)
    for i in range(n):
        bad = abi.record_fields_equal(recs[i], port[i], skip=("trace_hash",))
        assert not bad, "%s step %d (batch, lobo_run): %r" % (name, i, G.describe_diff(recs[i], port[i], bad))
    gold, _k = G.records(name)
    assert len(gold) <= n
    for i, g in enumerate(gold):
        bad = abi.record_fields_equal(g, recs[i], skip=("trace_hash",))
        assert not bad, "%s step %d (reference, batch): %r" % (name, i, G.describe_diff(g, recs[i], bad))
    M = cfg.memory_size
    for t in range(len(th)):
        ref = np.ctypeslib.as_array(L.lobo_theta(h, t), shape=(M,))
        assert th[t].tobytes() == ref.tobytes(), (name, t)
    so = abi.EnvStats()
    L.lobo_stats(h, C.byref(so))
    assert bytes(st) == bytes(so), name
    assert traces == L.lobo_sum_traces(h), name
    L.lobo_destroy(h)


def _log_run(oracle, algo, n_envs, n_ticks, M, log, at=()):
    """A shared batch of the synthetic flow; with the log on, (log, dense dtheta) of the ticks in `at` come back"""
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
    cfg = config.from_dict(y, n_envs=n_envs, shared_policy=True, flow_seed=33)
    L, b = _batch(oracle, cfg)
    L.lobo_batch_log(b, 1 if log else 0)
    streams = [oracle.lib_generate(cfg, i, n_ticks) for i in range(n_envs)]
    cap = n_ticks
    recs = (abi.StepRecord * (n_envs * cap))()
    cnt = (C.c_int32 * n_envs)()
    msgs = (abi.TickMsg * n_envs)()
    nt = 2 if algo == "double_q_learn" else 1
    seen, tally = {}, S.Tally()
    for t in range(n_ticks):
        for i in range(n_envs):
            msgs[i] = streams[i][t]
        L.lobo_batch_accumulate(b, msgs, C.addressof(recs), C.addressof(cnt), cap)
        if log:
            lg = S.log_entries(L, b)
            d = np.concatenate([np.ctypeslib.as_array(L.lobo_batch_dtheta(b, k), shape=(M,)) for k in range(nt)])
            r = S.check(lg, d, M)  # the oracle's own env-order sum obeys the bound
            assert not r["bad"], (algo, t, r["bad"])
            tally.add(r)
            if t in at:
                seen[t] = (lg, d.copy())
        L.lobo_batch_apply(b)
    th = b"".join(np.ctypeslib.as_array(L.lobo_batch_theta(b, k), shape=(M,)).tobytes() for k in range(nt))
    out = {"theta": th, "records": bytes(recs), "count": list(cnt), "steps": L.lobo_batch_steps(b), "seen": seen,
           "tally": tally}
    L.lobo_batch_destroy(b)
    return out


@pytest.mark.parametrize("algo", ["q_learn", "sarsa", "double_q_learn"])
def test_the_log_changes_no_number(oracle, algo):
    """With the log on the batch adds exactly what it adds with it off; its own dtheta passes the checker every tick."""
    on = _log_run(oracle, algo, 8, 300, 2048, True)
    off = _log_run(oracle, algo, 8, 300, 2048, False)
    assert on["steps"] == off["steps"] > 200
    assert on["theta"] == off["theta"] and on["records"] == off["records"] and on["count"] == off["count"]
    t = on["tally"]
    assert t.max_k >= 3 and t.touched > 1000 and t.fraction > 0.1, t


_MUT = {}


def _mutation_tick(oracle):
    """(log, dtheta) of the last tick of a 64-env Double-Q run with a sensitive weight of three or more contributions"""
    if not _MUT:
        M, n = 2048, 600
        seen = _log_run(oracle, "double_q_learn", 64, n, M, True, at=set(range(n)))["seen"]
        for t in sorted(seen, reverse=True):
            _u, k, _s, _tol, sens = S.sums(seen[t][0], M)
            if (sens & (k >= 3)).any():
                _MUT["tick"] = seen[t]
                break
    return _MUT["tick"]


@pytest.mark.parametrize("how", ["drop", "double", "move"])
def test_checker_flags_one_wrong_addition(oracle, how):
    """The oracle's own Double-Q dtheta passes; the same dtheta summed without one contribution, with one twice, or with
    one in the other table does not -- at the sensitive weight with the most contributions of the tick."""
    M = 2048
    lg, d = _mutation_tick(oracle)
    assert not S.check(lg, d, M)["bad"]
    bad_d, k = S.mutate(lg, d, M, how, np.random.default_rng(7))
    assert k >= 3, k  # the bound, not only the bitwise rule, has to catch it
    r = S.check(lg, bad_d, M)
    assert r["bad"], (how, k)
    # the sparse form of the same dtheta is held to the same rules
    nz = np.flatnonzero(bad_d)
    assert S.check(lg, (nz, bad_d[nz]), M)["bad"]
    nz = np.flatnonzero(d)
    assert not S.check(lg, (nz, d[nz]), M)["bad"]


def test_checker_flags_a_stray_and_a_k1_change(oracle):
    M, tick = 2048, 299
    lg, d = _log_run(oracle, "q_learn", 16, 300, M, True, at=(tick,))["seen"][tick]
    uniq, k, s, _tol, _sens = S.sums(lg, M)
    untouched = np.setdiff1d(np.arange(M), uniq)[0]
    x = d.copy()
    x[untouched] = 1e-300
    assert S.check(lg, x, M)["bad"][0][:3] == (0, int(untouched), 0)
    one = uniq[k == 1]
    if len(one):
        x = d.copy()
        x[one[0]] = np.nextafter(x[one[0]], np.inf)  # one ulp off a single addition
        assert S.check(lg, x, M)["bad"]
