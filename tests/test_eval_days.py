"""Evaluation over several test days, as src/main.cpp:216-244 runs it: GoGreedy once, ONE Intraday object built before
the loop, and for each test day LoadData, a new Backtester, Initialise, the steps and ClearInventory.  Base::Initialise
(base.cpp:123-150) does not clear everything: Accumulator::clear keeps its sum and RollingMean its mean and variance
(A13), the position and the greedy agent's rand() state carry on too, so from the second day on the state variables
start from the previous day's leftovers.

The fixtures (tests/golden/eval_days.json, digests_ed_*.bin) are the reference's own records of every day
(tools/make_golden.py --eval-days).  Here the CPU oracle reproduces them with the port's sequence -- lobo_new_env for
the first day, lobo_reset (plus the day's market, for a day of another ticker) for every later one -- and
backtest.write_logs renders the reference's multi-day profit_log.csv and test_stats.csv from those records.  The
sensitivity test shows that each case pins the carried state: a new env object per day differs from it on day 2."""
import ctypes as C
import functools
import hashlib
import json
import os
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, backtest, config
from rl_markets_b200 import lib as rlm_lib

with open(os.path.join(G.GOLD, "eval_days.json")) as _f:
    CASES = json.load(_f)
_VENUE = {c["name"]: c for c in G.venue_manifest()}
CAP = 4000


def case_ids():
    return [c["name"] for c in CASES]


def case(name):
    return next(c for c in CASES if c["name"] == name)


def train_config(c, **kw):
    """the case's config, its training day's flow"""
    cfg = config.from_dict(c["yaml"], flow_seed=c["flow_seed"], **kw)
    cfg.flow.t0_ms = c["t0_ms"]
    return cfg


def day_flow(c, k):
    """synthetic-flow parameters of test day k (a generated day)"""
    day = c["days"][k]
    flow = config.from_dict(c["yaml"], flow_seed=day["flow_seed"]).flow
    flow.t0_ms = day["t0_ms"]
    return flow


def day_market(c, k):
    """abi.Market of test day k when it is a day of a named ticker, else None (the config's market)"""
    return config.market(c["days"][k]["ticker"]) if "ticker" in c["days"][k] else None


@functools.lru_cache(maxsize=None)
def day_messages(name, k, env_index=None):
    """test day k of case `name` as one env's message stream -> (ctypes TickMsg array, message count).  A generated
    day is the flow of env `env_index` (default: the case's env); a venue day is the CSV pair tools/venue_csv.py writes,
    checked against the sha256 stored with the fixture and ingested."""
    c = case(name)
    day = c["days"][k]
    if "venue" not in day:
        n = day["ticks"]
        return rlm_lib.flow_generate(day_flow(c, k), c["env"] if env_index is None else env_index, 0, n), n
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day(_VENUE[day["venue"]], d)
        for p, key in ((md, "md_sha256"), (tas, "tas_sha256")):
            assert hashlib.sha256(open(p, "rb").read()).hexdigest() == day[key], (name, k, p)
        msgs, n, _t = rlm_lib.ingest_csv(md, tas)
    return msgs, n


def assert_digests(recs, name, tag):
    want = G.digests(name)
    assert len(recs) == len(want), (tag, len(recs), len(want))
    for i, r in enumerate(recs):
        assert G.record_digest(r) == want[i], (tag, "first differing record", i)


def day_stats_match(st, s):
    """rlm_env_stats / lobo_stats after a day against the reference's summary of that day (after ClearInventory)"""
    return (st.terminal, st.position, st.episode_pnl, st.episode_reward, st.ask_transactions, st.bid_transactions,
            st.market_buys, st.market_sells) == (1, s["test_position"], s["test_ep_pnl"], s["test_ep_reward"],
                                                 s["test_ask_tx"], s["test_bid_tx"], s["test_market_buys"],
                                                 s["test_market_sells"])


def oracle_evaluation(oracle, c, carry=True, env_index=None, theta=None):
    """The oracle through the case: train on its day until the close (or load the tables `theta` instead),
    HandleTerminal, GoGreedy, backtest, then every test day -- lobo_new_env before day 1 and, carry=True, lobo_reset
    (+ the day's market) before each later day; carry=False builds a new env object for every day.
    -> (training records, [(records, stats) per day])"""
    L = oracle.lib()
    env_index = c["env"] if env_index is None else env_index
    cfg = train_config(c)
    h = L.lobo_create(C.byref(cfg), env_index)
    assert h
    train_recs = []
    if theta is not None:
        import oracle_policy
        for k, th in enumerate(theta):
            oracle_policy.set_theta(L, h, k, th, cfg.memory_size)
    else:
        ticks = rlm_lib.flow_generate(cfg.flow, env_index, 0, c["ticks"])
        recs = (abi.StepRecord * c["ticks"])()
        used = C.c_int64()
        n = L.lobo_run(h, ticks, c["ticks"], -1, recs, c["ticks"], C.byref(used))
        assert n > 100 and L.lobo_is_terminal(h) == 1
        train_recs = [recs[i] for i in range(n)]
    L.lobo_handle_terminal(h, 0)   # Learner::RunEpisode, serial.cpp:79
    L.lobo_go_greedy(h)            # main.cpp:217
    L.lobo_set_backtest(h, 1)
    days = []
    for k in range(len(c["days"])):
        if k == 0 or not carry:
            L.lobo_new_env(h)      # environment::Intraday<> env(c), main.cpp:219
        else:
            L.lobo_reset(h)        # LoadData + the new Backtester's Initialise on the same env object
        mk = day_market(c, k)
        if mk is not None:
            import oracle_market
            oracle_market.set_market(h, mk)  # LoadData(ticker, ...): make_market (intraday.cpp:141-150)
        msgs, n = day_messages(c["name"], k, None if env_index == c["env"] else env_index)
        recs = (abi.StepRecord * CAP)()
        used = C.c_int64()
        steps = L.lobo_run(h, msgs, n, -1, recs, CAP, C.byref(used))
        assert 0 <= steps <= CAP and L.lobo_is_terminal(h) == 1, (c["name"], k, steps)
        st = abi.EnvStats()
        L.lobo_stats(h, C.byref(st))
        days.append(([recs[i] for i in range(steps)], st))
    L.lobo_destroy(h)
    return train_recs, days


@functools.lru_cache(maxsize=None)
def _carried(oracle, name):
    return oracle_evaluation(oracle, case(name))


@pytest.mark.parametrize("name", case_ids())
def test_oracle_reproduces_every_day(oracle, name):
    c = case(name)
    train_recs, days = _carried(oracle, name)
    assert len(days) == len(c["days"]) >= 2
    assert_digests(train_recs, name + "_train", (name, "train"))
    for k, (recs, st) in enumerate(days):
        assert len(recs) == c["days"][k]["n_records"] > 100, (name, k)
        assert_digests(recs, "%s_day%d" % (name, k), (name, "day", k))
        assert day_stats_match(st, c["days"][k]["summary"]), (name, k)


@pytest.mark.parametrize("name", case_ids())
def test_multi_day_logs_match_the_reference_files(oracle, name):
    """One profit_log.csv over every day (the Backtester ctor of day 2 on finds the loggers registered and writes no
    second header) and the test_stats.csv Base::writeStats leaves after the last day."""
    c = case(name)
    _train, days = _carried(oracle, name)
    recs = [r for d, _st in days for r in d]
    last = days[-1][1]

    class Handle:  # what backtest.write_logs reads of a handle
        cfg = train_config(c)

        def records(self, env):
            return recs, None

        def stats(self, env, n):
            return [last]

        def theta(self, policy):
            return b""

    with tempfile.TemporaryDirectory() as d:
        out = backtest.write_logs(Handle(), d, env=0)
        for key, fname in (("profit_log", "profit_log.csv"), ("test_stats", "test_stats.csv")):
            got = hashlib.sha256(open(out[key], "rb").read()).hexdigest()
            assert got == c["logs_sha256"][fname], (name, fname)


@pytest.mark.parametrize("name", case_ids())
def test_a_new_env_object_per_day_differs_on_day_two(oracle, name):
    """Sensitivity: every case tells main.cpp's one env object from a new one per day, in a state variable of some
    day-2 record -- a case that did not would pin nothing of what the env carries."""
    c = case(name)
    _t, carried = _carried(oracle, name)
    _t2, fresh = oracle_evaluation(oracle, c, carry=False)
    assert [bytes(r) for r in fresh[0][0]] == [bytes(r) for r in carried[0][0]], "day 1 is the same in both"
    assert first_state_difference(carried[1][0], fresh[1][0]) is not None, (name, "day 2 does not depend on day 1")


def first_state_difference(a, b):
    """index of the first record pair that differs in the state variables (None: no pair does)"""
    for i in range(min(len(a), len(b))):
        if "state" in abi.record_fields_equal(a[i], b[i]):
            return i
    return None
