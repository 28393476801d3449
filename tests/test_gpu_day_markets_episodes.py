"""Day markets across episodes, in backtest mode and in shared-policy training, against the CPU oracle whose env takes
the day's market as the reference's Intraday::LoadData does (tests/oracle_market.py), bitwise.

* Episodes: two envs, three training episodes each; every episode is rlm_handle_terminal, rlm_assign_days to a day of
  another market, rlm_reset (main.cpp:53-58 with LoadData(ticker, ...) before each episode).  One boundary is the
  midprice-memo case: env 0's second day is its first day with the book of the first episode's last tick on the first
  100 rows after the open, replayed under LSE group B after a first day under group A -- so the first midprice the
  second episode converts is the one whose group A tick count next_state_tail has memoised, and it stays there into the
  first learner step.
* The same boundary reached by calling rlm_set_day_markets again with other markets under the same indices.
* rlm_new_env between two days under day markets: the records start again and the closing record is terminal.
* Backtest mode, independent and shared policies: a loaded table, GoGreedy, each env its day under its market.
* Shared-policy Q-learning over five days under four markets (one closing mid-run) with the lockstep checker."""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest

import golden_util as G
import oracle_market as OM
import oracle_policy
from rl_markets_b200 import abi, config
from rl_markets_b200 import lib as rlm_lib
from test_gpu_tape import _library

pytestmark = pytest.mark.gpu

with open(os.path.join(G.GOLD, "day_markets.json")) as _f:
    DM = json.load(_f)
_VENUE = {c["name"]: c for c in G.venue_manifest()}
CAP = 3000
MSG = C.sizeof(abi.TickMsg)


def _day(ticker):
    case = _VENUE[next(d["venue_case"] for d in DM["days"] if d["ticker"] == ticker)]
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day(case, d)
        msgs, n, _t = rlm_lib.ingest_csv(md, tas)
    return msgs, n


def _cfg(n_envs, env0, shared=False, algo="q_learn"):
    y = dict(DM["yaml"])
    y = json.loads(json.dumps(y))
    y["learning"]["algorithm"] = algo
    cfg = config.from_dict(y, n_envs=n_envs, env_index0=env0, source=abi.SOURCE_TAPE, shared_policy=shared)
    cfg.record_envs, cfg.record_cap = n_envs, CAP
    return cfg


def _oracle_env(oracle, cfg, b):
    c = abi.Config.from_buffer_copy(bytes(cfg))
    c.shared_policy = 0
    return oracle.lib().lobo_create(C.byref(c), cfg.env_index0 + b)


def _oracle_run(oracle, h, msgs, n):
    L = oracle.lib()
    recs = (abi.StepRecord * CAP)()
    used = C.c_int64()
    k = L.lobo_run(h, msgs, n, -1, recs, CAP, C.byref(used))
    return [recs[i] for i in range(k)], used.value


def _assert_records(got, want, tag):
    assert len(got) == len(want), (tag, len(got), len(want))
    for i in range(len(got)):
        bad = abi.record_fields_equal(got[i], want[i])
        assert not bad, (tag, i, G.describe_diff(got[i], want[i], bad))


def _oracle_theta(oracle, h, M):
    p = oracle.lib().lobo_theta(h, 0)
    return bytes((C.c_double * M).from_address(C.addressof(p.contents)))


def _memo_day(base, n, last_msg, open_lo, rows=100):
    """`base` with the book of `last_msg` on `rows` rows from the open on: the first midprice NextState converts is the
    memoised one, and it stays there through the warm-up (the longest window holds 60 values) into the first step, so
    the mid-price window the first state reads (mpm: its oldest value against its newest) holds its tick counts"""
    out = (abi.TickMsg * n)()
    C.memmove(out, base, n * MSG)
    j = next(i for i in range(n) if out[i].time_ms > open_lo)
    assert out[j - 1].flags == 0
    for r in range(j, j + rows):
        t, d = out[r].time_ms, out[r].date
        C.memmove(C.addressof(out) + r * MSG, C.addressof(last_msg), MSG)
        out[r].time_ms, out[r].date, out[r].flags, out[r].n_tx = t, d, 0, 0
    return out


@pytest.mark.parametrize("env", [{"RLM_ENGINE": "s"}, {"RLM_ROUNDS": "1"}, {"RLM_ENV_VARIANT": "1"}], ids=["s", "rounds1", "thread"])
def test_episodes_across_markets_and_the_midprice_memo(rlm, oracle, monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    L = oracle.lib()
    cfg = _cfg(2, 70)
    aal, baes, pa = _day("AAL.L"), _day("BAES.L"), _day("X.PA")
    A, Bm, E = config.market("AAL.L"), config.market("BAES.L"), config.market("X.PA")
    # env 0's first episode on the oracle: where it ends decides the memo day
    h0 = _oracle_env(oracle, cfg, 0)
    OM.set_market(h0, A)
    recs0, used0 = _oracle_run(oracle, h0, *aal)
    last = aal[0][used0 - 1]
    mid = (float(last.ask_px[0]) + float(last.bid_px[0])) / 2.0
    assert recs0[-1].terminal == 1 and recs0[-1].midprice == mid, "the first episode ends on the last message's book"
    assert L.lobo_to_ticks(C.byref(config.from_dict(DM["yaml"], ticker="AAL.L")), mid) != \
        L.lobo_to_ticks(C.byref(config.from_dict(DM["yaml"], ticker="BAES.L")), mid), "the two tables differ there"
    memo = (_memo_day(aal[0], aal[1], last, A.open_ms + 30 * 60000), aal[1])
    days = [aal, baes, pa, memo]  # day 3 runs under LSE B
    day_market = [0, 1, 2, 1]
    plan = [[0, 1], [3, 2], [2, 0]]  # episode -> day of env 0, env 1
    markets = [A, Bm, E]
    m = rlm.BatchedMarket(cfg)
    buf, offs = _library(days)
    m.load_days(buf, offs)
    m.set_day_markets(markets, day_market)
    hs = [h0, _oracle_env(oracle, cfg, 1)]
    n_before = [0, 0]
    for ep, ds in enumerate(plan):
        if ep:
            m.handle_terminal(ep)
        m.assign_days(ds)
        if ep:
            m.reset()
        T = max(days[d][1] for d in ds)
        m.run_ticks(T)
        m.sync()
        st = m.stats()
        for b, d in enumerate(ds):
            h = hs[b]
            if ep:
                L.lobo_handle_terminal(h, ep)
                OM.set_market(h, markets[day_market[d]])
                L.lobo_reset(h)
                want, _u = _oracle_run(oracle, h, *days[d])
            elif b == 0:
                want = recs0
            else:
                OM.set_market(h, markets[day_market[d]])
                want, _u = _oracle_run(oracle, h, *days[d])
            got, _k = m.records(b)
            _assert_records(got[n_before[b]:], want, ("episode", ep, "env", b))
            n_before[b] = len(got)
            assert want[-1].terminal == 1 and st[b].terminal == 1, (ep, b)
            so = abi.EnvStats()
            L.lobo_stats(h, C.byref(so))
            assert bytes(st[b]) == bytes(so), (ep, b)
            assert bytes(m.theta(b)) == _oracle_theta(oracle, h, cfg.memory_size), (ep, b)
    for h in hs:
        L.lobo_destroy(h)
    m.close()


def test_new_markets_under_the_same_indices_forget_the_memo(rlm, oracle):
    """rlm_set_day_markets again with other markets and the same day -> market indices: env 0's market changes from
    LSE A to LSE B although its index stays 0, on the memo day of the test above"""
    L = oracle.lib()
    cfg = _cfg(1, 72)
    aal = _day("AAL.L")
    A, Bm = config.market("AAL.L"), config.market("BAES.L")
    h = _oracle_env(oracle, cfg, 0)
    OM.set_market(h, A)
    want1, used = _oracle_run(oracle, h, *aal)
    last = aal[0][used - 1]
    memo = _memo_day(aal[0], aal[1], last, A.open_ms + 30 * 60000)
    m = rlm.BatchedMarket(cfg)
    buf, offs = _library([aal, (memo, aal[1])])
    m.load_days(buf, offs)
    m.set_day_markets([A], [0, 0])
    m.assign_days([0])
    m.run_ticks(aal[1])
    m.sync()
    m.handle_terminal(1)
    m.set_day_markets([Bm], [0, 0])
    m.assign_days([1])
    m.reset()
    m.run_ticks(aal[1])
    m.sync()
    L.lobo_handle_terminal(h, 1)
    OM.set_market(h, Bm)
    L.lobo_reset(h)
    want2, _u = _oracle_run(oracle, h, memo, aal[1])
    got, _k = m.records(0)
    _assert_records(got, want1 + want2, "memo under a replaced market")
    assert bytes(m.theta(0)) == _oracle_theta(oracle, h, cfg.memory_size)
    L.lobo_destroy(h)
    m.close()


def test_new_env_between_days_keeps_the_closing_record_terminal(rlm):
    """records start again at rlm_new_env; the second day's closing record still gets its market's close"""
    cfg = _cfg(1, 61)  # (env 61 on the BAES.L day: day_markets.json's reference run)
    baes, aal = _day("BAES.L"), _day("AAL.L")
    m = rlm.BatchedMarket(cfg)
    buf, offs = _library([baes, aal])
    m.load_days(buf, offs)
    m.set_day_markets([config.market("BAES.L"), config.market("AAL.L")], [0, 1])
    m.assign_days([0])
    m.run_ticks(baes[1])
    m.sync()
    first, _k = m.records(0)
    assert [G.record_digest(r) for r in first] == G.digests("daymkt_venue_baes_l")
    m.new_env()
    m.assign_days([1])
    m.run_ticks(aal[1])
    m.sync()
    second, _k = m.records(0)
    assert 0 < len(second) < len(first)  # (the AAL day has fewer steps: a stale fix-up mark would skip all of them)
    assert second[-1].terminal == 1 and sum(r.terminal for r in second) == 1
    m.close()


@pytest.mark.parametrize("shared", [False, True], ids=["independent", "shared"])
def test_backtest_across_markets(rlm, oracle, shared):
    L = oracle.lib()
    tickers = ["AAL.L", "BAES.L", "X.PA", "X.ST", "X.I", "X.CO"]
    days = [_day(t) for t in tickers]
    markets = [config.market(t) for t in tickers]
    B = len(tickers)
    cfg = _cfg(B, 80, shared=shared)
    M = cfg.memory_size
    rng = np.random.default_rng(7)
    thetas = [rng.uniform(-1.0, 1.0, M) for _ in range(1 if shared else B)]
    m = rlm.BatchedMarket(cfg)
    for p, th in enumerate(thetas):
        m.write_theta((C.c_double * M)(*th), p, 0)
    buf, offs = _library(days)
    m.load_days(buf, offs)
    m.set_day_markets(markets, list(range(B)))
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    m.run_ticks(max(n for _a, n in days))
    m.sync()
    st = m.stats()
    for b in range(B):
        h = _oracle_env(oracle, cfg, b)
        OM.set_market(h, markets[b])
        oracle_policy.set_theta(L, h, 0, (C.c_double * M)(*thetas[0 if shared else b]), M)
        L.lobo_go_greedy(h)
        L.lobo_set_backtest(h, 1)
        want, _u = _oracle_run(oracle, h, *days[b])
        got, _k = m.records(b)
        _assert_records(got, want, ("backtest", tickers[b]))
        so = abi.EnvStats()
        L.lobo_stats(h, C.byref(so))
        assert st[b].terminal == 1 and bytes(st[b]) == bytes(so), tickers[b]
        L.lobo_destroy(h)
    m.close()


def test_shared_lockstep_across_markets(rlm, oracle):
    """Q-learning, one table of 4096 weights, 64 envs on five synthetic days under four markets: LSE A (the config's),
    LSE B, the Irish market, and LSE B closing 75 s into the run, so that its envs end their episode mid-run"""
    from test_gpu_shared_lockstep import MSG as LMSG, Lockstep, _cfg as lockstep_cfg, _report
    n_ticks, n_days, day_len = 600, 5, 700
    cfg = lockstep_cfg("q_learn", 4096, 64, seed=55, source=abi.SOURCE_TAPE)
    short = config.market("BAES.L")
    short.close_ms = cfg.flow.t0_ms + 30 * 60000 + 300 * cfg.flow.dt_ms
    markets = [config.market("AAL.L"), config.market("BAES.L"), config.market("X.I"), short]
    day_market = [0, 1, 2, 3, 3]
    days = [rlm.flow_generate(cfg.flow, 100 + d, 0, day_len) for d in range(n_days)]
    lib = (abi.TickMsg * (n_days * day_len))()
    for d, a in enumerate(days):
        C.memmove(C.addressof(lib) + d * day_len * LMSG, a, day_len * LMSG)
    offs = [d * day_len for d in range(n_days + 1)]
    msgs = np.empty((n_ticks, cfg.n_envs, LMSG), dtype=np.uint8)
    for b in range(cfg.n_envs):
        msgs[:, b, :] = np.frombuffer(days[b % n_days], dtype=np.uint8).reshape(day_len, LMSG)[:n_ticks]

    def setup(m, first, n):
        m.load_days(lib, offs)
        m.assign_days([(first + i) % n_days for i in range(n)])
        m.set_day_markets(markets, day_market)

    ls = Lockstep(rlm, oracle, cfg, msgs, setup=setup)
    try:
        for e in range(cfg.n_envs):
            OM.batch_set_market(ls.b, e, markets[day_market[e % n_days]])
        ls.run(n_ticks)
        t = ls.finish("markets")
        _report("markets", ls, n_ticks)
        assert ls.compared > cfg.record_envs * 20
        assert t.max_k >= 3 and t.fraction >= 0.99, t
        st = ls.ms[0].stats()
        ended = [b for b in range(cfg.n_envs) if st[b].terminal]
        assert ended == [b for b in range(cfg.n_envs) if day_market[b % n_days] == 3], ended
    finally:
        ls.close()
