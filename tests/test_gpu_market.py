"""The market side away from the default synthetic day, on every tick kernel, against the reference and the CPU oracle,
bitwise.

Venue days (tests/golden manifest entries with venue_day, tools/venue_csv.py): one whole trading day per venue tick table
whose best bid crosses a band boundary many times and which ends at the venue's own close.  Four envs per case: the env
carrying the case's seeds replays the case's day and must give the reference's records through the terminal step; the
other envs replay other days of the same writer and must give the oracle's records, theta and statistics.  This runs on
the tape source through the tick-synchronous warp kernel, the round-paced kernel, the thread-per-env kernel, the default
selection in 100-tick calls and the split surface (act / env_step / agent_update), and on the stream source (the case's
day for every env) through the persistent and fused engines RLM_ENGINE=F, f and p.

Every other end-to-end run keeps the price inside LSE group A's [1000, 5000) band and ends at the LSE close.  Here the
synthetic flow straddles band boundaries of other venue tables, with tick sizes the flow's float prices do not hit
exactly (Euronext 0.005 | 0.01 at 50, Nordic 0.5 | 1.0 at 1000, Euronext 0.001 | 0.005 at 10), and each day ends at its
own venue's close (Paris 17:30, Stockholm 17:30, the Irish 16:16 plus 40 ms).  A thin, fast flow (three lots per level,
spreads mostly three ticks, a move almost every 100 ms row, prints that never / always reach the second level) drives
the book paths a deep book never meets.  The oracle's conversions are pinned to the reference at every band boundary by
units.json market_sweep (test_oracle_golden.py::test_market_band_sweep).

Each flow runs 40 envs on the generator source (default long-call selection, RLM_ROUNDS=0, the thread-per-env kernel,
one env per CTA of the warp-per-env kernel) and on the stream source (default selection, RLM_ENGINE=F, f, p); six
sampled envs equal the oracle fed the host rendering of the same flow (rlm_flow_generate, which honours every
parameter), and the stream run of those host messages equals the generator run in every env, so the in-kernel flow
(flow_next_warp, rlm_flow_next) equals rlm_flow_apply at these parameters.

The reference's throw: ToPrice of a negative tick count (market.cpp:112) is ERR_TICK_RANGE on the device, reported by
rlm_sync as RLM_ERR_INVALID_ARGUMENT.  On a Nordic bottom-band day the oracle raises at some step s in every env, and every
kernel gives the oracle's records before s and the matching error."""
import ctypes as C
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, config
from rl_markets_b200 import lib as rlm_lib
from test_gpu_tape import _assert_port, _assert_same, _library, _wide

pytestmark = pytest.mark.gpu

B, N_TICKS, OPEN_ROWS = 40, 1500, 1200
SAMPLED = [0, 7, 13, 22, 31, 39]


def _flow(cfg, **kw):
    f = cfg.flow
    for k, v in kw.items():
        setattr(f, k, v)
    # the day ends at the venue's close (close - 30 min, market.cpp:67-70) OPEN_ROWS rows after the first one
    f.t0_ms = int(cfg.close_ms) - 30 * 60000 - OPEN_ROWS * f.dt_ms
    assert f.t0_ms >= int(cfg.open_ms) + 30 * 60000


_THIN = dict(band_px0=10.0, band_ts=0.001, band_tick0=0, mid0_tick=0, tick_lo=-120, tick_hi=120, vol0=3, dt_ms=100,
             p_move_u12=4000, p_spread_u12=2048, spread_c1_u12=300, spread_c2_u12=800)
# (id, ticker, flow parameters, yaml overrides)
FLOWS = [
    ("euronext50", "X.PA", dict(band_px0=50.0, band_ts=0.005, band_tick0=0, mid0_tick=0, tick_lo=-70, tick_hi=70,
                                p_deep_u2=2), {}),
    ("nordic1000", "X.ST", dict(band_px0=1000.0, band_ts=0.5, band_tick0=0, mid0_tick=0, tick_lo=-50, tick_hi=50,
                                p_move_u12=2048), {"market.target_price.type": "book"}),
    ("irish_thin_deep0", "X.I", dict(_THIN, p_deep_u2=0), {"market.order_size": 2}),
    ("irish_thin_deep4", "X.I", dict(_THIN, p_deep_u2=4), {"market.order_size": 2, "learning.algorithm": "sarsa"}),
]
GEN_ENGINES = [("default", {}), ("rounds0", {"RLM_ROUNDS": "0"}), ("thread", {"RLM_ENV_VARIANT": "1"}),
               ("envw1", {"RLM_ENVW_WARPS": "1"})]
STREAM_ENGINES = [("stream-default", {}), ("stream-F", {"RLM_ENGINE": "F"}), ("stream-f", {"RLM_ENGINE": "f"}),
                  ("stream-p", {"RLM_ENGINE": "p"})]


def _config(ticker, flow, over, source, n_envs=B):
    y = config.example_dict(**{"learning.memory_size": 8192, "data.symbols": [ticker], **over})
    cfg = config.from_dict(y, n_envs=n_envs, source=source, flow_seed=5)
    _flow(cfg, **flow)
    cfg.record_envs, cfg.record_cap = n_envs, 2000
    return cfg


def _host_days(cfg, n_envs):
    """[(messages, N_TICKS)] per env: the host rendering of the handle's flow (rlm_flow_generate, no GPU)"""
    return [(rlm_lib.flow_generate(cfg.flow, cfg.env_index0 + b, 0, N_TICKS), N_TICKS) for b in range(n_envs)]


def _run(rlm, monkeypatch, env, cfg, per_env=None):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = rlm.BatchedMarket(cfg)
    if per_env is not None:
        m.load_ticks(_wide(per_env, N_TICKS), N_TICKS)
    m.run_ticks(N_TICKS)
    m.sync()
    for k in env:
        monkeypatch.delenv(k)
    return m


@pytest.mark.parametrize("fid,ticker,flow,over", FLOWS, ids=[f[0] for f in FLOWS])
def test_flow_parameters_on_every_engine(rlm, oracle, monkeypatch, fid, ticker, flow, over):
    cfg_g = _config(ticker, flow, over, abi.SOURCE_GENERATOR)
    cfg_s = _config(ticker, flow, over, abi.SOURCE_STREAM)
    days = _host_days(cfg_g, B)
    # the flow does reach both sides of its band boundary, in float
    bids = sorted({d[0][t].bid_px[0] for d in days[:4] for t in range(N_TICKS)})
    assert bids[0] < flow["band_px0"] < bids[-1], (fid, bids[0], bids[-1])
    ref = None
    for eid, env in GEN_ENGINES + STREAM_ENGINES:
        stream = eid.startswith("stream")
        m = _run(rlm, monkeypatch, env, cfg_s if stream else cfg_g, days if stream else None)
        st = m.stats(0, B)
        for b in range(B):  # every env ends its day at the venue's close
            assert st[b].terminal == 1, (fid, eid, b)
        for b in SAMPLED:
            _assert_port(m, oracle, m.cfg, b, days[b][0], N_TICKS)
        if eid == "default":
            ref = m
            continue
        if eid == "stream-default":
            _assert_same(ref, m, B)
            ref.close()
        m.close()


VENUE = G.venue_manifest()
VB = 4
# (id, environment, source, how the day is run: None = one long call, an int = calls of that many ticks, "split")
VENUE_KERNELS = [
    ("tape-s", {"RLM_ENGINE": "s"}, abi.SOURCE_TAPE, None),
    ("tape-rounds1", {"RLM_ROUNDS": "1"}, abi.SOURCE_TAPE, None),
    ("tape-thread", {"RLM_ENV_VARIANT": "1"}, abi.SOURCE_TAPE, None),
    ("tape-default", {}, abi.SOURCE_TAPE, 100),
    ("tape-split", {}, abi.SOURCE_TAPE, "split"),
    ("stream-F", {"RLM_ENGINE": "F"}, abi.SOURCE_STREAM, None),
    ("stream-f", {"RLM_ENGINE": "f"}, abi.SOURCE_STREAM, None),
    ("stream-p", {"RLM_ENGINE": "p"}, abi.SOURCE_STREAM, None),
]


def _venue_params():
    out = []
    for case in VENUE:
        for kid, env, source, how in VENUE_KERNELS:
            pid = "%s-%s" % (case["name"], kid)
            if kid == "stream-F" and case["algo"].endswith("r_learn"):
                out.append(pytest.param(case, env, source, how, id=pid + "-rerouted",
                                        marks=pytest.mark.skip(reason="the fused engine leaves R-learning to the tick-synchronous engine")))
            else:
                out.append(pytest.param(case, env, source, how, id=pid))
    return out


_DAYS = {}


def _venue_days(case):
    """[(messages, n)] of env b: the case's own day for b = 0, other days of the same writer for the others"""
    if case["name"] not in _DAYS:
        days = []
        with tempfile.TemporaryDirectory() as d:
            for b in range(VB):
                md, tas = G.venue_day(case, d, seed=None if b == 0 else case["day_seed"] + 7919 * b)
                msgs, n, ticks = rlm_lib.ingest_csv(md, tas)
                assert n == ticks
                days.append((msgs, n))
        _DAYS[case["name"]] = days
    return _DAYS[case["name"]]


_VPORT = {}


def _venue_port(oracle, case, cfg, b, msgs, n):
    key = (case["name"], b, cfg.source == abi.SOURCE_STREAM)
    if key not in _VPORT:
        _VPORT[key] = oracle.run_port(cfg, cfg.env_index0 + b, msgs, rec_cap=2000)
    return _VPORT[key]


def _run_split(m, cap):
    """Runner::RunEpisode per env until every env has reported its terminal step; one more round lets the envs that
    reported it last finish their episode (their next env_step ends it without a further step)."""
    m.env_step(None)
    m.agent_update()
    done = [False] * m.cfg.n_envs
    for _k in range(cap):
        _rew, term = m.env_step(m.act())
        m.agent_update()
        done = [d or t != 0 for d, t in zip(done, term)]
        if all(done):
            _rew, term = m.env_step(m.act())
            m.agent_update()
            assert list(term) == [1] * m.cfg.n_envs, list(term)
            return
    raise AssertionError("an env did not reach its close in %d steps" % cap)


@pytest.mark.parametrize("case,env,source,how", _venue_params())
def test_venue_day_on_every_tick_kernel(rlm, oracle, monkeypatch, case, env, source, how):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    days = _venue_days(case)
    if source == abi.SOURCE_STREAM:
        days = [days[0]] * VB  # tick-aligned: the case's day for every env, each env with its own seeds
    cfg = config.from_dict(case["yaml"], n_envs=VB, env_index0=case["env"], source=source)
    cfg.record_envs, cfg.record_cap = VB, 2000
    m = rlm.BatchedMarket(cfg)
    T = max(n for _a, n in days)
    if source == abi.SOURCE_TAPE:
        buf, offs = _library(days)
        m.load_days(buf, offs)  # env b on day b
    else:
        m.load_ticks(_wide(days, T), T)
    if how == "split":
        _run_split(m, case["n_records"] + 200)
    else:
        for _k in range(0, T, how or T):
            m.run_ticks(how or T)
    m.sync()
    st = m.stats()
    recs, _keep = m.records(0)
    gold = G.digests(case["name"])
    assert len(recs) == len(gold) == case["n_records"], (len(recs), len(gold))
    bad = [i for i in range(len(gold)) if G.record_digest(recs[i]) != gold[i]]
    if bad:  # name the fields through the oracle, which equals the reference on this day (test_venue_days.py)
        port = _venue_port(oracle, case, cfg, 0, *days[0])
        i = bad[0]
        raise AssertionError((case["name"], "reference record", i, G.describe_diff(
            port["records"][i], recs[i], abi.record_fields_equal(port["records"][i], recs[i]))))
    for b in range(VB):
        assert st[b].terminal == 1, b  # every env ends its day at its venue's close
        if b:
            _assert_port(m, oracle, cfg, b, *days[b])
        port = _venue_port(oracle, case, cfg, b, *days[b])
        assert bytes(m.theta(b)) == bytes((C.c_double * cfg.memory_size)(*port["theta"])), b
        assert bytes(st[b]) == bytes(port["stats"]), b
    m.close()


def _throw_config(source, env):
    # Copenhagen's bottom band (tick 0.0001) with the flow on a half-tick grid near zero: best bids of 0.00025 .. 0.00045
    # are 3 or 4 ticks, so `book` quoting with a bid level above that (action 6: 4, action 8: 5) asks ToPrice for a
    # negative tick count, and a bid level equal to it places an order at price 0, which the reference's Order rejects
    flow = dict(band_px0=0.0, band_ts=0.00005, band_tick0=0, mid0_tick=6, tick_lo=1, tick_hi=16)
    cfg = _config("X.CO", flow, {"market.target_price.type": "book", "policy.eps_init": 0.2}, source, 1)
    cfg.env_index0 = env
    return cfg


def _oracle_until_throw(oracle, capfd, cfg, msgs):
    """(the oracle's records before the step at which it raises, what it raised)"""
    L = oracle.lib()
    h = L.lobo_create(C.byref(cfg), cfg.env_index0)
    recs = (abi.StepRecord * N_TICKS)()
    used = C.c_int64(0)
    capfd.readouterr()
    rc = L.lobo_run(h, msgs, N_TICKS, -1, recs, N_TICKS, C.byref(used))
    s = L.lobo_total_steps(h)
    L.lobo_destroy(h)
    assert rc == -1, "the oracle did not raise"
    return [recs[i] for i in range(s)], capfd.readouterr().err


@pytest.mark.parametrize("eid,env", GEN_ENGINES + STREAM_ENGINES, ids=[e[0] for e in GEN_ENGINES + STREAM_ENGINES])
def test_negative_tick_count_is_an_invalid_argument(rlm, oracle, monkeypatch, capfd, eid, env):
    """One env per handle, so that the device's error flags belong to it: where the oracle first raises for a negative tick
    count, rlm_sync reports RLM_ERR_INVALID_ARGUMENT with "invalid price/ticks"; where it first raises for an order at
    price 0, the flags name a non-positive price.  Either way the records before that step equal the oracle's."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    stream = eid.startswith("stream")
    kinds = []
    for b in range(8):
        cfg = _throw_config(abi.SOURCE_STREAM if stream else abi.SOURCE_GENERATOR, b)
        days = _host_days(cfg, 1)
        want, raised = _oracle_until_throw(oracle, capfd, cfg, days[0][0])
        m = rlm.BatchedMarket(cfg)
        if stream:
            m.load_ticks(_wide(days, N_TICKS), N_TICKS)
        m.run_ticks(N_TICKS)
        with pytest.raises(rlm.RlmError) as ei:
            m.sync()
        if "Invalid number of ticks" in raised:
            kinds.append("ticks")
            assert ei.value.code == abi.RLM_ERR_INVALID_ARGUMENT and "invalid price/ticks" in str(ei.value), (b, str(ei.value))
        else:
            assert "Order price must be non-zero" in raised, raised
            kinds.append("price")
            assert "non-positive price" in str(ei.value), (b, str(ei.value))
        recs, _k = m.records(0)
        assert len(recs) >= len(want), (eid, b, len(recs), len(want))
        for i in range(len(want)):
            bad = abi.record_fields_equal(recs[i], want[i])
            assert not bad, (eid, b, i, G.describe_diff(recs[i], want[i], bad))
        m.close()
    assert kinds.count("ticks") >= 4 and "price" in kinds, kinds
