"""Tape days under their tickers' markets (rlm_set_day_markets), bitwise, on every tick kernel that reads the tape.

The nine venue days (tools/venue_csv.py, one per tick table, the Irish 16:16 plus 40 ms close among them) form one
library under one yaml whose own market is AAL.L's (LSE group A).  Env b < 9 replays day b with seed
random_seed + env_index0 + b and must give the reference's records (tests/golden/day_markets.json, ref_driver --symbol
<the day's ticker>); envs 9..17 replay the days in the opposite order, so a market follows its day and not the env index,
and must give the records, theta and statistics of the CPU oracle whose config carries the day's ticker.  Every env ends
its day at its own venue's close."""
import ctypes as C
import json
import os
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, config, ingest
from rl_markets_b200 import lib as rlm_lib
from test_gpu_market import _run_split
from test_gpu_tape import _library

pytestmark = pytest.mark.gpu

with open(os.path.join(G.GOLD, "day_markets.json")) as _f:
    DM = json.load(_f)
ND = len(DM["days"])
B = 2 * ND
DAY = list(range(ND)) + list(reversed(range(ND)))  # the day of env b
KERNELS = [("s", {"RLM_ENGINE": "s"}, None), ("rounds1", {"RLM_ROUNDS": "1"}, None), ("thread", {"RLM_ENV_VARIANT": "1"}, None),
           ("default-100", {}, 100), ("split", {}, "split")]
_VENUE = {c["name"]: c for c in G.venue_manifest()}
_DAYS = []


def _days():
    """[(messages, n)] of the nine days, in day_markets.json order"""
    if not _DAYS:
        with tempfile.TemporaryDirectory() as d:
            for day in DM["days"]:
                md, tas = G.venue_day(_VENUE[day["venue_case"]], d)
                msgs, n, _t = rlm_lib.ingest_csv(md, tas)
                _DAYS.append((msgs, n))
    return _DAYS


def _cfg(ticker=None, n_envs=B, shared=False):
    cfg = config.from_dict(DM["yaml"], n_envs=n_envs, env_index0=DM["env0"], source=abi.SOURCE_TAPE, ticker=ticker,
                           shared_policy=shared)
    cfg.record_envs, cfg.record_cap = n_envs, 2000
    return cfg


def _markets():
    markets, day_market = ingest.day_markets([(day["ticker"], None, None) for day in DM["days"]])
    assert len(markets) == ND  # six tick tables, and the days that share one differ in their hours
    return markets, day_market


def _handle(rlm, day_markets=True, same=False):
    m = rlm.BatchedMarket(_cfg())
    buf, offs = _library(_days())
    m.load_days(buf, offs)
    m.assign_days(DAY[ND:], env0=ND)
    if day_markets:
        markets, day_market = _markets()
        if same:  # every day under a copy of the config's market
            markets, day_market = [config.config_market(m.cfg)], [0] * ND
        m.set_day_markets(markets, day_market)
    return m


def _run(m, how):
    T = max(n for _a, n in _days())
    if how == "split":
        _run_split(m, max(d["n_records"] for d in DM["days"]) + 200)
    else:
        for _k in range(0, T, how or T):
            m.run_ticks(how or T)
    m.sync()


_PORT = {}


def _port(oracle, b):
    day = DM["days"][DAY[b]]
    key = (b, DAY[b])
    if key not in _PORT:
        msgs, _n = _days()[DAY[b]]
        _PORT[key] = oracle.run_port(_cfg(ticker=day["ticker"], n_envs=1), DM["env0"] + b, msgs, rec_cap=2000)
    return _PORT[key]


def _assert_oracle(m, oracle, b, st):
    port = _port(oracle, b)
    recs, _k = m.records(b)
    assert len(recs) == port["steps"], (b, len(recs), port["steps"])
    for i in range(port["steps"]):
        bad = abi.record_fields_equal(recs[i], port["records"][i])
        assert not bad, (b, i, G.describe_diff(recs[i], port["records"][i], bad))
    assert bytes(m.theta(b)) == bytes((C.c_double * m.cfg.memory_size)(*port["theta"])), b
    assert bytes(st[b]) == bytes(port["stats"]), b


def _assert_reference(m, b):
    day = DM["days"][DAY[b]]
    assert day["env"] == DM["env0"] + b
    recs, _k = m.records(b)
    gold = G.digests(day["name"])
    assert len(recs) == len(gold) == day["n_records"], (b, len(recs), len(gold))
    bad = [i for i in range(len(gold)) if G.record_digest(recs[i]) != gold[i]]
    assert not bad, (day["name"], "first differing record", bad[0])


@pytest.mark.parametrize("kid,env,how", KERNELS, ids=[k[0] for k in KERNELS])
def test_mixed_library_against_reference_and_oracle(rlm, oracle, monkeypatch, kid, env, how):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = _handle(rlm)
    _run(m, how)
    st = m.stats()
    for b in range(B):
        assert st[b].terminal == 1, b  # at its own venue's close
        if b < ND:
            _assert_reference(m, b)
        _assert_oracle(m, oracle, b, st)
    m.close()


@pytest.mark.parametrize("kid,env,how", KERNELS[:3], ids=[k[0] for k in KERNELS[:3]])
def test_day_markets_equal_to_the_config_change_nothing(rlm, monkeypatch, kid, env, how):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ma, mb = _handle(rlm, day_markets=False), _handle(rlm, same=True)
    _run(ma, how)
    _run(mb, how)
    for b in range(B):
        ra, _k = ma.records(b)
        rb, _k = mb.records(b)
        assert len(ra) == len(rb) > 20
        assert all(bytes(x) == bytes(y) for x, y in zip(ra, rb)), b
        assert bytes(ma.theta(b)) == bytes(mb.theta(b)), b
    assert bytes(ma.stats()) == bytes(mb.stats())
    ma.close()
    mb.close()


def test_shared_policy_across_markets_per_env_close(rlm):
    """One theta across the nine markets: every env ends at its own venue's close, with exactly one terminal record."""
    cfg = _cfg(shared=True)
    m = rlm.BatchedMarket(cfg)
    buf, offs = _library(_days())
    m.load_days(buf, offs)
    m.assign_days(DAY[ND:], env0=ND)
    m.set_day_markets(*_markets())
    _run(m, None)
    st = m.stats()
    for b in range(B):
        assert st[b].terminal == 1, b
        recs, _k = m.records(b)
        assert recs[-1].terminal == 1 and sum(r.terminal for r in recs) == 1, b
        close = config.market(DM["days"][DAY[b]]["ticker"]).close_ms
        assert close - 30 * 60000 <= recs[-1].time_ms < close - 30 * 60000 + 60000, b
    m.close()


def test_errors_change_nothing_and_load_days_drops_the_markets(rlm):
    markets, day_market = _markets()
    mk = (abi.Market * len(markets))(*markets)
    L = rlm.load()

    def call(m, mk_=mk, n=len(markets), dm=day_market, nd=ND):
        arr = (C.c_int32 * max(len(dm), 1))(*dm)
        return L.rlm_set_day_markets(m.h, mk_, n, arr, nd)

    gen = rlm.BatchedMarket(config.from_dict(DM["yaml"], n_envs=2))
    assert call(gen) == abi.RLM_ERR_INVALID_ARGUMENT  # not a tape handle
    gen.close()
    empty = rlm.BatchedMarket(_cfg())
    assert call(empty) == abi.RLM_ERR_INVALID_ARGUMENT  # no library
    empty.close()
    m = _handle(rlm, day_markets=False)
    assert call(m, nd=ND - 1, dm=day_market[:-1]) == abi.RLM_ERR_INVALID_ARGUMENT  # wrong n_days
    assert call(m, dm=day_market[:-1] + [len(markets)]) == abi.RLM_ERR_INVALID_ARGUMENT  # index out of range
    assert call(m, dm=[-1] + day_market[1:]) == abi.RLM_ERR_INVALID_ARGUMENT
    bad = (abi.Market * len(markets))(*markets)
    bad[2].band_px[1] = bad[2].band_px[0]  # bands must ascend
    assert call(m, mk_=bad) == abi.RLM_ERR_INVALID_ARGUMENT
    bad = (abi.Market * len(markets))(*markets)
    bad[1].band_ts[0] = 0.0
    assert call(m, mk_=bad) == abi.RLM_ERR_INVALID_ARGUMENT
    bad = (abi.Market * len(markets))(*markets)
    bad[0].n_bands = 33
    assert call(m, mk_=bad) == abi.RLM_ERR_INVALID_ARGUMENT
    # the failed calls left the handle as it was: it equals a handle that never saw them
    ref = _handle(rlm, day_markets=False)
    _run(m, None)
    _run(ref, None)
    for b in range(B):
        ra, _k = m.records(b)
        rb, _k = ref.records(b)
        assert [bytes(x) for x in ra] == [bytes(y) for y in rb], b
    ref.close()
    m.close()
    # rlm_load_days after rlm_set_day_markets: every day under the config's market again
    m = _handle(rlm)
    buf, offs = _library(_days())
    m.load_days(buf, offs)
    m.assign_days(DAY[ND:], env0=ND)
    ref = _handle(rlm, day_markets=False)
    _run(m, None)
    _run(ref, None)
    for b in range(B):
        ra, _k = m.records(b)
        rb, _k = ref.records(b)
        assert [bytes(x) for x in ra] == [bytes(y) for y in rb], b
        assert bytes(m.theta(b)) == bytes(ref.theta(b)), b
    assert bytes(m.stats()) == bytes(ref.stats())
    m.close()
    ref.close()


def test_file_sample_end_to_end(rlm):
    """AAL.L and BAES.L days in an md_dir / tas_dir tree -> ingest.file_sample -> load_day_library: one handle, two
    markets (LSE A and B), each env the reference's records for its day."""
    names = {"AAL.L": "venue_aal_l", "BAES.L": "venue_baes_l"}
    with tempfile.TemporaryDirectory() as d:
        md_dir, tas_dir = os.path.join(d, "mdx"), os.path.join(d, "tsx")
        for sym, case in names.items():
            os.makedirs(os.path.join(md_dir, sym))
            os.makedirs(os.path.join(tas_dir, sym))
            md, tas = G.venue_day(_VENUE[case], d)
            f = os.path.join(md_dir, sym, "v_md_1.csv")
            os.rename(md, f)
            loc = f.find("md_")
            tf = tas_dir + f[len(md_dir):]
            os.rename(tas, tf[:loc + 1] + "tas" + tf[loc + 3:])
        samples = ingest.file_sample(md_dir, tas_dir, ["AAL.L", "BAES.L"])
        assert [s for s, _m, _t in samples] == ["AAL.L", "BAES.L"]
        m = rlm.BatchedMarket(_cfg(n_envs=2))
        assert m.load_day_library(samples) == 2
    _run(m, None)
    for b, sym in enumerate(["AAL.L", "BAES.L"]):
        day = next(x for x in DM["days"] if x["ticker"] == sym)
        assert day["env"] == DM["env0"] + b
        recs, _k = m.records(b)
        gold = G.digests(day["name"])
        assert len(recs) == len(gold) and [G.record_digest(r) for r in recs] == gold, sym
    m.close()
