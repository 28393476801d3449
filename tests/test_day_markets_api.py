"""Day markets on the host side (rlm_set_day_markets, no GPU): the entry point, the rlm_market layout, the ticker ->
market mapping, the library's market index, and the fixtures of tests/test_gpu_day_markets.py against the CPU oracle
run under each day's market."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, config, ingest
from rl_markets_b200 import lib as rlm_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _day_markets():
    with open(os.path.join(G.GOLD, "day_markets.json")) as f:
        return json.load(f)


def test_entry_point_is_exported_and_bound():
    assert "rlm_set_day_markets" in rlm_lib.EXPORTS
    L = rlm_lib.load()
    assert L.rlm_set_day_markets.argtypes[1] is C.POINTER(abi.Market)
    m = (abi.Market * 1)(config.market("AAL.L"))
    dm = (C.c_int32 * 1)(0)
    assert L.rlm_set_day_markets(None, m, 1, dm, 1) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_set_day_markets(None, None, 0, None, 0) == abi.RLM_ERR_INVALID_ARGUMENT
    assert "bad arguments" in L.rlm_last_error().decode()


def test_market_layout_matches_the_header():
    src = r'''
#include <stddef.h>
#include <stdio.h>
#include "rlm.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu %zu\n", sizeof(rlm_market), offsetof(rlm_market, n_bands), offsetof(rlm_market, pad),
         offsetof(rlm_market, band_px), offsetof(rlm_market, band_ts), offsetof(rlm_market, open_ms), offsetof(rlm_market, close_ms));
  return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        c, exe = os.path.join(d, "layout.c"), os.path.join(d, "layout")
        with open(c, "w") as f:
            f.write(src)
        subprocess.check_call(["cc", "-I" + os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(x) for x in subprocess.check_output([exe]).split()]
    M = abi.Market
    want = [C.sizeof(M)] + [getattr(M, k).offset for k in ("n_bands", "pad", "band_px", "band_ts", "open_ms", "close_ms")]
    assert got == want


@pytest.mark.parametrize("ticker", ["X." + v for v in ("AS", "BR", "CO", "DE", "HE", "I", "MC", "MI", "OL", "PA", "S", "VX", "ST", "VI")]
                         + ["AAL.L", "BATS.L", "GSK.L", "VOD.L", "HSBA.L", "BAES.L", "UU.L", "LGEN.L", "LSE.L", "NXT.L"])
def test_market_agrees_with_venue_table(ticker):
    bands, mo, mc = config.venue_table(ticker)
    m = config.market(ticker)
    assert m.n_bands == len(bands) and (m.open_ms, m.close_ms) == (mo, mc)
    assert [(m.band_px[i], m.band_ts[i]) for i in range(m.n_bands)] == list(bands)
    # the same fields as the config's venue block
    cfg = config.from_dict(config.example_dict(**{"learning.memory_size": 4096}), ticker=ticker)
    assert bytes(config.config_market(cfg)) == bytes(m)


@pytest.mark.parametrize("ticker,msg", [("X.ZZ", "Unknown exchange venue"), ("ABC.L", "Unknown symbol")])
def test_market_raises_on_unknown_tickers(ticker, msg):
    with pytest.raises(ValueError, match=msg):
        config.market(ticker)


def test_day_markets_deduplicate_in_first_seen_order():
    samples = [("BAES.L", "a", "b"), ("AAL.L", "a", "b"), ("UU.L", "a", "b"), ("X.PA", "a", "b"), ("VOD.L", "a", "b"),
               ("X.AS", "a", "b"), ("X.DE", "a", "b"), ("BAES.L", "a", "b")]
    markets, day_market = ingest.day_markets(samples)
    # LSE B, LSE A, Euronext with Paris hours (Xetra's are the same), Euronext with Amsterdam's
    assert day_market == [0, 1, 0, 2, 1, 3, 2, 0]
    assert [bytes(m) for m in markets] == [bytes(config.market(t)) for t in ("BAES.L", "AAL.L", "X.PA", "X.AS")]
    assert not config.same_market(config.market("AAL.L"), config.market("BAES.L"))


def test_fixtures_equal_the_oracle_under_each_days_market(oracle):
    """The reference's digests of the mixed library (tools/make_golden.py --day-markets) are the oracle's records when the
    oracle's config carries the day's ticker: the fixtures describe one yaml whose days differ only in their market."""
    dm = _day_markets()
    venue = {c["name"]: c for c in G.venue_manifest()}
    assert len(dm["days"]) == 9
    with tempfile.TemporaryDirectory() as d:
        for day in dm["days"]:
            case = venue[day["venue_case"]]
            md, tas = G.venue_day(case, d)
            msgs, n, _t = rlm_lib.ingest_csv(md, tas)
            cfg = config.from_dict(dm["yaml"], env_index0=dm["env0"], source=abi.SOURCE_TAPE, ticker=day["ticker"])
            port = oracle.run_port(cfg, day["env"], msgs, rec_cap=2000)
            gold = G.digests(day["name"])
            assert port["steps"] == len(gold) == day["n_records"]
            assert [G.record_digest(r) for r in port["records"]] == gold, day["name"]


def test_oracle_market_replacement_is_the_tickers_market(oracle):
    """tests/oracle_market.cpp: an oracle env created under AAL.L's market and given BAES.L's (LoadData's market
    replacement) replays the BAES.L day as the reference does under --symbol BAES.L"""
    import oracle_market as OM
    dm = _day_markets()
    day = next(x for x in dm["days"] if x["ticker"] == "BAES.L")
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day({c["name"]: c for c in G.venue_manifest()}[day["venue_case"]], d)
        msgs, n, _t = rlm_lib.ingest_csv(md, tas)
    cfg = config.from_dict(dm["yaml"], env_index0=dm["env0"], source=abi.SOURCE_TAPE, ticker="AAL.L")
    L = oracle.lib()
    h = L.lobo_create(C.byref(cfg), day["env"])
    OM.set_market(h, config.market("BAES.L"))
    recs = (abi.StepRecord * 2000)()
    used = C.c_int64()
    k = L.lobo_run(h, msgs, n, -1, recs, 2000, C.byref(used))
    L.lobo_destroy(h)
    assert [G.record_digest(recs[i]) for i in range(k)] == G.digests(day["name"])
