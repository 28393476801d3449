"""Whole trading days of other venues (tools/venue_csv.py): the best bid crosses one band boundary of the venue's tick
table many times and the day ends at the venue's own close.  The oracle, fed what rlm_ingest_csv makes of each CSV pair,
must give the reference's records on the same files (stored as digests by tools/make_golden.py VENUE_CASES) through the
terminal step; the reference is run again where oracle/_ref is built.  No GPU."""
import ctypes as C
import hashlib
import json
import os
import subprocess
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, config, lib

CASES = G.venue_manifest()
IDS = [c["name"] for c in CASES]


def _sha(path):
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def reference_on_day(oracle, case, y, md, tas, d):
    """(raw step records, summary without wall-clock fields) of oracle/_ref/ref_driver on a venue day, for the seed of the
    case's env"""
    y_run = json.loads(json.dumps(y))
    y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + case["env"]
    cfgp, dump = os.path.join(d, "cfg.yaml"), os.path.join(d, "steps.bin")
    oracle.write_ref_yaml(cfgp, y_run)
    out = subprocess.check_output([oracle.REF_DRIVER, "--config", cfgp, "--symbol", case["ticker"], "--md", md, "--tas", tas,
                                   "--dump", dump, "--steps", "-1"])
    summary = json.loads(out.decode().strip().splitlines()[-1])
    for k in ("seconds", "steps_per_s"):
        summary.pop(k, None)
    return open(dump, "rb").read(), summary


def _rows(path):
    return [r.split(",") for r in open(path).read().split("\n")[1:] if r]


def test_every_tick_table_and_the_irish_close():
    tables = [tuple(config.venue_table(c["ticker"])[0]) for c in CASES]
    assert len(set(tables)) == 6 and len(CASES) == 9  # LSE A and B, Euronext, Nordic, Milan, Vienna
    assert {config.venue_table(c["ticker"])[2] for c in CASES} >= {16 * 3600000 + 16 * 60000 + 40}  # the Irish close


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_venue_day(oracle, case):
    y = case["yaml"]
    cfg = config.from_dict(y)
    bands, _mo, _mc = config.venue_table(case["ticker"])
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day(case, d)
        # the writer still writes the files the reference ran on
        assert (_sha(md), _sha(tas)) == (case["md_sha256"], case["tas_sha256"])
        rows = _rows(md)
        msgs, n, ticks = lib.ingest_csv(md, tas)
        if oracle.have_ref():
            raw, _summary = reference_on_day(oracle, case, y, md, tas, d)
            live = (abi.StepRecord * (len(raw) // C.sizeof(abi.StepRecord))).from_buffer_copy(raw)
            assert [G.record_digest(r) for r in live] == G.digests(case["name"])
    # the best bid crosses the boundary at least 20 times; no price comes within half a tick of the top band
    b = case["boundary"]
    above = [float(r[12]) >= b for r in rows]
    assert sum(1 for i in range(1, len(above)) if above[i] != above[i - 1]) >= 20
    top_px, top_ts = bands[-1]
    assert max(float(r[6]) for r in rows) < top_px - top_ts / 2
    # one message per row: no row shares a timestamp, no row has more than four print prices
    assert n == ticks == len(rows), (n, ticks, len(rows))
    port = oracle.run_port(cfg, case["env"], msgs, rec_cap=2000)
    gold = G.digests(case["name"])
    assert port["steps"] == len(gold) == case["n_records"] > 500
    assert port["stats"].terminal == 1
    bad = [i for i in range(len(gold)) if G.record_digest(port["records"][i]) != gold[i]]
    assert not bad, (case["name"], "first differing record", bad[0])
