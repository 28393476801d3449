#!/usr/bin/env python3
"""Generate tests/golden/* from the UNMODIFIED reference compiled into oracle/_ref (run where
the reference sources are present, see oracle/Makefile; the fixtures are committed so that
machines without the reference can check against them).
  --reference-checks   only the fixtures of reference_checks() below
  --day-markets        only tests/golden/day_markets.json and its digests (day_market_fixtures())
  --eval-days          only tests/golden/eval_days.json and its digests (eval_days_fixtures())
  --q-values           only tests/golden/q_values.json (tools/ref_q_values.cpp on the reference: Agent::getQ / getQb)
  --training-logs      only tests/golden/training_logs.json and tl_<case>_{model,training}_log.csv (tools/ref_train_logs.cpp:
                       the reference trained with logging.log_learning on)

  tests/golden/units.json          reference unit-level vectors (oracle/_ref/ref_units)
  tests/golden/steps_<name>.bin    first N rlm_step_record of a reference run (oracle/_ref/ref_driver)
  tests/golden/bt_*_{profit_log,test_stats}.csv   the reference's own evaluation logs for the backtest cases
  tests/golden/digests_venue_*.bin per-record digests of the reference on whole venue days (tools/venue_csv.py)
  tests/golden/manifest.json       the configs that produced them
"""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle_lib as ol  # noqa: E402
from rl_markets_b200 import abi, config  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")
N_RECORDS = 400
CASES = [
    dict(name="q_learn_m65536", algo="q_learn", M=65536, flow_seed=7, env=0, ticks=2500, over={}),
    dict(name="sarsa_m16384", algo="sarsa", M=16384, flow_seed=7, env=1, ticks=2500, over={}),
    dict(name="double_q_m65536", algo="double_q_learn", M=65536, flow_seed=9, env=2, ticks=2500, over={}),
    dict(name="q_learn_m5003_greedy", algo="q_learn", M=5003, flow_seed=11, env=3, ticks=2500,
         over={"policy.eps_init": 0.05}),
    dict(name="q_learn_m4096_random_init", algo="q_learn", M=4096, flow_seed=13, env=5, ticks=2500,
         over={"learning.random_init": True, "debug.random_seed": 77}),
    # SURVEY 8f rank 2: R-learning agents (agent.cpp:357-467) and the Boltzmann policy (policy.cpp:85-122)
    dict(name="r_learn_m16384", algo="r_learn", M=16384, flow_seed=15, env=6, ticks=2500, over={"policy.eps_init": 0.3}),
    dict(name="online_r_learn_m16384", algo="online_r_learn", M=16384, flow_seed=15, env=7, ticks=2500,
         over={"policy.eps_init": 0.3}),
    dict(name="double_r_learn_m8209", algo="double_r_learn", M=8209, flow_seed=17, env=8, ticks=2500,
         over={"policy.eps_init": 0.3, "learning.alpha_start": 0.01}),
    dict(name="sarsa_boltzmann_m8192", algo="sarsa", M=8192, flow_seed=19, env=9, ticks=2500,
         over={"policy.type": "boltzmann", "policy.tau_init": 0.05, "policy.tau_floor": 0.01, "policy.tau_T": 10}),
]


# SURVEY 8f rank 2, the rest: every reward measure (base.cpp:166-237), all 13 state variables (intraday.cpp:315-409),
# the Random policy (policy.cpp:27-30), and the other two target-price / quote rules (base.cpp:101-112, intraday.cpp:64-82).
# 150 records each keep the fixtures small.
_ALL_VARS = ["pos", "spd", "mpm", "imb", "svl", "vol", "rsi", "vwap", "a_dist", "a_queue", "b_dist", "b_queue", "last_action"]
F2_CASES = [
    dict(name="rew_none", algo="q_learn", M=8192, flow_seed=31, env=10, ticks=1200, over={"reward.measure": "none"}),
    dict(name="rew_pnl", algo="q_learn", M=8192, flow_seed=31, env=11, ticks=1200, over={"reward.measure": "pnl"}),
    dict(name="rew_spread", algo="sarsa", M=8192, flow_seed=31, env=12, ticks=1200, over={"reward.measure": "spread"}),
    dict(name="rew_normed", algo="q_learn", M=8192, flow_seed=31, env=13, ticks=1200,
         over={"reward.measure": "normed", "reward.pnl_lookback": 12}),
    dict(name="rew_lovol", algo="q_learn", M=8192, flow_seed=31, env=14, ticks=1200, over={"reward.measure": "lovol"}),
    dict(name="rew_mm_linear", algo="q_learn", M=8192, flow_seed=31, env=15, ticks=1200,
         over={"reward.measure": "mm_linear", "reward.pos_weight": 0.5, "reward.pnl_weight": 0.75}),
    dict(name="rew_mm_exp", algo="q_learn", M=8192, flow_seed=31, env=16, ticks=1200,
         over={"reward.measure": "mm_exp", "reward.pos_weight": 0.02, "reward.pnl_weight": 1.0}),
    dict(name="rew_mm_div", algo="double_q_learn", M=8192, flow_seed=31, env=17, ticks=1200, over={"reward.measure": "mm_div"}),
    dict(name="vars13", algo="q_learn", M=16384, flow_seed=33, env=18, ticks=1200,
         over={"state.variables": _ALL_VARS, "state.lookback.rsi": 10, "state.lookback.vwap": 20}),
    dict(name="vars13_sarsa_defaults", algo="sarsa", M=16384, flow_seed=33, env=19, ticks=1200,
         over={"state.variables": list(reversed(_ALL_VARS))}),  # rsi / vwap lookbacks 0 -> windows of 1
    dict(name="policy_random", algo="q_learn", M=8192, flow_seed=35, env=20, ticks=1200, over={"policy.type": "random"}),
    dict(name="policy_greedy", algo="sarsa", M=8192, flow_seed=35, env=21, ticks=1200, over={"policy.type": "greedy"}),
    dict(name="tp_microprice", algo="q_learn", M=8192, flow_seed=37, env=22, ticks=1200,
         over={"market.target_price.type": "microprice", "market.target_price.lookback": 5}),  # -> tp::MidPrice (A1)
    dict(name="tp_book", algo="q_learn", M=8192, flow_seed=37, env=23, ticks=1200, over={"market.target_price.type": "book"}),
]
N_F2_RECORDS = 150

# The learner's configuration space beyond the defaults (9 actions, 8 or 13 variables, gamma*lambda = 0.829, tables of
# 4096..65536): action counts whose Q sums and action hash terms sit elsewhere, feature groups of other sizes, trace lists
# far longer than one batch of the update table (derived cap 13 408) and none at all (lambda = 0), staged tables that are
# not powers of two, the first size past the staging limit, and tables smaller than a step's 32 tiles per group.
# Which learner kernel a case reaches (rlm_create): staged for even M <= 8192, the one-warp learner otherwise, the
# three-warp kernel for the R-learning agents.  150 records each, like F2_CASES.
_VARS11 = ["pos", "spd", "mpm", "imb", "svl", "vol", "rsi", "vwap", "a_dist", "b_dist", "last_action"]
_LONG = {"learning.gamma": 0.999, "learning.lambda": 0.99}
CONFIG_CASES = [
    dict(name="act1_q", algo="q_learn", M=8192, flow_seed=61, env=30, ticks=1200, over={"learning.n_actions": 1}),
    dict(name="act2_random", algo="q_learn", M=16384, flow_seed=61, env=31, ticks=1200,
         over={"learning.n_actions": 2, "policy.type": "random"}),
    dict(name="act5_double_q", algo="double_q_learn", M=65536, flow_seed=63, env=32, ticks=1200, over={"learning.n_actions": 5}),
    dict(name="act7_r_learn", algo="r_learn", M=16384, flow_seed=63, env=33, ticks=1200,
         over={"learning.n_actions": 7, "policy.eps_init": 0.3}),
    dict(name="vars4_sarsa", algo="sarsa", M=16384, flow_seed=65, env=34, ticks=1200,
         over={"state.variables": ["pos", "spd", "mpm", "imb"]}),
    dict(name="vars11_q", algo="q_learn", M=8192, flow_seed=65, env=35, ticks=1200,
         over={"state.variables": _VARS11, "state.lookback.rsi": 6, "state.lookback.vwap": 9}),
    dict(name="long_traces_sarsa", algo="sarsa", M=65536, flow_seed=67, env=36, ticks=1200, over=dict(_LONG)),
    dict(name="long_traces_q", algo="q_learn", M=16384, flow_seed=67, env=37, ticks=1200, over=dict(_LONG, **{"policy.eps_init": 0.05})),
    dict(name="lambda0_q", algo="q_learn", M=8192, flow_seed=69, env=38, ticks=1200, over={"learning.lambda": 0.0}),
    dict(name="m6000_staged", algo="q_learn", M=6000, flow_seed=69, env=39, ticks=1200, over={}),
    dict(name="m8190_staged_sarsa", algo="sarsa", M=8190, flow_seed=71, env=40, ticks=1200, over={}),
    dict(name="m8194_gather", algo="q_learn", M=8194, flow_seed=71, env=41, ticks=1200, over={}),
    dict(name="m2_staged", algo="q_learn", M=2, flow_seed=73, env=42, ticks=1200, over={}),
    dict(name="m1_gather", algo="sarsa", M=1, flow_seed=73, env=43, ticks=1200, over={}),
    dict(name="m3_gather", algo="q_learn", M=3, flow_seed=75, env=44, ticks=1200, over={}),
    dict(name="m97_gather", algo="sarsa", M=97, flow_seed=75, env=45, ticks=1200, over={}),
]

# N training episodes on ONE Intraday and ONE Learner-equivalent (main.cpp:45-60, serial.cpp:72-95): the day ends
# `open_ticks` rows after the first one, HandleTerminal(episode), LoadData of the same day again, Initialise.
EPISODE_CASES = [
    dict(name="ep3_q_learn_m8192", algo="q_learn", M=8192, flow_seed=41, env=24, ticks=700, open_ticks=500, episodes=3,
         over={"learning.omega": 0.9, "learning.alpha_start": 0.01, "policy.eps_T": 3}),
    dict(name="ep3_double_q_m8192", algo="double_q_learn", M=8192, flow_seed=43, env=25, ticks=700, open_ticks=500, episodes=3,
         over={"learning.omega": 0.8, "learning.alpha_start": 0.01, "policy.eps_T": 2}),
    dict(name="ep2_sarsa_boltzmann_m8192", algo="sarsa", M=8192, flow_seed=45, env=26, ticks=700, open_ticks=500, episodes=2,
         over={"policy.type": "boltzmann", "policy.tau_init": 0.05, "policy.tau_floor": 0.01, "policy.tau_T": 2}),
]

# Real-data shapes (SURVEY 8f rank 1): a CSV pair with depth rows that share a timestamp (A21), a crossed book (the reference
# swallows the next row into the same tick), rows with a zero price (dropped) and bursts of 5..9 distinct print prices;
# the reference runs on the files, rlm_ingest_csv + the packed stream have to reproduce it.
INGEST_CASES = [
    dict(name="ingest_messy_q_learn", algo="q_learn", M=8192, flow_seed=51, env=27, ticks=1300, messy_seed=3,
         features=["dup", "zero", "cross", "burst"], over={}),
    dict(name="ingest_messy_sarsa", algo="sarsa", M=8192, flow_seed=53, env=28, ticks=1300, messy_seed=5,
         features=["dup", "zero", "cross", "burst"], over={}),
]

# train on one (short) synthetic day until the close, then main.cpp's evaluation phase (GoGreedy, a NEW Intraday,
# Backtester::RunEpisode) on another one: steps_<name>.bin = training records, steps_<name>_test.bin = evaluation
BACKTEST_CASES = [
    dict(name="bt_q_learn_m8192", algo="q_learn", M=8192, flow_seed=21, env=4, ticks=1200, train_open_ticks=900,
         test=dict(flow_seed=22, env=4, ticks=1000, open_ticks=700), over={"policy.eps_T": 3}),
    dict(name="bt_double_q_m8192", algo="double_q_learn", M=8192, flow_seed=23, env=5, ticks=1200, train_open_ticks=900,
         test=dict(flow_seed=24, env=5, ticks=1000, open_ticks=700), over={"learning.alpha_start": 0.01}),
]


# Whole trading days of other venues (tools/venue_csv.py): the best bid crosses one band boundary of the venue's tick
# table many times, and the day ends at the venue's own close.  One case per distinct tick table, each with its own agent
# and quote rule; target-price quoting puts quotes inside the window below a boundary where ToTicks subtracts a tick.
# X.S is a thin book (1..20 lots per level, order size 10, positions within +-20): market orders walk past the depth the
# book shows, cancellations meet volume queued behind an order, and an order's level vanishes.  The CSV pairs are not
# committed: the tests write them again and check them against the sha256 stored here.
VENUE_CASES = [
    dict(name="venue_aal_l", ticker="AAL.L", boundary=5000.0, day_seed=101, algo="q_learn", M=8192, env=50,
         over={"market.target_price.type": "book", "state.variables": _ALL_VARS, "state.lookback.rsi": 10,
               "state.lookback.vwap": 20}),
    dict(name="venue_baes_l", ticker="BAES.L", boundary=500.0, day_seed=102, algo="sarsa", M=8192, env=51, over={}),
    dict(name="venue_x_pa", ticker="X.PA", boundary=50.0, day_seed=103, algo="double_q_learn", M=8192, env=52,
         over={"market.target_price.type": "microprice", "market.target_price.lookback": 5}),
    dict(name="venue_x_st", ticker="X.ST", boundary=5000.0, day_seed=104, algo="r_learn", M=8192, env=53,
         over={"policy.eps_init": 0.3}),
    dict(name="venue_x_mi", ticker="X.MI", boundary=2.0, day_seed=105, algo="q_learn", M=5003, env=54,
         over={"policy.type": "boltzmann", "policy.tau_init": 0.05, "policy.tau_floor": 0.01, "policy.tau_T": 10}),
    dict(name="venue_x_vi", ticker="X.VI", boundary=10.0, day_seed=106, algo="sarsa", M=4096, env=55,
         over={"market.target_price.type": "vwap", "reward.measure": "mm_linear", "reward.pos_weight": 0.5}),
    dict(name="venue_x_i", ticker="X.I", boundary=10.0, day_seed=107, algo="double_q_learn", M=8192, env=56, over={}),
    dict(name="venue_x_co", ticker="X.CO", boundary=0.5, day_seed=108, algo="q_learn", M=8192, env=57,
         over={"reward.measure": "pnl"}),
    dict(name="venue_x_s", ticker="X.S", boundary=1000.0, day_seed=109, algo="q_learn", M=4096, env=58, thin=True,
         over={"market.order_size": 10, "market.pos_ub": 20, "market.pos_lb": -20, "policy.eps_init": 0.5}),
]


def venue_yaml(c):
    return config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], "data.symbols": [c["ticker"]],
                                  **c["over"]})


def file_sha256(path):
    import hashlib
    return hashlib.sha256(open(path, "rb").read()).hexdigest()


def day_t0(cfg, open_ticks, dt_ms=250):
    """t0 such that the market closes (venue close - 30 min, market.cpp:67-70) `open_ticks` rows after the first one."""
    return int(cfg.close_ms) - 30 * 60000 - open_ticks * dt_ms


def main():
    os.makedirs(GOLD, exist_ok=True)
    units = subprocess.check_output([ol.REF_UNITS]).decode()
    json.loads(units)
    with open(os.path.join(GOLD, "units.json"), "w") as f:
        f.write(units)
    manifest = []
    for c in CASES:
        y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
        # the reference seeds every generator with debug.random_seed (main.cpp:84-88); env b of a batch uses
        # random_seed + b, so the single-env reference run for env b gets that seed
        seed = y["debug"]["random_seed"] + c["env"]
        y_run = json.loads(json.dumps(y))
        y_run["debug"]["random_seed"] = seed
        ref = ol.run_ref(y_run, c["flow_seed"], c["env"], c["ticks"])
        recs = ref["records"][:N_RECORDS]
        with open(os.path.join(GOLD, "steps_%s.bin" % c["name"]), "wb") as f:
            for r in recs:
                f.write(bytes(r))
        manifest.append(dict(c, yaml=y, n_records=len(recs), summary=ref["summary"]))
        print(c["name"], len(recs), "records;", ref["summary"]["steps"], "reference steps")
    for c in F2_CASES:
        manifest.append(short_case(c))
    for c in EPISODE_CASES:
        y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
        y_run = json.loads(json.dumps(y))
        y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + c["env"]
        cfg = config.from_dict(y)
        t0 = day_t0(cfg, c["open_ticks"])
        ref = ol.run_ref(y_run, c["flow_seed"], c["env"], c["ticks"], t0_ms=t0, episodes=c["episodes"])
        assert ref["summary"]["terminal"] == 1
        with open(os.path.join(GOLD, "steps_%s.bin" % c["name"]), "wb") as f:
            for r in ref["records"]:
                f.write(bytes(r))
        manifest.append(dict(c, yaml=y, multi_episode=True, t0_ms=t0, n_records=len(ref["records"]), summary=ref["summary"]))
        print(c["name"], len(ref["records"]), "records over", c["episodes"], "episodes")
    import tempfile
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import messy_csv
    for c in INGEST_CASES:
        y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
        y_run = json.loads(json.dumps(y))
        y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + c["env"]
        md_out, tas_out = os.path.join(GOLD, c["name"] + "_md.csv"), os.path.join(GOLD, c["name"] + "_tas.csv")
        with tempfile.TemporaryDirectory() as d:
            md, tas = os.path.join(d, "c_md_1.csv"), os.path.join(d, "c_tas_1.csv")
            subprocess.check_call([ol.FLOW_CSV, "--seed", str(c["flow_seed"]), "--env", str(c["env"]), "--ticks", str(c["ticks"]),
                                   "--md", md, "--tas", tas])
            messy_csv.make_messy(md, tas, md_out, tas_out, seed=c["messy_seed"], features=c["features"])
            cfgp, dump = os.path.join(d, "cfg.yaml"), os.path.join(d, "steps.bin")
            ol.write_ref_yaml(cfgp, y_run)
            out = subprocess.check_output([ol.REF_DRIVER, "--config", cfgp, "--symbol", "AAL.L", "--md", md_out, "--tas", tas_out,
                                           "--dump", dump, "--steps", "-1"])
            summary = json.loads(out.decode().strip().splitlines()[-1])
            raw = open(dump, "rb").read()
        with open(os.path.join(GOLD, "steps_%s.bin" % c["name"]), "wb") as f:
            f.write(raw)
        n = len(raw) // C.sizeof(abi.StepRecord)
        manifest.append(dict(c, yaml=y, ingest=True, n_records=n, summary=summary))
        print(c["name"], n, "records from the reference on the messy CSV pair")
    for c in BACKTEST_CASES:
        y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
        seed = y["debug"]["random_seed"] + c["env"]
        y_run = json.loads(json.dumps(y))
        y_run["debug"]["random_seed"] = seed
        cfg = config.from_dict(y)
        t0 = day_t0(cfg, c["train_open_ticks"])
        test = dict(c["test"], t0_ms=day_t0(cfg, c["test"]["open_ticks"]))
        ref = ol.run_ref(y_run, c["flow_seed"], c["env"], c["ticks"], t0_ms=t0, test=dict(test, logs=True))
        # the evaluation logs as the reference itself writes them (Backtester's profit_log, Base::writeStats)
        for fname in ("profit_log.csv", "test_stats.csv"):
            with open(os.path.join(GOLD, "%s_%s" % (c["name"], fname)), "w") as f:
                f.write(ref["logs"][fname])
        assert ref["summary"]["terminal"] == 1
        for suffix, recs in (("", ref["records"]), ("_test", ref["test_records"])):
            with open(os.path.join(GOLD, "steps_%s%s.bin" % (c["name"], suffix)), "wb") as f:
                for r in recs:
                    f.write(bytes(r))
        manifest.append(dict(c, yaml=y, backtest=True, t0_ms=t0, test=test, n_records=len(ref["records"]),
                             n_test_records=len(ref["test_records"]), summary=ref["summary"]))
        print(c["name"], len(ref["records"]), "training records;", len(ref["test_records"]), "evaluation records")
    for c in CONFIG_CASES:
        manifest.append(short_case(c))
    import golden_util
    import test_venue_days
    for c in VENUE_CASES:
        y = venue_yaml(c)
        with tempfile.TemporaryDirectory() as d:
            md, tas = golden_util.venue_day(c, d)
            raw, summary = test_venue_days.reference_on_day(ol, c, y, md, tas, d)
            sha = dict(md_sha256=file_sha256(md), tas_sha256=file_sha256(tas))
        recs = list((abi.StepRecord * (len(raw) // C.sizeof(abi.StepRecord))).from_buffer_copy(raw))
        assert summary["terminal"] == 1 and len(recs) == summary["steps"]
        _write_digests(c["name"], recs)  # whole days: 8-byte digests per record instead of ~220 KB of records each
        manifest.append(dict(c, yaml=y, venue_day=True, n_records=len(recs), summary=summary, **sha))
    _keep_wall_clock(manifest)
    with open(os.path.join(GOLD, "manifest.json"), "w") as f:
        json.dump(manifest, f, indent=1)
    reference_checks()


def _keep_wall_clock(manifest, path=os.path.join(GOLD, "manifest.json")):
    """The reference's run time is in the summaries it printed; an entry whose outputs did not change keeps the stored
    time, so that regenerating leaves the fixture file (manifest.json, eval_days.json) as it was."""
    if not os.path.exists(path):
        return
    old = {c["name"]: c for c in json.load(open(path))}
    clock = ("seconds", "steps_per_s")
    for c in manifest:
        o = old.get(c["name"])
        if o is None or "summary" not in o:
            continue
        same = {k: v for k, v in o["summary"].items() if k not in clock} == {k: v for k, v in c["summary"].items() if k not in clock}
        if same and json.dumps(dict(o, summary=None)) == json.dumps(dict(json.loads(json.dumps(c)), summary=None)):
            c["summary"] = o["summary"]


def short_case(c):
    """The first N_F2_RECORDS records of a single-episode reference run -> steps_<name>.bin; returns the manifest entry."""
    y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
    y_run = json.loads(json.dumps(y))
    y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + c["env"]
    ref = ol.run_ref(y_run, c["flow_seed"], c["env"], c["ticks"])
    recs = ref["records"][:N_F2_RECORDS]
    assert len(recs) == N_F2_RECORDS, (c["name"], len(recs))
    with open(os.path.join(GOLD, "steps_%s.bin" % c["name"]), "wb") as f:
        for r in recs:
            f.write(bytes(r))
    print(c["name"], len(recs), "records;", ref["summary"]["steps"], "reference steps")
    return dict(c, yaml=y, n_records=len(recs), summary=ref["summary"])


def _write_digests(name, recs):
    import golden_util
    with open(os.path.join(GOLD, "digests_%s.bin" % name), "wb") as f:
        for r in recs:
            f.write(golden_util.record_digest(r))
    print(name, len(recs), "record digests")


def reference_checks():
    """What the reference answered in the tests that compare with it on inputs they make themselves:
      tests/golden/digests_live_<algo>_m<M>.bin      test_oracle_golden.py::test_live_reference_when_built
      tests/golden/digests_ingest_fresh_messy_pair.bin  test_ingest.py::test_live_reference_on_a_fresh_messy_pair
      tests/golden/file_pairing.json                  test_file_pairing.py (oracle/_ref/ref_files)"""
    import pathlib
    import tempfile
    import test_file_pairing
    import test_ingest
    import test_oracle_golden
    for algo, M, seed, over in test_oracle_golden._LIVE:
        y, cfg = test_oracle_golden.live_config(algo, M, seed, over)
        ref = ol.run_ref(y, 123, 0, 4000, want_theta=True, t0_ms=cfg.flow.t0_ms)
        _write_digests("live_%s_m%d" % (algo, M), ref["records"])
    with tempfile.TemporaryDirectory() as d:
        y, _cfg, md, tas = test_ingest.fresh_messy_pair(ol, d)
        _write_digests("ingest_fresh_messy_pair", test_ingest.reference_on_csv(ol, y, md, tas, d))
    pairing = {}
    for md_name, tas_name in (("depth", "trade"), ("md_data", "tas_data"), ("d", "trades_long")):
        with tempfile.TemporaryDirectory() as d:
            pairing["%s,%s" % (md_name, tas_name)] = test_file_pairing.reference_answers(pathlib.Path(d), md_name, tas_name)
    with open(os.path.join(GOLD, "file_pairing.json"), "w") as f:
        json.dump(pairing, f, indent=1)


# One tape library of all nine venue days under one yaml (the config's market is AAL.L's): env b replays day b under its
# ticker's market (rlm_set_day_markets) with seed random_seed + DAY_MARKETS_ENV0 + b, as ref_driver --symbol <ticker> does.
# Written to tests/golden/day_markets.json and digests_daymkt_<case>.bin, not into manifest.json, whose entries without a
# known flag join the single-episode tests.
DAY_MARKETS_ENV0 = 60


def day_markets_yaml():
    return config.example_dict(**{"learning.memory_size": 8192, "learning.algorithm": "q_learn", "data.symbols": ["AAL.L"]})


def day_market_fixtures():
    import tempfile
    import golden_util
    import test_venue_days
    y = day_markets_yaml()
    days = []
    for b, c in enumerate(golden_util.venue_manifest()):
        case = dict(c, env=DAY_MARKETS_ENV0 + b)
        with tempfile.TemporaryDirectory() as d:
            md, tas = golden_util.venue_day(c, d)
            raw, summary = test_venue_days.reference_on_day(ol, case, y, md, tas, d)
        recs = list((abi.StepRecord * (len(raw) // C.sizeof(abi.StepRecord))).from_buffer_copy(raw))
        assert summary["terminal"] == 1 and len(recs) == summary["steps"]
        name = "daymkt_" + c["name"]
        _write_digests(name, recs)
        days.append(dict(name=name, venue_case=c["name"], ticker=c["ticker"], env=DAY_MARKETS_ENV0 + b, n_records=len(recs),
                         summary=summary))
    with open(os.path.join(GOLD, "day_markets.json"), "w") as f:
        json.dump(dict(yaml=y, env0=DAY_MARKETS_ENV0, days=days), f, indent=1)


# Evaluation over several test days (main.cpp:216-244): train until the close, GoGreedy, then ONE Intraday object for
# every test day -- LoadData, a new Backtester, Initialise, the steps, ClearInventory.  What Initialise leaves alone
# (the window sums of Accumulator::clear and RollingMean, A13; position; the greedy agent's rand()) runs from one day
# into the next.  A day is a synthetic stream (flow_seed, ticks, open_ticks; env = the case's) or a venue day
# (venue = a VENUE_CASES name, under its ticker's market).  Written to tests/golden/eval_days.json and
# digests_ed_<case>_{train,day<d>}.bin, not into manifest.json.
def _ed(name, algo, M, env, flow_seed, over, n_days=3, days=None):
    days = days or [dict(flow_seed=flow_seed + 1 + d, ticks=1000, open_ticks=700) for d in range(n_days)]
    return dict(name=name, algo=algo, M=M, env=env, flow_seed=flow_seed, ticks=1200, train_open_ticks=900, over=over, days=days)


_VARS4 = ["pos", "spd", "vol", "svl"]
EVAL_DAYS_CASES = [
    _ed("ed_double_q_default", "double_q_learn", 8192, 70, 201, {"learning.alpha_start": 0.01}),
    _ed("ed_q_vars13_micro_m5003", "q_learn", 5003, 71, 205,
        {"state.variables": _ALL_VARS, "state.lookback.rsi": 10, "state.lookback.vwap": 20,
         "market.target_price.type": "microprice", "market.target_price.lookback": 5}),
    _ed("ed_sarsa", "sarsa", 8192, 72, 209, {}, n_days=2),
    _ed("ed_r_learn", "r_learn", 8192, 73, 213, {"policy.eps_init": 0.3}, n_days=2),
    _ed("ed_online_r_learn", "online_r_learn", 8192, 74, 217, {"policy.eps_init": 0.3}, n_days=2),
    _ed("ed_double_r_learn", "double_r_learn", 8209, 75, 221, {"policy.eps_init": 0.3, "learning.alpha_start": 0.01}, n_days=2),
    _ed("ed_act5_vars4", "q_learn", 8192, 76, 225, {"learning.n_actions": 5, "state.variables": _VARS4}),
    _ed("ed_tickers_aal_baes", "q_learn", 8192, 77, 229, {}, days=[dict(venue="venue_aal_l"), dict(venue="venue_baes_l")]),
]


def eval_days_yaml(c):
    return config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})


def eval_day_inputs(c, d):
    """The days of case c as ol.run_ref takes them (venue days written as CSV pairs into directory d), and the same
    days with their t0_ms / ticker filled in for the fixture."""
    import golden_util
    cfg = config.from_dict(eval_days_yaml(c))
    venues = {v["name"]: v for v in VENUE_CASES}
    runs, days = [], []
    for k, day in enumerate(c["days"]):
        if "venue" in day:
            v = venues[day["venue"]]
            sub = os.path.join(d, "day%d" % k)
            os.makedirs(sub)
            md, tas = golden_util.venue_day(v, sub)
            runs.append(dict(md=md, tas=tas, symbol=v["ticker"]))
            days.append(dict(day, ticker=v["ticker"], md_sha256=file_sha256(md), tas_sha256=file_sha256(tas)))
        else:
            t = dict(day, env=c["env"], t0_ms=day_t0(cfg, day["open_ticks"]))
            runs.append(t)
            days.append(t)
    return runs, days


def eval_days_fixtures():
    import tempfile
    import hashlib
    out = []
    for c in EVAL_DAYS_CASES:
        y = eval_days_yaml(c)
        y_run = json.loads(json.dumps(y))
        y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + c["env"]
        t0 = day_t0(config.from_dict(y), c["train_open_ticks"])
        with tempfile.TemporaryDirectory() as d:
            runs, days = eval_day_inputs(c, d)
            runs[0] = dict(runs[0], logs=True)
            ref = ol.run_ref(y_run, c["flow_seed"], c["env"], c["ticks"], t0_ms=t0, tests=runs)
        assert ref["summary"]["terminal"] == 1
        _write_digests(c["name"] + "_train", ref["records"])
        per_day = ref["summary"]["test_days"]
        for k, recs in enumerate(ref["test_days"]):
            assert len(recs) == per_day[k]["test_steps"] > 100, (c["name"], k, len(recs))
            _write_digests("%s_day%d" % (c["name"], k), recs)
            days[k] = dict(days[k], n_records=len(recs), summary=per_day[k])
        logs = {n: hashlib.sha256(ref["logs"][n].encode()).hexdigest() for n in ("profit_log.csv", "test_stats.csv")}
        out.append(dict(c, yaml=y, t0_ms=t0, days=days, n_records=len(ref["records"]), logs_sha256=logs,
                        summary={k: v for k, v in ref["summary"].items() if k != "test_days"}))
    path = os.path.join(GOLD, "eval_days.json")
    _keep_wall_clock(out, path)
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


def build_ref_q_values():
    """Compile tools/ref_q_values.cpp against the reference objects oracle/Makefile built into oracle/_ref/obj, with that
    recipe's flags (REF, as there, is where the reference sources lie) -> oracle/_ref/ref_q_values."""
    import glob
    ref = os.environ.get("REF", "/root/reference")
    objs = sorted(glob.glob(os.path.join(ol.REF_DIR, "obj", "**", "*.o"), recursive=True))
    if not objs or not os.path.exists(os.path.join(ref, "include", "rl", "agent.h")):
        raise SystemExit("--q-values needs the reference sources ($REF) and oracle/_ref/obj (make -C oracle all)")
    spdlog = subprocess.check_output([sys.executable, "-c", "import flashinfer, os; print(os.path.join(os.path.dirname("
                                      "flashinfer.__file__), 'data', 'spdlog', 'include'))"]).decode().strip()
    exe = os.path.join(ol.REF_DIR, "ref_q_values")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++11", "-O3", "-DNDEBUG", "-ffp-contract=off", "-fPIC", "-w",
                           "-I" + os.path.join(ref, "include"), "-I" + os.path.join(ROOT, "oracle", "shim"), "-I" + spdlog,
                           "-I" + os.path.join(ROOT, "include"), "-include", "spdlog/spdlog.h",
                           "-include", "spdlog/sinks/rotating_file_sink.h", os.path.join(ROOT, "tools", "ref_q_values.cpp")]
                          + objs + ["-o", exe, "-lpthread"])
    return exe


def q_values_fixture():
    """getQ / getQb of the reference's QLearn / DoubleQLearn on random_init tables for a list of states."""
    doc = subprocess.check_output([build_ref_q_values()]).decode()
    json.loads(doc)
    with open(os.path.join(GOLD, "q_values.json"), "w") as f:
        f.write(doc)


# Training logs (logging.log_learning): model_log.csv of Agent::HandleTransition and training_log.csv of
# Learner::RunEpisode, written by the reference itself (tools/ref_train_logs.cpp).  A case trains one agent for `episodes`
# episodes on one Intraday, episode e on day e % len(days) (main.cpp:45-60); a day is a synthetic stream (flow_seed,
# ticks, open_ticks; env = the case's) or a venue day (a VENUE_CASES name, under its ticker's market).  Enough episodes
# that several 1000-update windows close, inside episodes and spanning episode boundaries.  Written to
# tests/golden/training_logs.json and tl_<case>_{model_log,training_log}.csv, not into manifest.json.
def _tl(name, algo, M, env, flow_seed, over, episodes=8, days=None):
    days = days or [dict(flow_seed=flow_seed, ticks=2100, open_ticks=1800)]
    return dict(name=name, algo=algo, M=M, env=env, over=over, episodes=episodes, days=days)


TRAINING_LOG_CASES = [
    _tl("tl_q_learn_eps", "q_learn", 8192, 80, 301, {"policy.eps_T": 5}),
    _tl("tl_sarsa_boltzmann", "sarsa", 8192, 81, 303,
        {"policy.type": "boltzmann", "policy.tau_init": 0.05, "policy.tau_floor": 0.01, "policy.tau_T": 10}),
    _tl("tl_double_q_greedy", "double_q_learn", 8192, 82, 305, {"policy.type": "greedy", "learning.alpha_start": 0.01}),
    _tl("tl_r_learn", "r_learn", 8192, 83, 307, {"policy.eps_init": 0.3}),
    _tl("tl_online_r_learn", "online_r_learn", 8192, 84, 309, {"policy.eps_init": 0.3}),
    _tl("tl_double_r_learn", "double_r_learn", 8209, 85, 311, {"policy.eps_init": 0.3, "learning.alpha_start": 0.01}),
    _tl("tl_q_learn_two_days", "q_learn", 5003, 86, 313, {}, episodes=9,
        days=[dict(flow_seed=313, ticks=1500, open_ticks=1200), dict(flow_seed=314, ticks=2400, open_ticks=2100)]),
    _tl("tl_venue_aal", "q_learn", 8192, 87, 0, {}, episodes=4, days=[dict(venue="venue_aal_l")]),
]


def training_logs_yaml(c, out_dir=None):
    y = config.example_dict(**{"learning.memory_size": c["M"], "learning.algorithm": c["algo"], **c["over"]})
    if out_dir is not None:  # Agent's / Learner's ctors open <output_dir>model_log.csv / training_log.csv
        y["logging"] = {"log_learning": True, "max_size": 1 << 40}
        y["output_dir"] = out_dir
    return y


def build_ref_train_logs():
    """Compile tools/ref_train_logs.cpp against the reference objects oracle/Makefile built into oracle/_ref/obj, with that
    recipe's flags -> oracle/_ref/ref_train_logs."""
    import glob
    ref = os.environ.get("REF", "/root/reference")
    objs = sorted(glob.glob(os.path.join(ol.REF_DIR, "obj", "**", "*.o"), recursive=True))
    if not objs or not os.path.exists(os.path.join(ref, "include", "rl", "agent.h")):
        raise SystemExit("--training-logs needs the reference sources ($REF) and oracle/_ref/obj (make -C oracle all)")
    spdlog = subprocess.check_output([sys.executable, "-c", "import flashinfer, os; print(os.path.join(os.path.dirname("
                                      "flashinfer.__file__), 'data', 'spdlog', 'include'))"]).decode().strip()
    exe = os.path.join(ol.REF_DIR, "ref_train_logs")
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++14", "-O3", "-DNDEBUG", "-ffp-contract=off", "-fPIC", "-w",
                           "-I" + os.path.join(ref, "include"), "-I" + os.path.join(ROOT, "oracle", "shim"), "-I" + spdlog,
                           "-include", "spdlog/spdlog.h", "-include", "spdlog/sinks/rotating_file_sink.h",
                           os.path.join(ROOT, "tools", "ref_train_logs.cpp")]
                          + objs + ["-o", exe, "-lpthread"])
    return exe


def training_logs_fixtures():
    import tempfile
    import golden_util
    exe = build_ref_train_logs()
    venues = {v["name"]: v for v in VENUE_CASES}
    out = []
    for c in TRAINING_LOG_CASES:
        y = training_logs_yaml(c)
        cfg = config.from_dict(y)
        with tempfile.TemporaryDirectory() as d:
            logs = os.path.join(d, "logs") + "/"
            os.makedirs(logs)
            y_run = json.loads(json.dumps(training_logs_yaml(c, logs)))
            y_run["debug"]["random_seed"] = y["debug"]["random_seed"] + c["env"]
            cfgp = os.path.join(d, "cfg.yaml")
            ol.write_ref_yaml(cfgp, y_run)
            cmd, days = [exe, "--config", cfgp, "--episodes", str(c["episodes"])], []
            for k, day in enumerate(c["days"]):
                if "venue" in day:
                    v = venues[day["venue"]]
                    sub = os.path.join(d, "day%d" % k)
                    os.makedirs(sub)
                    md, tas = golden_util.venue_day(v, sub)
                    days.append(dict(day, ticker=v["ticker"], md_sha256=file_sha256(md), tas_sha256=file_sha256(tas)))
                    cmd += ["--symbol", v["ticker"], "--md", md, "--tas", tas]
                else:
                    t0 = day_t0(cfg, day["open_ticks"])
                    md, tas = os.path.join(d, "d%d_md_1.csv" % k), os.path.join(d, "d%d_tas_1.csv" % k)
                    subprocess.check_call([ol.FLOW_CSV, "--seed", str(day["flow_seed"]), "--env", str(c["env"]), "--ticks", str(day["ticks"]),
                                           "--dt-ms", "250", "--md", md, "--tas", tas, "--t0-ms", str(t0)])
                    days.append(dict(day, t0_ms=t0))
                    cmd += ["--symbol", y["data"]["symbols"][0], "--md", md, "--tas", tas]
            summary = json.loads(subprocess.check_output(cmd).decode().strip().splitlines()[-1])
            files = {}
            for n in ("model_log", "training_log"):
                with open(os.path.join(logs, n + ".csv")) as f:
                    files[n] = f.read()
                with open(os.path.join(GOLD, "%s_%s.csv" % (c["name"], n)), "w") as f:
                    f.write(files[n])
        n_rows = len(files["model_log"].splitlines())
        assert n_rows >= 2, (c["name"], n_rows)
        out.append(dict(c, yaml=y, days=days, episode_ids=[e["episode_id"] for e in summary["episodes"]], model_log_rows=n_rows))
    with open(os.path.join(GOLD, "training_logs.json"), "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    if sys.argv[1:] == ["--q-values"]:
        q_values_fixture()
    elif sys.argv[1:] == ["--training-logs"]:
        training_logs_fixtures()
    elif sys.argv[1:] == ["--reference-checks"]:
        reference_checks()
    elif sys.argv[1:] == ["--day-markets"]:
        day_market_fixtures()
    elif sys.argv[1:] == ["--eval-days"]:
        eval_days_fixtures()
    else:
        main()
