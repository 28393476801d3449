"""main.cpp:216-244 through the class surface (include/rlm_facade.hpp): examples/serial_driver trains, then GoGreedy, ONE
new Intraday and per test day LoadData + experiment::serial::Backtester::RunEpisode.  Its per-day lines must equal a
fused-path handle taken through the same sequence -- handle_terminal, go_greedy, rlm_new_env, then per day set_flow +
reset (synthetic days) or assign_days + reset (CSV pairs on the tape source) -- and its training lines and theta what
tests/test_gpu_facade.py and tests/test_gpu_tape.py hold."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import pytest

import golden_util as G
from rl_markets_b200 import abi, lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "examples", "serial_driver")
MSG = C.sizeof(abi.TickMsg)


def _run(args):
    assert os.path.exists(DRIVER), "examples/serial_driver is built by __graft_entry__.build()"
    lines = [json.loads(l) for l in subprocess.check_output([DRIVER] + args).decode().strip().splitlines()]
    return [l for l in lines if "episode" in l], [l for l in lines if "test_day" in l]


def _day_matches(st, line, tag):
    assert st.terminal == 1, tag
    assert (st.steps, st.episode_reward, st.episode_pnl, st.ask_transactions + st.bid_transactions) == \
        (line["steps"], line["reward"], line["pnl"], line["transactions"]), (tag, line)
    assert st.episode_reward / st.total_ticks == line["mean_reward"], tag  # Base::getMeanEpisodeReward (base.cpp:249-252)


@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_serial_driver_test_days_match_the_fused_path(rlm, algo):
    M, open_ticks, episodes, seeds = 8192, 400, 2, [51, 52]
    with tempfile.TemporaryDirectory() as d:
        thp = os.path.join(d, "theta.bin")
        eps, days = _run(["--episodes", str(episodes), "--algo", algo, "--memory-size", str(M), "--open-ticks", str(open_ticks),
                          "--theta", thp] + [a for s in seeds for a in ("--test-seed", str(s))])
        raw = open(thp, "rb").read()
    assert len(eps) == episodes and all(e["steps"] > 40 for e in eps)
    assert [l["test_day"] for l in days] == [1, 2] and all(l["steps"] > 40 for l in days)
    L = rlm.load()
    cfg = abi.Config()
    rlm.check(L.rlm_config_default(C.byref(cfg)))
    cfg.algorithm = abi.ALGO[algo]
    cfg.memory_size = M
    cfg.flow.seed = 41
    cfg.flow.t0_ms = int(cfg.close_ms) - 30 * 60000 - open_ticks * cfg.flow.dt_ms
    m = rlm.BatchedMarket(cfg)
    for ep in range(episodes):                    # the training lines, as tests/test_gpu_facade.py checks them
        m.run_ticks(open_ticks + 200)
        m.sync()
        st = m.stats(0, 1)[0]
        assert st.terminal == 1
        assert st.steps == eps[ep]["steps"] and st.episode_pnl == eps[ep]["pnl"] and st.episode_reward == eps[ep]["reward"]
        m.handle_terminal(ep)
        if ep + 1 < episodes:
            m.reset()
    assert bytes(m.theta(0, 0)) == raw
    m.go_greedy()                                 # main.cpp:217
    m.set_mode(abi.MODE_BACKTEST)
    m.new_env(None)                               # environment::Intraday<> env(c), main.cpp:219
    for k, s in enumerate(seeds):
        flow = abi.FlowParams.from_buffer_copy(bytes(m.cfg.flow))
        flow.seed = s
        m.set_flow(flow)                          # env.LoadData(...)
        m.reset()                                 # Backtester::RunEpisode: Initialise
        m.run_ticks(open_ticks + 200)
        m.sync()
        _day_matches(m.stats(0, 1)[0], days[k], (algo, "day", k))
    assert bytes(m.theta(0, 0)) == raw, "evaluation must not touch theta"
    m.close()


def test_serial_driver_test_days_on_csv_pairs(rlm):
    """trained on a golden CSV pair (tape source), tested on two venue days the test writes: per test day
    Intraday::LoadData(ticker, md, tas) on one new env object equals assign_days + reset on a fused day library"""
    case = G.ingest_manifest()[0]
    venue = next(v for v in G.venue_manifest() if v["ticker"] == "AAL.L")
    md, tas = G.ingest_paths(case)
    M, episodes = case["M"], 1
    with tempfile.TemporaryDirectory() as d:
        pairs = []
        for k, seed in enumerate((venue["day_seed"], venue["day_seed"] + 1)):
            sub = os.path.join(d, "day%d" % k)
            os.mkdir(sub)
            pairs.append(G.venue_day(venue, sub, seed=seed))
        eps, days = _run(["--md", md, "--tas", tas, "--episodes", str(episodes), "--algo", case["algo"], "--memory-size", str(M),
                          "--env", str(case["env"])] + [a for p, q in pairs for a in ("--test-md", p, "--test-tas", q)])
        per_day = [lib.ingest_csv(md, tas)[:2]] + [lib.ingest_csv(p, q)[:2] for p, q in pairs]
    assert len(eps) == episodes and eps[0]["steps"] == case["n_records"], eps
    assert [l["test_day"] for l in days] == [1, 2]
    offs = [0]
    for _a, n in per_day:
        offs.append(offs[-1] + n)
    buf = (abi.TickMsg * offs[-1])()
    for (a, n), o in zip(per_day, offs):
        C.memmove(C.addressof(buf) + o * MSG, a, n * MSG)
    L = rlm.load()
    cfg = abi.Config()
    rlm.check(L.rlm_config_default(C.byref(cfg)))
    cfg.algorithm = abi.ALGO[case["algo"]]
    cfg.memory_size = M
    cfg.env_index0 = case["env"]
    cfg.source = abi.SOURCE_TAPE
    m = rlm.BatchedMarket(cfg)
    m.load_days(buf, offs)
    m.run_ticks(per_day[0][1] + 7)
    m.sync()
    st = m.stats(0, 1)[0]
    assert st.steps == eps[0]["steps"] and st.episode_pnl == eps[0]["pnl"] and st.episode_reward == eps[0]["reward"]
    m.handle_terminal(0)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    for k in range(len(pairs)):
        m.assign_days([1 + k])
        if k == 0:
            m.new_env(None)                       # the test phase's env object (main.cpp:219)
        else:
            m.reset()                             # LoadData + Initialise on the same object
        m.run_ticks(per_day[1 + k][1] + 7)
        m.sync()
        _day_matches(m.stats(0, 1)[0], days[k], ("csv day", k))
    m.close()
