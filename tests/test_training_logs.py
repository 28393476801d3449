"""The reference's training logs (logging.log_learning) on the CPU: model_log.csv (Agent::HandleTransition,
src/rl/agent.cpp:86-101) and training_log.csv (Learner::RunEpisode, src/experiment/serial.cpp:72-94).

The fixtures (tests/golden/training_logs.json, tl_<case>_{model_log,training_log}.csv) are the files the unmodified
reference writes itself (tools/make_golden.py --training-logs).  Here the CPU oracle trains the same agent over the same
episodes: the sequential sum of its per-step |delta|, divided by 1000 on every 1000th update, gives the model_log values
bit for bit, and rl_markets_b200.train_logs renders both files byte for byte from the oracle's deltas and episode
statistics.  The bindings' argument checks need no device either."""
import ctypes as C
import functools
import hashlib
import json
import os
import struct
import tempfile

import pytest

import golden_util as G
import oracle_lib
from rl_markets_b200 import abi, config, train_logs
from rl_markets_b200 import lib as rlm_lib

with open(os.path.join(G.GOLD, "training_logs.json")) as _f:
    CASES = json.load(_f)
_VENUE = {c["name"]: c for c in G.venue_manifest()}
CAP = 8000


def case(name):
    return next(c for c in CASES if c["name"] == name)


def fixture(c, which):
    with open(os.path.join(G.GOLD, "%s_%s.csv" % (c["name"], which))) as f:
        return f.read()


def base_config(c, **kw):
    """the case's config, its first day's flow (env index c["env"] + b for env b)"""
    cfg = config.from_dict(c["yaml"], flow_seed=c["days"][0].get("flow_seed", 0), env_index0=c["env"], **kw)
    if "t0_ms" in c["days"][0]:
        cfg.flow.t0_ms = c["days"][0]["t0_ms"]
    return cfg


def day_flow(c, k):
    day = c["days"][k]
    flow = config.from_dict(c["yaml"], flow_seed=day["flow_seed"]).flow
    flow.t0_ms = day["t0_ms"]
    return flow


@functools.lru_cache(maxsize=None)
def day_messages(name, k, env_index=None):
    """day k of case `name` as one env's message stream -> (ctypes TickMsg array, message count)"""
    c = case(name)
    day = c["days"][k]
    if "venue" not in day:
        return rlm_lib.flow_generate(day_flow(c, k), c["env"] if env_index is None else env_index, 0, day["ticks"]), day["ticks"]
    with tempfile.TemporaryDirectory() as d:
        md, tas = G.venue_day(_VENUE[day["venue"]], d)
        for p, key in ((md, "md_sha256"), (tas, "tas_sha256")):
            assert hashlib.sha256(open(p, "rb").read()).hexdigest() == day[key], (name, k, p)
        msgs, n, _t = rlm_lib.ingest_csv(md, tas)
    return msgs, n


def policy_descr(cfg, episode):
    """Policy::descr() after HandleTerminal(episode) (policy.cpp:77-82,117-122): the oracle's schedule"""
    if cfg.policy_type == abi.POLICY["epsilon_greedy"]:
        e0, ef = float(cfg.eps_init), float(cfg.eps_floor)
        return e0 * pow(ef / e0, episode / float(cfg.eps_T))
    if cfg.policy_type == abi.POLICY["boltzmann"]:
        t0, tf = float(cfg.tau_init), float(cfg.tau_floor)
        return t0 * pow(tf / t0, episode / float(cfg.tau_T))
    return 0.0


@functools.lru_cache(maxsize=None)
def oracle_run(name, b=0):
    """The case's episodes on the CPU oracle for env b (global index c["env"] + b): per episode the TD errors of its
    steps in order and (reward, pnl, steps, descr) after HandleTerminal"""
    c = case(name)
    cfg = base_config(c)
    L = oracle_lib.lib()
    h = L.lobo_create(C.byref(cfg), c["env"] + b)
    assert h
    episodes = []
    try:
        for e in range(c["episodes"]):
            if e:
                L.lobo_reset(h)
            msgs, n = day_messages(name, e % len(c["days"]), c["env"] + b)
            recs = (abi.StepRecord * CAP)()
            used = C.c_int64()
            k = L.lobo_run(h, msgs, n, -1, recs, CAP, C.byref(used))
            assert 0 < k < CAP and recs[k - 1].terminal == 1, (name, e, k)
            st = abi.EnvStats()
            L.lobo_stats(h, C.byref(st))
            L.lobo_handle_terminal(h, e)
            episodes.append(dict(deltas=[recs[i].delta for i in range(k)], reward=st.episode_reward, pnl=st.episode_pnl,
                                 steps=st.steps, descr=policy_descr(cfg, e)))
    finally:
        L.lobo_destroy(h)
    return episodes


def expected_files(c, episodes):
    """(model_log.csv, training_log.csv) rendered by train_logs from per-episode deltas and statistics"""
    deltas = [d for ep in episodes for d in ep["deltas"]]
    vals, _agg, _n = train_logs.model_log_values(deltas)
    ml = "".join(line + "\n" for line in train_logs.model_log_lines(vals))
    rows = [train_logs.TRAINING_HEADER] + [
        train_logs.training_log_line(e + 1, c["episode_ids"][e], ep["reward"], ep["pnl"], ep["steps"], ep["descr"])
        for e, ep in enumerate(episodes)]
    return ml, "".join(r + "\n" for r in rows), vals


def _bits(x):
    return struct.pack("<d", x)


@pytest.mark.parametrize("name", [c["name"] for c in CASES])
def test_oracle_reproduces_the_reference_logs(name):
    c = case(name)
    eps = oracle_run(name)
    ml, tl, vals = expected_files(c, eps)
    want_ml = fixture(c, "model_log")
    # the values bit for bit: every logged line parses to the oracle's sequential sum / 1000.0
    assert [_bits(float(x)) for x in want_ml.split()] == [_bits(v) for v in vals], name
    assert ml == want_ml, name
    assert tl == fixture(c, "training_log"), name


def test_fixtures_cover_the_log_boundaries():
    """Every algorithm, the three Policy::descr() forms, 1000-update windows closing inside an episode and spanning an
    episode boundary, several days in one run and a venue day."""
    assert {c["algo"] for c in CASES} == set(abi.ALGO)
    assert {c["yaml"]["policy"]["type"] for c in CASES} >= {"epsilon_greedy", "boltzmann", "greedy"}
    assert any(len(c["days"]) > 1 for c in CASES) and any("venue" in d for c in CASES for d in c["days"])
    inside = spanning = 0
    for c in CASES:
        bounds, total = [], 0
        for ep in oracle_run(c["name"]):
            bounds.append((total, total + len(ep["deltas"])))
            total += len(ep["deltas"])
        assert c["model_log_rows"] == total // 1000 >= 2, c["name"]
        for k in range(1, total // 1000 + 1):
            lo, hi = 1000 * (k - 1), 1000 * k
            spanning += any(a <= lo < b < hi for a, b in bounds) or any(lo < a < hi for a, _b in bounds)
            inside += any(a < hi < b for a, b in bounds)
    assert inside > 0 and spanning > 0


def test_model_log_values_is_handle_transition():
    """the counter and the sum carry over calls, and reset on every 1000th update"""
    d = [((-1) ** i) * (i % 7) * 0.125 for i in range(2500)]
    whole, agg, n = train_logs.model_log_values(d)
    a, agg1, n1 = train_logs.model_log_values(d[:1234])
    b, agg2, n2 = train_logs.model_log_values(d[1234:], agg1, n1)
    assert a + b == whole and (agg2, n2) == (agg, n) and n == 500 and len(whole) == 2
    s = 0.0
    for x in d[:1000]:
        s += abs(x)
    assert whole[0] == s / 1000.0


def test_training_log_line_format():
    assert train_logs.training_log_line(3, "20100104", -12.5, 0.0, 412, 0.800000011920929) == "3,20100104,-12.5,0,412,0.800000011920929"
    assert train_logs.model_log_lines([0.0, 1.25e-05, 2.0]) == ["0", "1.25e-05", "2"]


def test_bindings_are_exported():
    for n in ("rlm_set_model_log", "rlm_read_model_log", "rlm_get_policy_descr"):
        assert n in rlm_lib.EXPORTS
    L = rlm_lib.load()
    for fn in (L.rlm_set_model_log, L.rlm_read_model_log, L.rlm_get_policy_descr):
        assert fn.argtypes


def test_null_handle_is_rejected():
    L = rlm_lib.load()
    out = C.c_double(7.0)
    assert L.rlm_set_model_log(None, 16) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_get_policy_descr(None, C.byref(out)) == abi.RLM_ERR_INVALID_ARGUMENT and out.value == 7.0
    rows, n = (C.c_double * 4)(), (C.c_int32 * 1)()
    assert L.rlm_read_model_log(None, 0, 1, rows, n) == abi.RLM_ERR_INVALID_ARGUMENT


def test_set_model_log_checks_its_argument_type():
    class Fake(rlm_lib.BatchedMarket):
        def __init__(self):
            self.h = C.c_void_p()

    for bad in (1.5, "8", True, None):
        with pytest.raises(TypeError):
            Fake().set_model_log(bad)


def test_facade_number_rendering_is_backtest_num(tmp_path):
    """rlm::log_num (include/rlm_facade.hpp, the class surface's log writer) prints every number as backtest._num does:
    the fixture values, integral values, exponents on both sides of repr's switch points and random doubles"""
    import random
    import shutil
    import subprocess
    from rl_markets_b200.backtest import _num
    cxx = shutil.which("g++") or shutil.which("c++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = tmp_path / "n.cpp"
    src.write_text('#include "rlm_facade.hpp"\n#include <cstdio>\n'
                   'int main() { double x; while (fread(&x, 8, 1, stdin) == 1) printf("%s\\n", rlm::log_num(x).c_str()); }\n')
    exe = tmp_path / "n"
    subprocess.check_call([cxx, "-std=c++17", "-I" + os.path.join(oracle_lib.ROOT, "include"), str(src), "-o", str(exe)])
    vals = [0.0, 1.0, -1.0, 5.0, -527.5, 0.800000011920929, 1.25e-05, 1e-4, 1e-5, 123456789012345.0, 1e15, 1e16, 2.5e16,
            -1e20, 0.1, 1 / 3, 1e-300, 5e-324, 1.7976931348623157e308, 12345.678, -0.0001234]
    for c in CASES:
        for which in ("model_log", "training_log"):
            for tok in fixture(c, which).replace("\n", ",").split(","):
                try:
                    vals.append(float(tok))
                except ValueError:
                    pass
    rng = random.Random(5)
    for _ in range(5000):
        vals.append(rng.choice([rng.uniform(-1e6, 1e6), rng.expovariate(1.0) * 10.0 ** rng.randint(-20, 20),
                                rng.randint(-10 ** 6, 10 ** 6) / rng.choice([1, 2, 4, 8, 1000])]))
    out = subprocess.run([str(exe)], input=b"".join(struct.pack("<d", v) for v in vals), capture_output=True, check=True)
    got = out.stdout.decode().split("\n")[:-1]
    assert got == [_num(v) for v in vals]
