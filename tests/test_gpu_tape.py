"""The tape source: a device-resident library of whole days (rlm_load_days) replayed through one cursor per env.

Everything is compared bitwise: step records (abi.record_fields_equal), theta bytes and rlm_env_stats bytes.  The tape
path must equal the stream path on the same per-env days, reproduce the reference's records on the golden CSV pairs on
every surface (fused, round-paced, split, facade), and stop an env at the end of its day inside performAction."""
import ctypes as C
import json
import os
import subprocess
import tempfile
import time

import pytest

import golden_util as G
from rl_markets_b200 import abi, ingest, lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVER = os.path.join(ROOT, "examples", "serial_driver")
MSG = C.sizeof(abi.TickMsg)


def _ingested():
    """[(case, msgs, n)] for the golden CSV pairs, in manifest order."""
    out = []
    for case in G.ingest_manifest():
        md, tas = G.ingest_paths(case)
        msgs, n, _ticks = lib.ingest_csv(md, tas)
        out.append((case, msgs, n))
    return out


def _head(arr, n):
    return (abi.TickMsg * n).from_buffer_copy((C.c_char * (n * MSG)).from_address(C.addressof(arr)))


def _library(days):
    """days: [(msgs, n)] -> (concatenated messages, offsets)"""
    offs = [0]
    for _a, n in days:
        offs.append(offs[-1] + n)
    buf = (abi.TickMsg * offs[-1])()
    for (a, n), o in zip(days, offs):
        C.memmove(C.addressof(buf) + o * MSG, a, n * MSG)
    return buf, offs


def _wide(per_env, T):
    """stream-source layout msgs[t][env] of the first T messages of every env's day"""
    B = len(per_env)
    wide = (abi.TickMsg * (T * B))()
    for b, (a, _n) in enumerate(per_env):
        for t in range(T):
            wide[t * B + b] = a[t]
    return wide


def _set_engine(monkeypatch, variant, rounds):
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    monkeypatch.setenv("RLM_ROUNDS", str(rounds))


def _assert_same(ma, mb, B, policies=None):
    for b in range(B):
        ra, _k1 = ma.records(b)
        rb, _k2 = mb.records(b)
        assert len(ra) == len(rb) > 20, (b, len(ra), len(rb))
        for i in range(len(ra)):
            bad = abi.record_fields_equal(ra[i], rb[i])
            assert not bad, (b, i, G.describe_diff(ra[i], rb[i], bad))
    for p in (range(B) if policies is None else policies):
        assert bytes(ma.theta(p)) == bytes(mb.theta(p)), p
    assert bytes(ma.stats()) == bytes(mb.stats())


def _assert_port(rlm_m, oracle, cfg, b, msgs, n):
    """env b of the handle against the CPU oracle fed the same n messages"""
    port = oracle.run_port(cfg, cfg.env_index0 + b, _head(msgs, n), rec_cap=2000)
    recs, _k = rlm_m.records(b)
    assert len(recs) == port["steps"] > 20, (b, len(recs), port["steps"])
    for i in range(port["steps"]):
        bad = abi.record_fields_equal(recs[i], port["records"][i])
        assert not bad, (b, i, G.describe_diff(recs[i], port["records"][i], bad))
    assert bytes(rlm_m.theta(b)) == bytes((C.c_double * cfg.memory_size)(*port["theta"])), b


ENGINES = [(0, 0), (0, 1), (1, 0)]  # (RLM_ENV_VARIANT, RLM_ROUNDS): warp-per-env, round-paced, thread-per-env


@pytest.mark.parametrize("variant,rounds", ENGINES)
def test_tape_equals_stream(rlm, oracle, monkeypatch, variant, rounds):
    """The same per-env days through rlm_run_ticks on both sources, calls split at odd lengths (a call boundary may fall
    inside a multi-message tick), envs sharing days and envs on days of their own."""
    _set_engine(monkeypatch, variant, rounds)
    ing = _ingested()
    case = ing[0][0]
    B = 6
    cfg_s = G.case_config(case, n_envs=B, env_index0=40, source=abi.SOURCE_STREAM)
    synth = lib.flow_generate(cfg_s.flow, 9, 0, 1400)
    days = [(ing[0][1], ing[0][2]), (ing[1][1], ing[1][2]), (synth, 1400)]
    assign = [2, 0, 0, 1, 2, 1]
    per_env = [days[d] for d in assign]
    T = min(n for _a, n in per_env)
    calls = [37, 129, 1, 250, T - 417]
    cfg_s.record_envs, cfg_s.record_cap = B, 1000
    ms = rlm.BatchedMarket(cfg_s)
    ms.load_ticks(_wide(per_env, T), T)
    for n in calls:
        ms.run_ticks(n)
    ms.sync()
    cfg_t = G.case_config(case, n_envs=B, env_index0=40, source=abi.SOURCE_TAPE)
    cfg_t.record_envs, cfg_t.record_cap = B, 1000
    mt = rlm.BatchedMarket(cfg_t)
    buf, offs = _library(days)
    mt.load_days(buf, offs)
    mt.assign_days(assign)
    mt.reset()
    for n in calls:
        mt.run_ticks(n)
    mt.sync()
    assert mt.tape_pos() == [T] * B
    assert mt.counters().ticks == ms.counters().ticks
    _assert_same(ms, mt, B)
    for b in (0, 3):
        _assert_port(mt, oracle, cfg_t, b, per_env[b][0], T)
    ms.close()
    mt.close()


def _golden_handle(rlm, ing, ci, B, source=abi.SOURCE_TAPE):
    """A handle on the golden case ci's config whose env ci carries the case's seeds; library = every golden pair,
    env b on day b % n_days (so env ci replays case ci's pair)."""
    case = ing[ci][0]
    cfg = G.case_config(case, n_envs=B, env_index0=case["env"] - ci, source=source)
    cfg.record_envs, cfg.record_cap = B, 1000
    m = rlm.BatchedMarket(cfg)
    if source == abi.SOURCE_TAPE:
        buf, offs = _library([(a, n) for _c, a, n in ing])
        m.load_days(buf, offs)
    return m, cfg


def _assert_golden(m, case, b):
    recs, _k = m.records(b)
    gold, _k2 = G.records(case["name"])
    assert len(recs) == len(gold) == case["n_records"], (case["name"], len(recs), len(gold))
    for i, g in enumerate(gold):
        bad = abi.record_fields_equal(g, recs[i])
        assert not bad, "%s step %d (reference, cuda): %r" % (case["name"], i, G.describe_diff(g, recs[i], bad))


@pytest.mark.parametrize("variant,rounds", ENGINES)
def test_golden_pairs_from_one_library(rlm, oracle, monkeypatch, variant, rounds):
    """Both golden CSV pairs in one library, envs alternating days: the env with a case's seeds reproduces the reference's
    records on it, every other env the oracle's on its day; every env ends having consumed its whole day."""
    _set_engine(monkeypatch, variant, rounds)
    ing = _ingested()
    B = 4
    longest = max(n for _c, _a, n in ing)
    for ci in range(len(ing)):
        m, cfg = _golden_handle(rlm, ing, ci, B)
        m.run_ticks(longest // 3)
        m.run_ticks(longest)  # more than any day holds: envs stop at the end of theirs
        m.sync()
        _assert_golden(m, ing[ci][0], ci)
        assert m.tape_pos() == [ing[b % len(ing)][2] for b in range(B)]
        for b in range(B):
            if b != ci:
                _assert_port(m, oracle, cfg, b, ing[b % len(ing)][1], ing[b % len(ing)][2])
        m.close()


def test_backtest_on_tape_equals_stream(rlm):
    """Backtester::_step on the tick-synchronous engine reads the tape like the stream."""
    ing = _ingested()
    case, msgs, n = ing[0]
    B = 2
    out = []
    for source in (abi.SOURCE_STREAM, abi.SOURCE_TAPE):
        cfg = G.case_config(case, n_envs=B, env_index0=case["env"], source=source)
        cfg.record_envs, cfg.record_cap = B, 1000
        m = rlm.BatchedMarket(cfg)
        m.set_mode(abi.MODE_BACKTEST)
        if source == abi.SOURCE_STREAM:
            m.load_ticks(_wide([(msgs, n)] * B, n), n)
        else:
            m.load_days(msgs, [0, n])
        m.run_ticks(n // 2)
        m.run_ticks(n - n // 2)
        m.sync()
        out.append(m)
    _assert_same(out[0], out[1], B)
    for m in out:
        m.close()


def test_split_surface_on_tape(rlm, oracle):
    """act -> env_step -> agent_update on the golden pairs: the reference's records, terminal_out == 2 on the env_step after
    an env's last complete step, act == -1 from then on, and a prompt return once every env is out of data."""
    ing = _ingested()
    B = 4
    for ci in range(len(ing)):
        m, cfg = _golden_handle(rlm, ing, ci, B)
        steps = [len(oracle.run_port(cfg, cfg.env_index0 + b, _head(*ing[b % len(ing)][1:]), rec_cap=2000)["records"])
                 for b in range(B)]
        _rew, term = m.env_step(None)
        assert not any(term)
        m.agent_update()
        first2 = [None] * B
        k = 0
        while None in first2:
            k += 1
            assert k <= max(steps) + 2, (k, first2, steps)
            a = m.act()
            for b in range(B):
                assert (a[b] == -1) == (first2[b] is not None), (b, k, a[b])
            _rew, term = m.env_step(a)
            for b in range(B):
                assert term[b] in (0, 2)
                if term[b] == 2 and first2[b] is None:
                    first2[b] = k
                assert (term[b] == 2) == (first2[b] is not None)
            m.agent_update()
        assert first2 == [s + 1 for s in steps], (first2, steps)
        t0 = time.time()
        _rew, term = m.env_step(m.act())
        assert list(term) == [2] * B and time.time() - t0 < 5.0
        m.sync()
        _assert_golden(m, ing[ci][0], ci)
        assert m.tape_pos() == [ing[b % len(ing)][2] for b in range(B)]
        m.close()


def test_split_run_then_fused_run_on_tape(rlm, oracle):
    ing = _ingested()
    m, cfg = _golden_handle(rlm, ing, 0, 2)
    m.env_step(None)
    m.agent_update()
    for _k in range(100):
        m.env_step(m.act())
        m.agent_update()
    m.run_ticks(max(n for _c, _a, n in ing))  # the fused path continues each env where the split surface left it
    m.sync()
    _assert_golden(m, ing[0][0], 0)
    _assert_port(m, oracle, cfg, 1, ing[1][1], ing[1][2])
    assert m.tape_pos() == [ing[0][2], ing[1][2]]
    m.close()


def test_episodes_and_reassignment(rlm, oracle):
    """Episode 1 on day A until the close, handle_terminal, assign_days to day B, reset, episode 2: the oracle with
    lobo_handle_terminal + lobo_reset fed B's messages."""
    from rl_markets_b200 import config
    n_envs, cap = 4, 900
    y = config.example_dict(**{"learning.memory_size": 8192, "learning.omega": 0.9, "learning.alpha_start": 0.01,
                               "policy.eps_T": 3})
    cfg = config.from_dict(y, n_envs=n_envs, flow_seed=41, dt_ms=250, source=abi.SOURCE_TAPE)
    cfg.flow.t0_ms = int(cfg.close_ms) - 30 * 60000 - 500 * 250  # the market closes 500 rows after the first one
    cfg.record_envs, cfg.record_cap = n_envs, cap
    flow_b = abi.FlowParams.from_buffer_copy(bytes(cfg.flow))
    flow_b.seed = 4242
    L_A, L_B = 700, 600
    days = [(lib.flow_generate(cfg.flow, b, 0, L_A), L_A) for b in range(n_envs)]
    days += [(lib.flow_generate(flow_b, b, 0, L_B), L_B) for b in range(n_envs)]
    m = rlm.BatchedMarket(cfg)
    buf, offs = _library(days)
    m.load_days(buf, offs)
    m.assign_days(list(range(n_envs)))
    m.run_ticks(L_A)
    m.sync()
    assert all(s.terminal == 1 for s in m.stats())
    m.handle_terminal(1)
    m.assign_days([n_envs + b for b in range(n_envs)])
    m.reset()
    m.run_ticks(300)
    m.sync()
    assert m.tape_pos() == [300] * n_envs
    L = oracle.lib()
    st = m.stats()
    for b in range(n_envs):
        h = L.lobo_create(C.byref(cfg), b)
        recs = (abi.StepRecord * cap)()
        used = C.c_int64()
        n1 = L.lobo_run(h, days[b][0], L_A, -1, recs, cap, C.byref(used))
        assert L.lobo_is_terminal(h) == 1
        L.lobo_handle_terminal(h, 1)
        L.lobo_reset(h)
        recs2 = (abi.StepRecord * cap)()
        n2 = L.lobo_run(h, days[n_envs + b][0], 300, -1, recs2, cap, C.byref(used))
        got, _k = m.records(b)
        assert len(got) == n1 + n2 and n1 > 50 and n2 > 20, (b, len(got), n1, n2)
        for i in range(n1):
            assert not abi.record_fields_equal(got[i], recs[i]), (b, i)
        for i in range(n2):
            bad = abi.record_fields_equal(got[n1 + i], recs2[i])
            assert not bad, (b, i, bad)
        so = abi.EnvStats()
        L.lobo_stats(h, C.byref(so))
        assert bytes(st[b]) == bytes(so), b
        assert bytes(m.theta(b)) == bytes((C.c_double * cfg.memory_size).from_address(C.addressof(L.lobo_theta(h, 0).contents)))
        L.lobo_destroy(h)
    m.close()


def test_shared_policy_on_tape_equals_stream(rlm):
    from rl_markets_b200 import config
    ing = _ingested()
    B = 4
    y = config.example_dict(**{"learning.memory_size": 8192, "learning.algorithm": "q_learn"})
    synth = None
    out = []
    for source in (abi.SOURCE_STREAM, abi.SOURCE_TAPE):
        cfg = config.from_dict(y, n_envs=B, flow_seed=5, shared_policy=True, source=source)
        cfg.record_envs, cfg.record_cap = B, 1000
        if synth is None:
            synth = lib.flow_generate(cfg.flow, 3, 0, 1200)
        days = [(ing[0][1], ing[0][2]), (synth, 1200), (ing[1][1], ing[1][2])]
        per_env = [days[b % 3] for b in range(B)]
        T = min(n for _a, n in per_env)
        m = rlm.BatchedMarket(cfg)
        if source == abi.SOURCE_STREAM:
            m.load_ticks(_wide(per_env, T), T)
        else:
            buf, offs = _library(days)
            m.load_days(buf, offs)
        m.run_ticks(301)
        m.run_ticks(T - 301)
        m.sync()
        out.append(m)
    _assert_same(out[0], out[1], B, policies=[0])
    assert out[1].tape_pos() == [T] * B
    for m in out:
        m.close()


@pytest.mark.parametrize("ci", [0, 1])
def test_serial_driver_on_a_csv_pair_matches_the_fused_tape_path(rlm, ci):
    """examples/serial_driver --md --tas: serial.cpp's loop through the facade (Intraday::LoadData(ticker, md, tas) +
    RunEpisode, two episodes) leaves exactly the theta of rlm_run_ticks on the same pair."""
    assert os.path.exists(DRIVER), "examples/serial_driver is built by __graft_entry__.build()"
    case, msgs, n = _ingested()[ci]
    md, tas = G.ingest_paths(case)
    M, episodes = case["M"], 2
    with tempfile.TemporaryDirectory() as d:
        thp = os.path.join(d, "theta.bin")
        out = subprocess.check_output([DRIVER, "--md", md, "--tas", tas, "--episodes", str(episodes), "--algo", case["algo"],
                                       "--memory-size", str(M), "--env", str(case["env"]), "--theta", thp]).decode()
        raw = open(thp, "rb").read()
    eps = [json.loads(l) for l in out.strip().splitlines()]
    assert len(eps) == episodes and eps[0]["steps"] == case["n_records"], eps
    L = rlm.load()
    cfg = abi.Config()
    rlm.check(L.rlm_config_default(C.byref(cfg)))
    cfg.algorithm = abi.ALGO[case["algo"]]
    cfg.memory_size = M
    cfg.env_index0 = case["env"]
    cfg.source = abi.SOURCE_TAPE
    m = rlm.BatchedMarket(cfg)
    m.load_days(msgs, [0, n])
    for ep in range(episodes):
        m.run_ticks(n + 7)
        m.sync()
        st = m.stats(0, 1)[0]
        assert st.steps == eps[ep]["steps"] and st.episode_pnl == eps[ep]["pnl"] and st.episode_reward == eps[ep]["reward"]
        assert m.tape_pos() == [n]
        m.handle_terminal(ep)
        if ep + 1 < episodes:
            m.reset()
    assert bytes(m.theta(0, 0)) == raw
    m.close()


def test_tape_errors(rlm, monkeypatch):
    from rl_markets_b200 import config
    y = config.example_dict(**{"learning.memory_size": 4096, "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=2, source=abi.SOURCE_TAPE)
    m = rlm.BatchedMarket(cfg)
    L = rlm.load()

    def code(fn, *a):
        with pytest.raises(rlm.RlmError) as ei:
            fn(*a)
        return ei.value.code

    assert code(m.run_ticks, 10) == abi.RLM_ERR_INVALID_ARGUMENT  # no library yet
    msgs = lib.flow_generate(cfg.flow, 0, 0, 30)
    assert code(m.load_days, msgs, [0, 20, 10, 30]) == abi.RLM_ERR_INVALID_ARGUMENT  # offsets go backwards
    assert code(m.load_days, msgs, [5, 30]) == abi.RLM_ERR_INVALID_ARGUMENT
    m.load_days(msgs, [0, 10, 30])
    assert code(m.assign_days, [0, 2]) == abi.RLM_ERR_INVALID_ARGUMENT  # day 2 does not exist
    assert code(m.assign_days, [-1]) == abi.RLM_ERR_INVALID_ARGUMENT
    assert code(m.assign_days, [0, 1], 1) == abi.RLM_ERR_INVALID_ARGUMENT  # env range
    assert code(m.load_ticks, _wide([(msgs, 30)] * 2, 30), 30) == abi.RLM_ERR_INVALID_ARGUMENT
    assert code(m.new_env, abi.FlowParams.from_buffer_copy(bytes(cfg.flow))) == abi.RLM_ERR_INVALID_ARGUMENT
    m.new_env(None)
    m.assign_days([1, 0])
    m.run_ticks(25)
    m.sync()
    assert m.tape_pos() == [20, 10]
    m.reset()
    assert m.tape_pos() == [0, 0]
    m.close()
    for engine in ("F", "f", "p"):
        monkeypatch.setenv("RLM_ENGINE", engine)
        with pytest.raises(rlm.RlmError) as ei:
            rlm.BatchedMarket(cfg)
        assert ei.value.code == abi.RLM_ERR_UNSUPPORTED, engine
    monkeypatch.delenv("RLM_ENGINE")
    assert L.rlm_load_days(None, None, None, 1) == abi.RLM_ERR_INVALID_ARGUMENT


def test_day_library_loads(rlm):
    """ingest.day_library -> BatchedMarket.load_days on the golden pairs: env b replays pair b % 2 to its end."""
    samples = [("AAL.L",) + G.ingest_paths(c) for c in G.ingest_manifest()]
    msgs, offs = ingest.day_library(samples)
    case = G.ingest_manifest()[0]
    cfg = G.case_config(case, n_envs=3, source=abi.SOURCE_TAPE)
    m = rlm.BatchedMarket(cfg)
    m.load_days(msgs, offs)
    m.run_ticks(offs[-1])
    m.sync()
    assert m.tape_pos() == [offs[1], offs[2] - offs[1], offs[1]]
    m.close()
