"""Checkpoints (rlm_save / rlm_load): a run saved at any point between two calls and loaded into a fresh handle of the
same config continues bit for bit as the run that was never interrupted.

Run A: ops before, save, ops after.  Run B: a fresh handle (the same day library on the tape source), load, the ops after.
Everything observable is compared bitwise: every weight table, occupancy, rlm_env_stats, counters, state, reward,
actions, rho, records, tape positions, model_log rows and Policy::descr.  Then: resuming under other engines, save ->
load -> save giving the same bytes, the packed size of every table, and rejections that leave a handle untouched."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

from rl_markets_b200 import abi, config, lib

pytestmark = pytest.mark.gpu

B = 64
M = 4096
SEC = struct.Struct("<IIQQQ")  # one section table entry: id, table, offset, bytes, count
THETA, THETA_B, DTHETA = 64, 65, 66


def _cfg(algo="q_learn", policy="epsilon_greedy", random_init=False, source=abi.SOURCE_GENERATOR, shared=False, n_envs=B, mem=M,
         n_actions=None):
    over = {"learning.memory_size": mem, "learning.algorithm": algo, "policy.type": policy, "learning.random_init": random_init}
    if n_actions:
        over["learning.n_actions"] = n_actions
    cfg = config.from_dict(config.example_dict(**over), n_envs=n_envs, flow_seed=7, source=source, shared_policy=shared, env_index0=3)
    cfg.record_envs, cfg.record_cap = 4, 4000
    return cfg


def _library(cfg, n_days=3, ticks=(2200, 1700, 2600)):
    """synthetic days of the config's flow, one after the other"""
    offs, parts = [0], []
    for d in range(n_days):
        parts.append(lib.flow_generate(cfg.flow, 100 + d, 0, ticks[d]))
        offs.append(offs[-1] + ticks[d])
    buf = (abi.TickMsg * offs[-1])()
    for p, o in zip(parts, offs):
        C.memmove(C.addressof(buf) + o * C.sizeof(abi.TickMsg), p, C.sizeof(p))
    return buf, offs


def _stream_chunk(cfg, t0, n):
    """msgs[t][env] of ticks t0 .. t0+n-1 of every env's synthetic flow"""
    per = [lib.flow_generate(cfg.flow, cfg.env_index0 + b, t0, n) for b in range(cfg.n_envs)]
    wide = (abi.TickMsg * (n * cfg.n_envs))()
    for b, a in enumerate(per):
        for t in range(n):
            wide[t * cfg.n_envs + b] = a[t]
    return wide


class Setup:
    """A handle of one case: config, engine switches and (tape) day library, rebuilt identically for run B."""

    def __init__(self, cfg, env=None, library=None, day_markets=False, model_log=0):
        self.cfg, self.env, self.library, self.day_markets, self.model_log = cfg, env or {}, library, day_markets, model_log

    def make(self, monkeypatch, env=None, fresh=False):
        for k in ("RLM_ROUNDS", "RLM_ENV_VARIANT", "RLM_AGENT_VARIANT", "RLM_GRAPHS", "RLM_SUBBATCHES"):
            monkeypatch.delenv(k, raising=False)
        for k, v in (self.env if env is None else env).items():
            monkeypatch.setenv(k, v)
        cfg = abi.Config.from_buffer_copy(bytes(self.cfg))
        m = lib.BatchedMarket(cfg)
        if self.library is not None:
            buf, offs = self.library
            m.load_days(buf, offs)
            m.assign_days([(3 * b + 1) % (len(offs) - 1) for b in range(cfg.n_envs)])
            if self.day_markets:
                markets = [config.config_market(cfg), config.market("AAL.L")]
                markets[1].close_ms -= 2 * 3600000  # the second market closes two hours earlier
                m.set_day_markets(markets, [b % 2 for b in range(len(offs) - 1)])
            m.reset()
        if self.model_log and fresh:
            m.set_model_log(self.model_log)
        return m


def _observe(m, mlog=False):
    cfg = m.cfg
    pol = 1 if cfg.shared_policy else cfg.n_envs
    o = {"theta": [bytes(m.theta(p, t)) for p in range(pol) for t in range(m.n_tables)]}
    if not cfg.shared_policy:
        o["occ"] = list(m.occupancy())
    c = m.counters()
    o["counters"] = (c.ticks, c.steps, c.sum_traces, c.terminal_envs)
    o["stats"] = bytes(m.stats())
    o["state"], o["reward"], o["actions"], o["rho"] = bytes(m.state()), bytes(m.rewards()), bytes(m.actions()), bytes(m.rho())
    o["records"] = [m.records(b)[0] for b in range(cfg.record_envs)]
    if cfg.source == abi.SOURCE_TAPE:
        o["tape_pos"] = m.tape_pos()
    if mlog:
        o["model_log"] = m.model_log()
    o["descr"] = m.policy_descr()
    return o


INT_FIELDS = ["step", "action", "time_ms", "terminal", "position", "ask_level", "bid_level", "ask_transactions", "bid_transactions",
              "market_buys", "market_sells", "lo_vol_step", "n_traces"]


def _close(x, y):
    return x == y or abs(x - y) <= 1e-5 * max(abs(x), abs(y), 1e-12)


def _assert_same(a, b, tag, shared=False):
    """bitwise; shared=True: a shared policy trained after the load, whose fp64 atomics sum dtheta in a free order (as
    on any shared handle): integer state exact, weights, rewards and TD errors within 1e-5 relative"""
    for k in a:
        if k == "records":
            for e, (ra, rb) in enumerate(zip(a[k], b[k])):
                assert len(ra) == len(rb), (tag, e, len(ra), len(rb))
                for i in range(len(ra)):
                    if shared:
                        for f in INT_FIELDS:
                            assert getattr(ra[i], f) == getattr(rb[i], f), (tag, "env", e, "record", i, f)
                        assert bytes(ra[i].state) == bytes(rb[i].state) and bytes(ra[i].ask) == bytes(rb[i].ask), (tag, e, i)
                        for f in ("delta", "reward", "pnl_step", "ep_reward", "ep_pnl"):
                            assert _close(getattr(ra[i], f), getattr(rb[i], f)), (tag, "env", e, "record", i, f)
                    else:
                        bad = abi.record_fields_equal(ra[i], rb[i])
                        assert not bad, (tag, "env", e, "record", i, bad)
        elif k == "theta":
            assert len(a[k]) == len(b[k])
            for i in range(len(a[k])):
                if shared:
                    np.testing.assert_allclose(np.frombuffer(b[k][i]), np.frombuffer(a[k][i]), rtol=1e-5, atol=1e-12)
                else:
                    assert a[k][i] == b[k][i], (tag, "table", i)
        elif shared and k in ("stats", "reward", "rho"):
            continue  # (the float columns; their integer state is in the records and counters)
        else:
            assert a[k] == b[k], (tag, k)


# ---- the call sequences a save falls between --------------------------------------------------------------------------
def _split_begin(m):
    m.env_step(None)
    m.agent_update()


def _split_steps(m, n):
    for _ in range(n):
        m.env_step(m.act())
        m.agent_update()


def _shared_ticks(m, n):
    for _ in range(n):
        m.shared_tick_accumulate()
        m.apply_dtheta()


def _do(m, ops, memo=None):
    """run the ops; memo carries the actions of an `act` to the `env_step` that applies them, across a save and load"""
    memo = {} if memo is None else memo
    for op in ops:
        name, *arg = op
        if name == "run":
            m.run_ticks(arg[0])
        elif name == "term":
            m.handle_terminal(arg[0])
        elif name == "reset":
            m.reset()
        elif name == "backtest":
            m.go_greedy()
            m.set_mode(abi.MODE_BACKTEST)
        elif name == "train":
            m.set_mode(abi.MODE_TRAIN)
        elif name == "split_begin":
            _split_begin(m)
        elif name == "split":
            _split_steps(m, arg[0])
        elif name == "act":
            memo["actions"] = bytes(m.act())
        elif name == "env_step":
            m.env_step((C.c_int32 * m.cfg.n_envs).from_buffer_copy(memo["actions"]))
        elif name == "update":
            m.agent_update()
        elif name == "accumulate":
            m.shared_tick_accumulate()
        elif name == "apply":
            m.apply_dtheta()
        elif name == "shared":
            _shared_ticks(m, arg[0])
        elif name == "stream":
            t0, n = arg
            m.load_ticks(_stream_chunk(m.cfg, t0, n), n)
        else:
            raise ValueError(name)
    m.sync()


MID = ([("run", 300)], [("run", 137), ("run", 260)])
WARMUP = ([("run", 6)], [("run", 300)])
EPISODE = ([("run", 350), ("term", 1)], [("reset",), ("run", 300), ("term", 2), ("reset",), ("run", 200)])
BACKTEST = ([("run", 300), ("term", 1), ("reset",), ("backtest",), ("run", 150)], [("run", 200), ("train",), ("run", 100)])
SPLIT_ACT = ([("split_begin",), ("split", 40), ("act",)], [("env_step",), ("update",), ("split", 30), ("run", 150)])
SPLIT_STEP = ([("split_begin",), ("split", 40), ("act",), ("env_step",)], [("update",), ("split", 30), ("run", 150)])
SHARED = ([("shared", 120), ("accumulate",)], [("apply",), ("shared", 80), ("run", 140)])
ROUNDS = {"RLM_ROUNDS": "1"}
TICK_SYNC = {"RLM_ROUNDS": "0"}
THREAD = {"RLM_ENV_VARIANT": "1"}


def _cases():
    c = []
    for algo in abi.ALGO:
        c.append(("%s-mid" % algo, lambda a=algo: Setup(_cfg(a)), MID))
    for pol in ("boltzmann", "random", "greedy"):
        c.append(("sarsa-%s" % pol, lambda p=pol: Setup(_cfg("sarsa", p)), MID))
    c += [
        ("random_init-q", lambda: Setup(_cfg("q_learn", random_init=True)), EPISODE),
        ("random_init-double", lambda: Setup(_cfg("double_q_learn", random_init=True)), MID),
        ("warmup", lambda: Setup(_cfg("double_q_learn")), WARMUP),
        ("episode", lambda: Setup(_cfg("double_r_learn")), EPISODE),
        ("backtest", lambda: Setup(_cfg("double_q_learn")), BACKTEST),
        ("split-act", lambda: Setup(_cfg("q_learn")), SPLIT_ACT),
        ("split-env-step", lambda: Setup(_cfg("online_r_learn")), SPLIT_STEP),
        ("rounds", lambda: Setup(_cfg("double_q_learn"), ROUNDS), MID),
        ("tick-sync", lambda: Setup(_cfg("sarsa"), TICK_SYNC), EPISODE),
        ("thread-per-env", lambda: Setup(_cfg("q_learn"), THREAD), MID),
        ("model-log", lambda: Setup(_cfg("q_learn"), ROUNDS, model_log=8), ([("run", 3000)], [("run", 3000)])),
        ("tape", lambda: Setup(_cfg(source=abi.SOURCE_TAPE), ROUNDS, library=_library(_cfg())), EPISODE),
        ("tape-day-markets", lambda: Setup(_cfg("double_q_learn", source=abi.SOURCE_TAPE), library=_library(_cfg()), day_markets=True,
                                           model_log=4), ([("run", 900)], [("run", 900), ("term", 1), ("reset",), ("run", 400)])),
        ("tape-split", lambda: Setup(_cfg(source=abi.SOURCE_TAPE), library=_library(_cfg())), SPLIT_STEP),
        ("tape-thread", lambda: Setup(_cfg("sarsa", source=abi.SOURCE_TAPE), THREAD, library=_library(_cfg())), BACKTEST),
        ("stream", lambda: Setup(_cfg(source=abi.SOURCE_STREAM)), ([("stream", 0, 300), ("run", 300)], [("stream", 300, 250), ("run", 250)])),
        ("shared", lambda: Setup(_cfg("q_learn", shared=True)), SHARED),
        ("shared-double", lambda: Setup(_cfg("double_q_learn", shared=True), THREAD), SHARED),
        ("shared-backtest", lambda: Setup(_cfg("sarsa", shared=True)), BACKTEST),
        ("shared-tape", lambda: Setup(_cfg("q_learn", source=abi.SOURCE_TAPE, shared=True), library=_library(_cfg())), SHARED),
        ("shared-stream", lambda: Setup(_cfg("q_learn", source=abi.SOURCE_STREAM, shared=True)),
         ([("stream", 0, 200), ("shared", 200)], [("stream", 200, 150), ("run", 150)])),
    ]
    return c


CASES = _cases()


@pytest.mark.parametrize("name,make,ops", CASES, ids=[c[0] for c in CASES])
def test_resume_equals_uninterrupted(rlm, monkeypatch, tmp_path, name, make, ops):
    setup = make()
    before, after = ops
    path = str(tmp_path / "ck.rlm")
    memo = {}
    a = setup.make(monkeypatch, fresh=True)
    _do(a, before, memo)
    a.save(path)
    _do(a, after, dict(memo))
    want = _observe(a, setup.model_log > 0)
    a.close()
    b = setup.make(monkeypatch)
    b.load(path)
    _do(b, after, dict(memo))
    got = _observe(b, setup.model_log > 0)
    b.close()
    _assert_same(want, got, name, shared=bool(setup.cfg.shared_policy))
    assert want["counters"][1] > 0


@pytest.mark.parametrize("env", [TICK_SYNC, THREAD, {"RLM_GRAPHS": "0", "RLM_ROUNDS": "0"}], ids=["tick-sync", "thread", "no-graphs"])
def test_resume_across_engines(rlm, monkeypatch, tmp_path, env):
    """saved under the round-paced engine, continued under another: the same results"""
    setup = Setup(_cfg("double_q_learn", source=abi.SOURCE_TAPE), ROUNDS, library=_library(_cfg()), model_log=4)
    path = str(tmp_path / "ck.rlm")
    after = [("run", 700), ("term", 1), ("reset",), ("run", 500)]
    a = setup.make(monkeypatch, fresh=True)
    _do(a, [("run", 800)])
    a.save(path)
    _do(a, after)
    want = _observe(a, True)
    b = setup.make(monkeypatch, env=env)
    b.load(path)
    _do(b, after)
    _assert_same(want, _observe(b, True), str(env))


def _sections(path):
    data = open(path, "rb").read()
    n_sec, header_bytes = struct.unpack_from("<I", data, 12)[0], struct.unpack_from("<I", data, 24)[0]
    first = header_bytes - n_sec * SEC.size
    return data, [SEC.unpack_from(data, first + i * SEC.size) for i in range(n_sec)]


@pytest.mark.parametrize("case", ["tape-day-markets", "shared", "split-env-step"])
def test_round_trip_is_byte_identical(rlm, monkeypatch, tmp_path, case):
    _name, make, (before, _after) = next(c for c in CASES if c[0] == case)
    setup = make()
    a = setup.make(monkeypatch, fresh=True)
    _do(a, before)
    p1, p2 = str(tmp_path / "a.rlm"), str(tmp_path / "b.rlm")
    a.save(p1)
    b = setup.make(monkeypatch)
    b.load(p1)
    b.save(p2)
    assert open(p1, "rb").read() == open(p2, "rb").read()


def _nnz(buf):
    raw = bytes(buf)
    return sum(1 for i in range(0, len(raw), 8) if raw[i:i + 8] != b"\0" * 8)


def test_packed_size_and_special_words(rlm, monkeypatch, tmp_path):
    """file = header + raw sections + per table M/8 + 8 nnz, nnz counting every word that is not +0.0 bitwise; -0.0, NaN
    payloads, a dense random-init table and an empty table come back exact"""
    cfg = _cfg("double_q_learn", random_init=True, n_envs=8)
    m = lib.BatchedMarket(cfg)
    m.run_ticks(300)
    special = (C.c_double * M)()
    words = (C.c_uint64 * M).from_buffer(special)
    for i in range(0, M, 7):
        words[i] = 0x8000000000000000  # -0.0
    for i in range(3, M, 11):
        words[i] = 0x7FF80000DEADBEEF  # a quiet NaN with a payload
    words[5] = 0xFFF0000000000001  # a signalling NaN
    m.write_theta(special, policy=1)
    m.write_theta((C.c_double * M)(), policy=2, table=1)  # empty
    path = str(tmp_path / "ck.rlm")
    m.save(path)
    data, secs = _sections(path)
    header_bytes = struct.unpack_from("<I", data, 24)[0]
    assert len(data) == header_bytes + sum(s[3] for s in secs)
    tables = [s for s in secs if s[0] in (THETA, THETA_B)]
    assert len(tables) == 2 * cfg.n_envs
    nnz = {}
    for sid, table, _off, nbytes, count in tables:
        k = nnz[(sid, table)] = _nnz(m.theta(table, sid - THETA))
        assert count == k and nbytes == M // 8 + 8 * k, (sid, table, count, k)
    assert nnz[(THETA, 0)] == M and nnz[(THETA_B, 2)] == 0 and nnz[(THETA, 1)] == _nnz(special)
    n = lib.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
    n.load(path)
    for p in range(cfg.n_envs):
        for t in range(2):
            assert bytes(n.theta(p, t)) == bytes(m.theta(p, t)), (p, t)
    assert bytes(n.theta(1)) == bytes(special)


# ---- rejections ------------------------------------------------------------------------------------------------------
def _code(fn, *a):
    with pytest.raises(lib.RlmError) as ei:
        fn(*a)
    return ei.value.code


def test_rejections_leave_the_handle_untouched(rlm, monkeypatch, tmp_path):
    setup = Setup(_cfg("double_q_learn", source=abi.SOURCE_TAPE), library=_library(_cfg()))
    a = setup.make(monkeypatch)
    _do(a, [("run", 400)])
    path = str(tmp_path / "ck.rlm")
    a.save(path)
    data, secs = _sections(path)
    bad = []
    trunc = str(tmp_path / "trunc.rlm")
    open(trunc, "wb").write(data[:len(data) - 9])
    bad.append(("truncated", trunc, setup))
    sec = next(s for s in secs if s[0] == THETA and s[4] not in (0, M))
    flip = bytearray(data)
    flip[sec[2] + 3] ^= 0x10  # one bit of a packed bitmap
    p = str(tmp_path / "flip.rlm")
    open(p, "wb").write(bytes(flip))
    bad.append(("flipped bitmap bit", p, setup))
    magic = bytearray(data)
    magic[0] ^= 1
    p = str(tmp_path / "magic.rlm")
    open(p, "wb").write(bytes(magic))
    bad.append(("magic", p, setup))
    bad.append(("missing", str(tmp_path / "none.rlm"), setup))
    for what, kw in (("memory_size", {"mem": 2 * M}), ("n_envs", {"n_envs": B // 2}), ("algorithm", {"algo": "q_learn"}),
                     ("n_actions", {"n_actions": 7})):
        args = dict({"algo": "double_q_learn", "source": abi.SOURCE_TAPE}, **kw)
        bad.append((what, path, Setup(_cfg(**args), library=_library(_cfg()))))
    buf, offs = _library(_cfg())
    bad.append(("other offsets", path, Setup(setup.cfg, library=(buf, [0, offs[1] + 5] + offs[2:]))))
    changed = (abi.TickMsg * len(buf)).from_buffer_copy(bytes(buf))
    changed[offs[1] + 17].ask_vol[2] += 1
    bad.append(("one changed message", path, Setup(setup.cfg, library=(changed, offs))))
    for what, p, s in bad:
        m = s.make(monkeypatch)
        _do(m, [("run", 50)])
        assert _code(m.load, p) == abi.RLM_ERR_INVALID_ARGUMENT, what
        ref = s.make(monkeypatch)
        _do(ref, [("run", 50)])
        ops = [("run", 250), ("term", 1), ("reset",), ("run", 150)]
        _do(ref, ops)
        _do(m, ops)
        _assert_same(_observe(ref), _observe(m), what)
        m.close()
        ref.close()


def test_stream_with_unconsumed_ticks_is_refused(rlm, monkeypatch, tmp_path):
    setup = Setup(_cfg(source=abi.SOURCE_STREAM))
    m = setup.make(monkeypatch)
    _do(m, [("stream", 0, 300), ("run", 200)])
    path = str(tmp_path / "ck.rlm")
    assert _code(m.save, path) == abi.RLM_ERR_INVALID_ARGUMENT
    assert not os.path.exists(path)
    _do(m, [("run", 100)])
    ref = setup.make(monkeypatch)
    _do(ref, [("stream", 0, 300), ("run", 200), ("run", 100)])
    _assert_same(_observe(ref), _observe(m), "refused save")
    m.save(path)  # every uploaded tick consumed


def test_unsupported_engine(rlm, monkeypatch, tmp_path):
    monkeypatch.setenv("RLM_ENGINE", "p")
    m = lib.BatchedMarket(_cfg(source=abi.SOURCE_STREAM))
    assert _code(m.save, str(tmp_path / "ck.rlm")) == abi.RLM_ERR_UNSUPPORTED
    assert _code(m.load, str(tmp_path / "ck.rlm")) == abi.RLM_ERR_UNSUPPORTED
