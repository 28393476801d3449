"""Evaluation over several test days on the GPU, as src/main.cpp:216-244 runs it: train until the close, GoGreedy, one
env object for every test day -- rlm_new_env before the first day, then per later day LoadData + Initialise on the same
objects:
  generator  rlm_set_flow + rlm_reset      stream  rlm_reset + rlm_load_ticks      tape  rlm_assign_days + rlm_reset
Every record and rlm_env_stats after each day against the reference's own records (tests/golden/eval_days.json and
digests_ed_*, tools/make_golden.py --eval-days) for env 0 and against the CPU oracle for the other envs; on warp-per-env
and thread-per-env tick kernels, in whole-day calls and in 100-tick calls; and on a shared handle that loaded the trained
table.  The old sequence, rlm_new_env before every day, must differ from the reference on day 2.

Past one resident wave: the evaluation kernel serves at most one resident wave of steps per pass of its grid-stride
loop (SMs x 16 steps, Double-Q SMs x 12, from its __launch_bounds__); 32 768 envs under one shared table of 2^22 seeded
random weights, and 20 000 independent envs of 4096 weights each, put most steps into later passes.  Records and stats of
512 envs spread over the batch, the last 64 among them, against the oracle, bitwise."""
import concurrent.futures as cf
import ctypes as C
import functools
import os

import numpy as np
import pytest

import golden_util as G
import test_eval_days as ED
from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu
MSG = C.sizeof(abi.TickMsg)
CAP = 3000
CARRIED = ("n_traces", "trace_hash")  # a handle that loaded the table holds no traces (test_gpu_shared_backtest.py)
SOURCE = {"generator": abi.SOURCE_GENERATOR, "stream": abi.SOURCE_STREAM, "tape": abi.SOURCE_TAPE}


def _cases(source):
    """venue days of another ticker exist on the tape source only (rlm_set_day_markets)"""
    return [c for c in ED.CASES if source == "tape" or all("venue" not in d for d in c["days"])]


def _msgs(c, k, b):
    """messages of env b (global index case env + b) on test day k, k = -1: the training day -> (array, count)"""
    if k < 0:
        from rl_markets_b200 import lib
        return lib.flow_generate(ED.train_config(c).flow, c["env"] + b, 0, c["ticks"]), c["ticks"]
    return ED.day_messages(c["name"], k, None if b == 0 else c["env"] + b)


def _tick_major(per_env):
    """[(msgs, n)] of every env, the same n -> ctypes array laid out [tick][env] (rlm_load_ticks)"""
    n, B = per_env[0][1], len(per_env)
    assert all(p[1] == n for p in per_env)
    out = (abi.TickMsg * (n * B))()
    dst = np.frombuffer(out, dtype=np.uint8).reshape(n, B, MSG)
    for b, (m, _n) in enumerate(per_env):
        dst[:, b, :] = np.frombuffer((C.c_char * (n * MSG)).from_address(C.addressof(m)), dtype=np.uint8).reshape(n, MSG)
    return out


class Evaluation:
    """One handle through a case: training (or a loaded table), then every test day through `source`'s sequence.
    fresh=True: rlm_new_env before every day, the sequence that computes one reference process per test day."""

    def __init__(self, rlm, c, source, n_envs, chunk=None, theta=None, fresh=False):
        self.c, self.source, self.B, self.chunk = c, source, n_envs, chunk
        cfg = ED.train_config(c, n_envs=n_envs, env_index0=c["env"], source=SOURCE[source], shared_policy=theta is not None)
        cfg.record_envs, cfg.record_cap = n_envs, CAP
        self.m = m = rlm.BatchedMarket(cfg)
        n_days = len(c["days"])
        if source == "tape":  # library slot s (0: training, 1 + k: test day k) of env b is day s * B + b
            per = [_msgs(c, s - 1, b) for s in range(1 + n_days) for b in range(n_envs)]
            offs = [0]
            for _a, n in per:
                offs.append(offs[-1] + n)
            self._lib = buf = (abi.TickMsg * offs[-1])()
            for (a, n), o in zip(per, offs):
                C.memmove(C.addressof(buf) + o * MSG, a, n * MSG)
            m.load_days(buf, offs)
            if any("ticker" in d for d in c["days"]):
                markets = [config.config_market(cfg)] + [ED.day_market(c, k) or config.config_market(cfg) for k in range(n_days)]
                m.set_day_markets(markets, [s for s in range(1 + n_days) for _b in range(n_envs)])
            self._assign(0)
            m.reset()
        self.train_recs = None
        if theta is None:
            self._feed(-1)
            assert all(s.terminal for s in m.stats())
            self.train_recs = m.records(0)[0]
            m.handle_terminal(0)          # Learner::RunEpisode, serial.cpp:79
        else:
            for k, th in enumerate(theta):
                m.write_theta(th, 0, k)
        m.go_greedy()                     # main.cpp:217
        m.set_mode(abi.MODE_BACKTEST)     # experiment::serial::Backtester
        self.days = []
        for k in range(n_days):
            self._load(k, new=k == 0 or fresh)
            self._feed(k)
            recs = []
            for b in range(n_envs):
                r = m.records(b)[0]
                recs.append(r[self.seen[b]:])
                self.seen[b] = len(r)
            self.days.append((recs, list(m.stats())))

    def _assign(self, slot):
        self.m.assign_days([slot * self.B + b for b in range(self.B)])

    def _load(self, k, new):
        m = self.m
        if new:                           # environment::Intraday<> env(c) (main.cpp:219): records start again
            if self.source == "tape":
                self._assign(1 + k)
            m.new_env(ED.day_flow(self.c, k) if self.source == "generator" else None)
            self.seen = [0] * self.B
        else:                             # LoadData + the next Backtester's Initialise on the same env objects
            if self.source == "generator":
                m.set_flow(ED.day_flow(self.c, k))
            elif self.source == "tape":
                self._assign(1 + k)
            m.reset()

    def _feed(self, k):
        """the day's ticks (tape: its longest day's messages) in calls of `chunk` ticks; stream: loaded chunk by chunk"""
        per = [_msgs(self.c, k, b) for b in range(self.B)]
        n = max(p[1] for p in per)
        tm = _tick_major(per) if self.source == "stream" else None
        step = self.chunk or n
        for t in range(0, n, step):
            cnt = min(step, n - t)
            if tm is not None:
                self.m.load_ticks(C.addressof(tm) + t * self.B * MSG, cnt)
            self.m.run_ticks(cnt)
        self.m.sync()

    def close(self):
        self.m.close()


@functools.lru_cache(maxsize=None)
def _oracle(name, b, theta=None):
    """the oracle's carried evaluation of env b (global index case env + b): trained as the case trains, or under the
    loaded tables `theta`"""
    import oracle_lib
    c = ED.case(name)
    return ED.oracle_evaluation(oracle_lib, c, env_index=c["env"] + b, theta=theta)


def _trained_tables(rlm, c):
    """the table(s) a one-env handle trains on the case's training day (the device's, bitwise the reference's: the
    training records of test_every_day_matches_the_reference)"""
    cfg = ED.train_config(c, n_envs=1, env_index0=c["env"])
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(c["ticks"])
    m.sync()
    assert m.stats()[0].terminal
    m.handle_terminal(0)
    out = tuple(bytes(m.theta(0, k)) for k in range(2 if cfg.algorithm in (abi.ALGO["double_q_learn"], abi.ALGO["double_r_learn"]) else 1))
    m.close()
    return out


def _assert_records(got, want, tag, skip=()):
    assert len(got) == len(want), (tag, len(got), len(want))
    for i in range(len(got)):
        bad = abi.record_fields_equal(got[i], want[i], skip=skip)
        assert not bad, (tag, i, G.describe_diff(got[i], want[i], bad))


def _check(ev, skip=(), theta=None):
    c = ev.c
    if ev.train_recs is not None:
        ED.assert_digests(ev.train_recs, c["name"] + "_train", (c["name"], "train"))
    for k, (recs, stats) in enumerate(ev.days):
        tag = (c["name"], ev.source, "day", k)
        if not skip:
            ED.assert_digests(recs[0], "%s_day%d" % (c["name"], k), tag)
            assert ED.day_stats_match(stats[0], c["days"][k]["summary"]), tag
        for b in range(0 if skip else 1, ev.B):
            want, st = _oracle(c["name"], b, theta if b > 0 else None)[1][k]
            _assert_records(recs[b], want, tag + ("env", b), skip)
            assert bytes(stats[b]) == bytes(st), tag + ("env", b)


@pytest.mark.parametrize("chunk", [None, 100])  # whole-day calls, 100-tick calls
@pytest.mark.parametrize("variant", [0, 1])     # warp-per-env and thread-per-env tick kernels
@pytest.mark.parametrize("source", ["generator", "stream", "tape"])
def test_every_day_matches_the_reference(rlm, monkeypatch, source, variant, chunk):
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    for c in _cases(source):
        ev = Evaluation(rlm, c, source, n_envs=3, chunk=chunk)
        _check(ev)
        ev.close()


@pytest.mark.parametrize("source", ["generator", "stream", "tape"])
def test_a_shared_handle_that_loaded_the_trained_table(rlm, source):
    """env 0 is the reference process that trained the table; envs 1-2 are processes that loaded it.  (Shared policies
    exist for q_learn, sarsa and double_q_learn with an even memory_size.)"""
    for c in _cases(source):
        if c["algo"] not in ("q_learn", "sarsa", "double_q_learn") or c["M"] % 2:
            continue
        theta = _trained_tables(rlm, c)
        ev = Evaluation(rlm, c, source, n_envs=3, theta=theta)
        _check(ev, skip=CARRIED, theta=theta)
        ev.close()


def test_a_new_env_object_per_day_differs_from_the_reference(rlm):
    """rlm_new_env before every day zeroes what main.cpp's env object carries: day 2 cannot match the reference."""
    for c in ED.CASES:
        ev = Evaluation(rlm, c, "tape", n_envs=1, fresh=True)
        ED.assert_digests(ev.days[0][0][0], c["name"] + "_day0", (c["name"], "day 0"))
        recs = ev.days[1][0][0]
        gold = G.digests(c["name"] + "_day1")
        assert len(recs) != len(gold) or any(G.record_digest(r) != g for r, g in zip(recs, gold)), c["name"]
        ev.close()


@pytest.mark.parametrize("source", ["stream", "tape"])
def test_set_flow_is_for_the_generator_source(rlm, source):
    """the other sources change days with rlm_load_ticks / rlm_assign_days; the handle is left as it was"""
    c = ED.CASES[0]
    m = rlm.BatchedMarket(ED.train_config(c, n_envs=2, source=SOURCE[source]))
    before = bytes(m.cfg.flow)
    with pytest.raises(rlm.RlmError) as ei:
        m.set_flow(ED.day_flow(c, 0))
    assert ei.value.code == abi.RLM_ERR_INVALID_ARGUMENT
    assert ("rlm_assign_days" if source == "tape" else "rlm_load_ticks") in str(ei.value)
    assert bytes(m.cfg.flow) == before
    m.close()


# ---- past one resident wave -----------------------------------------------------------------------------------------
WAVE_T0_MS = 12 * 3600000  # 1 000 ticks of 250 ms from noon: the whole run is inside trading hours
WAVE_TICKS = 1000


def _spread(B, n=512, last=64):
    return sorted(set(np.linspace(0, B - last - 1, n - last).astype(int).tolist()) | set(range(B - last, B)))


def _random_table(seed, M):
    th = np.random.default_rng(seed).uniform(-1.0, 1.0, M)
    th[th == 0.0] = 0.5  # every weight nonzero
    return th


def _resident_wave(double):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * (12 if double else 16)


def _wave_run(rlm, cfg, tables):
    """load tables ((policy, table), weights) one after the other, GoGreedy, backtest, WAVE_TICKS ticks -> (handle, steps per eval launch)"""
    cfg.record_envs, cfg.record_cap = cfg.n_envs, 600
    m = rlm.BatchedMarket(cfg)
    for (p, k), th in tables:
        m.write_theta(th, p, k)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    flow = config.from_dict(config.example_dict(), flow_seed=cfg.flow.seed).flow
    flow.t0_ms = WAVE_T0_MS
    m.new_env(flow)
    m.set_profiling(True)
    s0 = m.counters().steps
    for _ in range(WAVE_TICKS // 250):
        m.run_ticks(250)
    m.sync()
    launches = m.kernel_times()["agent_launches"]
    return m, (m.counters().steps - s0) / max(launches, 1)


def _wave_oracle(m, envs, theta_of):
    """records and stats of each env in `envs` from the oracle (one reference process that loaded its table), compared"""
    import oracle_lib
    from rl_markets_b200 import lib
    import test_gpu_shared_backtest as SB
    cfg = m.cfg
    stats = m.stats()

    def one(b):
        msgs = lib.flow_generate(cfg.flow, cfg.env_index0 + b, 0, WAVE_TICKS)
        want, st, _k = SB._oracle_eval(oracle_lib, cfg, b, theta_of(b), msgs, WAVE_TICKS)
        return b, want, st

    n_steps = 0
    with cf.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        for b, want, st in ex.map(one, envs):
            got, _k = m.records(b)
            assert len(got) > 50, (b, len(got))
            _assert_records(got, want, ("env", b))
            assert bytes(stats[b]) == bytes(st), b
            n_steps += len(got)
    return n_steps


@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_shared_table_past_one_resident_wave(rlm, algo):
    B, M = 32768, 1 << 22
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
    cfg = config.from_dict(y, n_envs=B, shared_policy=True, flow_seed=4242, env_index0=3)
    double = algo == "double_q_learn"
    tables = [_random_table(17 + k, M) for k in range(2 if double else 1)]
    m, per_launch = _wave_run(rlm, cfg, [((0, k), t) for k, t in enumerate(tables)])
    assert per_launch > _resident_wave(double), (per_launch, _resident_wave(double))
    _wave_oracle(m, _spread(B), lambda b: tables)
    m.close()


def test_independent_tables_past_one_resident_wave(rlm):
    """20 000 envs x 4096 weights: policy * memory_size passes 16 384 * 4096; each env its own seeded table"""
    B, M = 20000, 4096
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=B, flow_seed=4343, env_index0=5)
    m, per_launch = _wave_run(rlm, cfg, (((b, 0), _random_table(100000 + b, M)) for b in range(B)))
    assert per_launch > _resident_wave(False), (per_launch, _resident_wave(False))
    _wave_oracle(m, _spread(B), lambda b: [_random_table(100000 + b, M)])
    m.close()
