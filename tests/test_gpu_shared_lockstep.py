"""Shared-policy training on the device, tick by tick, against the batch oracle -- bitwise everywhere but dtheta.

The only freedom of the synchronous algorithm is the order of each weight's sum in dtheta (DESIGN section 4).  Each tick
here takes that freedom away: the device accumulates, the oracle accumulates the same messages with its contribution log
on, the device's dtheta is checked against the exact sum of the logged contributions (tests/shared_lockstep.py: bitwise
where a weight has one or two of them, within the bound of any summation order above), and the device's dtheta is then
copied into the oracle before both apply it.  From there theta is the same on both sides every tick, so every record
field, theta, the statistics and the counters are compared bitwise at any scale.

With one env there is nothing to reorder: a shared handle of one env is the reference's Learner, trace_hash aside (a
shared record hashes theta_t, before the apply).  Those cases run through rlm_run_ticks' own accumulate / apply loop.
"""
import ctypes as C
import os

import numpy as np
import pytest

import golden_util as G
import shared_lockstep as S
from rl_markets_b200 import abi, config
from test_shared_lockstep_cpu import run_batch_one, shared_cases

pytestmark = pytest.mark.gpu

MSG = C.sizeof(abi.TickMsg)
# learner and tick kernels a shared handle can run; every switch is read by rlm_create
LEARNERS = [("one_warp", {}), ("agent3", {"RLM_AGENT_VARIANT": "3"}), ("agent1", {"RLM_AGENT_VARIANT": "1"}),
            ("env1", {"RLM_ENV_VARIANT": "1"})]
# fields that depend on the mm_exp reward: exp() is glibc's in the reference and CUDA's here (DESIGN section 4)
MM_EXP_CHAIN = {"reward", "ep_reward", "delta", "trace_hash"}


def _setenv(monkeypatch, env):
    for k, v in env.items():
        monkeypatch.setenv(k, v)


# ---- one env: the reference's algorithm

_ONE = {}


def _batch_one(oracle, case):
    if case["name"] not in _ONE:
        _ONE[case["name"]] = run_batch_one(oracle, case)
    return _ONE[case["name"]]


@pytest.mark.parametrize("learner,env", LEARNERS, ids=[l for l, _e in LEARNERS])
@pytest.mark.parametrize("name", [c["name"] for c in shared_cases()])
def test_one_env_shared_handle_is_the_reference(rlm, oracle, monkeypatch, name, learner, env):
    """A shared handle of one env (env_index0 = the case's env) driven by rlm_run_ticks: the golden records of the
    reference (every field but trace_hash), and the one-env batch oracle (every field, theta, statistics, counters)."""
    _setenv(monkeypatch, env)
    case = [c for c in shared_cases() if c["name"] == name][0]
    cfg = G.case_config(case, n_envs=1, env_index0=case["env"])
    cfg.shared_policy = 1
    cfg.record_envs, cfg.record_cap = 1, case["ticks"]
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(case["ticks"])
    m.sync()
    recs, _keep = m.records(0)
    o_recs, o_th, o_st, o_steps, o_traces, _k = _batch_one(oracle, case)
    mm_exp = case["yaml"]["reward"]["measure"] == "mm_exp"
    tol = MM_EXP_CHAIN if mm_exp else set()
    gold, _k2 = G.records(name)
    assert len(recs) == len(o_recs) == o_steps >= len(gold) > 100, (name, len(recs), len(o_recs), len(gold))
    for i, r in enumerate(recs):
        for ref, what, skip in ((o_recs[i], "batch oracle", ()), (gold[i] if i < len(gold) else None, "reference", ("trace_hash",))):
            if ref is None:
                continue
            bad = abi.record_fields_equal(r, ref, skip=skip)
            for f in [f for f in bad if f in tol and f != "trace_hash"]:
                x, y = getattr(r, f), getattr(ref, f)
                assert abs(x - y) <= 1e-5 * max(abs(x), abs(y)), (name, i, f, x, y)
            bad = [f for f in bad if f not in tol]
            assert not bad, "%s %s step %d (cuda, %s): %r" % (name, learner, i, what, G.describe_diff(r, ref, bad))
    M = cfg.memory_size
    for t, th in enumerate(o_th):
        got = np.frombuffer(m.theta(0, t), dtype=np.float64)
        if mm_exp:
            np.testing.assert_allclose(got, th, rtol=1e-5, atol=1e-12)
        else:
            assert got.tobytes() == th.tobytes(), (name, learner, t)
    st = m.stats()[0]
    if not mm_exp:
        assert bytes(st) == bytes(o_st), name
    cnt = m.counters()
    assert (cnt.steps, cnt.sum_traces) == (o_steps, o_traces), name
    assert M == len(o_th[0])
    m.close()


@pytest.mark.parametrize("learner,env", LEARNERS, ids=[l for l, _e in LEARNERS])
@pytest.mark.parametrize("name", [c["name"] for c in G.episode_manifest()])
def test_one_env_shared_handle_episodes_are_the_reference(rlm, monkeypatch, name, learner, env):
    """The multi-episode golden cases on a shared handle of one env: rlm_handle_terminal + rlm_reset between episodes,
    every record field but trace_hash against the reference."""
    _setenv(monkeypatch, env)
    case = [c for c in G.episode_manifest() if c["name"] == name][0]
    cfg = G.case_config(case, n_envs=1, env_index0=case["env"])
    cfg.shared_policy = 1
    cfg.flow.t0_ms = case["t0_ms"]
    cfg.record_envs, cfg.record_cap = 1, case["n_records"] + 16
    m = rlm.BatchedMarket(cfg)
    for ep in range(case["episodes"]):
        m.run_ticks(case["ticks"])
        m.sync()
        assert m.stats(0, 1)[0].terminal == 1
        m.handle_terminal(ep)
        m.reset()
    recs, _keep = m.records(0)
    gold, _k = G.records(name)
    assert len(recs) == len(gold) == case["n_records"], (name, len(recs), len(gold))
    for i, g in enumerate(gold):
        bad = abi.record_fields_equal(recs[i], g, skip=("trace_hash",))
        assert not bad, "%s %s step %d (cuda, reference): %r" % (name, learner, i, G.describe_diff(recs[i], g, bad))
    m.close()


# ---- lockstep


class Lockstep:
    """One or two device handles (the halves of the batch, each with its replica of theta) and the batch oracle over
    all of cfg's envs, advanced one tick at a time with the device's dtheta handed to the oracle."""

    def __init__(self, rlm, oracle, cfg, msgs, halves=1, setup=None):
        import torch
        from test_shared_policy_cpu import _oracle_batch
        self.torch = torch
        self.cfg, self.B, self.M = cfg, cfg.n_envs, cfg.memory_size
        self.nt = 2 if cfg.algorithm == abi.ALGO["double_q_learn"] else 1
        self.dense = self.M <= (1 << 16)
        self.msgs = msgs  # numpy uint8 [n_ticks, B, MSG]
        self.cap = cfg.record_cap
        n = self.B // halves
        self.ms = []
        for r in range(halves):
            c = abi.Config.from_buffer_copy(bytes(cfg))
            c.n_envs, c.env_index0 = n, cfg.env_index0 + r * n
            c.record_envs, c.record_cap = min(cfg.record_envs, n), self.cap
            m = rlm.BatchedMarket(c)
            if setup:
                setup(m, r * n, n)
            self.ms.append(m)
        self.stream = None
        if halves > 1:
            self.stream = torch.cuda.Stream()  # (a real stream: 0 would mean "the handle's own stream")
            for m in self.ms:
                m.set_stream(self.stream.cuda_stream)
        self.dth = [m.dtheta_tensor() for m in self.ms]
        L, self.b = _oracle_batch(cfg)
        self.L = S.bind(L)
        L.lobo_batch_log(self.b, 1)
        self.recs = (abi.StepRecord * (self.B * self.cap))()
        self.cnt = (C.c_int32 * self.B)()
        self.o_d = [np.ctypeslib.as_array(L.lobo_batch_dtheta(self.b, t), shape=(self.M,)) for t in range(self.nt)]
        self.o_th = [np.ctypeslib.as_array(L.lobo_batch_theta(self.b, t), shape=(self.M,)) for t in range(self.nt)]
        self.tally = S.Tally()
        self.t = 0

    def _device_dtheta(self):
        """the device's dtheta of this tick (the sum of the halves, which then goes back to both)"""
        torch = self.torch
        if len(self.ms) == 1:
            self.ms[0].sync()
            d = self.dth[0]
        else:
            with torch.cuda.stream(self.stream):
                d = self.dth[0] + self.dth[1]
                for x in self.dth:
                    x.copy_(d)
            self.stream.synchronize()
        if self.dense:
            return d.cpu().numpy()
        idx = torch.nonzero(d).flatten()
        return idx.cpu().numpy().astype(np.int64), d[idx].cpu().numpy()

    def _oracle_dtheta(self, log):
        if self.dense:
            return np.concatenate(self.o_d)
        idx = np.concatenate([np.flatnonzero(v) + t * self.M for t, v in enumerate(self.o_d)])
        return idx, np.concatenate([v[v != 0] for v in self.o_d])

    def device_theta(self, m, t):
        return np.frombuffer(m.theta(0, t), dtype=np.float64).copy()

    def tick(self, probe=False):
        for m in self.ms:
            m.shared_tick_accumulate()
        dev = self._device_dtheta()
        msgs = self.msgs[self.t]
        self.L.lobo_batch_accumulate(self.b, C.cast(msgs.ctypes.data, C.POINTER(abi.TickMsg)), C.addressof(self.recs),
                                     C.addressof(self.cnt), self.cap)
        log = S.log_entries(self.L, self.b)
        r = S.check(log, dev, self.M)
        assert not r["bad"], ("device dtheta", self.t, r["bad"])
        ro = S.check(log, self._oracle_dtheta(log), self.M)
        assert not ro["bad"], ("oracle dtheta", self.t, ro["bad"])
        self.tally.add(r)
        # the device's sum becomes the oracle's
        if self.dense:
            for t in range(self.nt):
                self.o_d[t][:] = dev[t * self.M:(t + 1) * self.M]
        else:
            for t in range(self.nt):
                self.o_d[t][log["feature"][log["table"] == t]] = 0.0
            idx, vals = dev
            for t in range(self.nt):
                sel = (idx // self.M) == t
                self.o_d[t][idx[sel] % self.M] = vals[sel]
        if probe:
            before = [[self.device_theta(m, t) for t in range(self.nt)] for m in self.ms]
            d_full = [self.o_d[t].copy() for t in range(self.nt)]
        self.L.lobo_batch_apply(self.b)
        for m in self.ms:
            m.apply_dtheta()
        if probe:
            for m, th0 in zip(self.ms, before):
                m.sync()
                for t in range(self.nt):
                    got = self.device_theta(m, t)
                    assert got.tobytes() == (th0[t] + d_full[t]).tobytes(), ("apply", self.t, t)
                    assert got.tobytes() == self.o_th[t].tobytes(), ("theta", self.t, t)
            for x in self.dth:
                assert int(self.torch.count_nonzero(x.view(self.torch.int64))) == 0, ("dtheta not cleared", self.t)
        self.t += 1

    def run(self, n_ticks, probes=4):
        at = {int(x) for x in np.linspace(n_ticks // 3, n_ticks - 1, probes)}
        for t in range(n_ticks):
            self.tick(probe=t in at)

    def finish(self, label):
        """every record field, theta, statistics and counters bitwise; returns the tally"""
        n = self.B // len(self.ms)
        steps = traces = 0
        compared = 0
        for r, m in enumerate(self.ms):
            m.sync()
            st = m.stats()
            for i in range(n):
                e = r * n + i
                so = abi.EnvStats()
                self.L.lobo_batch_stats(self.b, e, C.byref(so))
                assert bytes(st[i]) == bytes(so), (label, "stats", e)
                if i < m.cfg.record_envs:
                    got, _keep = m.records(i)
                    assert len(got) == min(self.cnt[e], self.cap), (label, e, len(got), self.cnt[e])
                    for j, g in enumerate(got):
                        o = self.recs[e * self.cap + j]
                        bad = abi.record_fields_equal(g, o)
                        assert not bad, "%s env %d step %d (cuda, oracle): %r" % (label, e, j, G.describe_diff(g, o, bad))
                    compared += len(got)
            for t in range(self.nt):
                assert self.device_theta(m, t).tobytes() == self.o_th[t].tobytes(), (label, "theta", r, t)
            c = m.counters()
            steps += c.steps
            traces += c.sum_traces
        assert steps == self.L.lobo_batch_steps(self.b), (label, steps)
        assert traces == self.L.lobo_batch_sum_traces(self.b), (label, traces)
        self.compared = compared
        return self.tally

    def close(self):
        self.L.lobo_batch_destroy(self.b)
        for m in self.ms:
            m.close()


def _generated(rlm, cfg, n_ticks, env_of=None):
    """[tick, env, MSG] bytes: env b's flow, or day env_of(b) of the flow when given"""
    out = np.empty((n_ticks, cfg.n_envs, MSG), dtype=np.uint8)
    for b in range(cfg.n_envs):
        src = env_of(b) if env_of else cfg.env_index0 + b
        s = rlm.flow_generate(cfg.flow, src, 0, n_ticks)
        out[:, b, :] = np.frombuffer(s, dtype=np.uint8).reshape(n_ticks, MSG)
    return out


def _cfg(algo, M, B, seed=33, cap=None, record_envs=None, source=abi.SOURCE_GENERATOR):
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
    cfg = config.from_dict(y, n_envs=B, shared_policy=True, flow_seed=seed, source=source)
    cfg.record_envs = B if record_envs is None else record_envs
    cfg.record_cap = cap or 600
    return cfg


def _report(label, ls, n_ticks):
    t = ls.tally
    print("\n[lockstep] %s: %d ticks, %d steps compared, %r" % (label, n_ticks, ls.compared, t))


def _lockstep(rlm, oracle, label, cfg, n_ticks, floor, halves=1, msgs=None, setup=None, min_k=3):
    msgs = _generated(rlm, cfg, n_ticks) if msgs is None else msgs
    ls = Lockstep(rlm, oracle, cfg, msgs, halves=halves, setup=setup)
    try:
        ls.run(n_ticks)
        t = ls.finish(label)
        _report(label, ls, n_ticks)
        assert ls.compared > cfg.record_envs * 20, (label, ls.compared)
        assert t.max_k >= min_k, (label, t)
        assert t.fraction >= floor, (label, t)
    finally:
        ls.close()
    return t


ALGOS = ["q_learn", "sarsa", "double_q_learn"]


@pytest.mark.parametrize("learner,env", LEARNERS, ids=[l for l, _e in LEARNERS])
@pytest.mark.parametrize("algo", ALGOS)
def test_lockstep_algorithm_by_learner(rlm, oracle, monkeypatch, algo, learner, env):
    """64 envs, M = 4096, 600 ticks, on each learner and tick kernel a shared handle can run"""
    _setenv(monkeypatch, env)
    _lockstep(rlm, oracle, "%s %s" % (algo, learner), _cfg(algo, 4096, 64), 600, 0.99)


def test_lockstep_two_weights_under_a_thousand_envs(rlm, oracle):
    """M = 2: every stepping env adds into the same two words"""
    _lockstep(rlm, oracle, "M=2 B=1000", _cfg("q_learn", 2, 1000, cap=300), 600, 0.98)


def test_lockstep_modulo_table_on_the_thread_per_env_kernel(rlm, oracle, monkeypatch):
    """M = 2 * 4099 (the modulo path of the tile hash), Double-Q, 257 envs: a partial last warp of the thread-per-env
    tick kernel, and its trailing action-selection pass after rlm_apply_dtheta"""
    monkeypatch.setenv("RLM_ENV_VARIANT", "1")
    _lockstep(rlm, oracle, "M=8198 double_q B=257 env1", _cfg("double_q_learn", 2 * 4099, 257), 600, 0.99)


def _host_available_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_lockstep_c3_table(rlm, oracle):
    """C3's table, M = 2^22, Q-learning, 64 envs; dtheta is fetched as its nonzero entries.  The oracle keeps dense
    traces: 32 MB per env."""
    need = 64 * (40 << 20) + (4 << 30)
    if _host_available_bytes() < need:
        pytest.skip("%.1f GB available on the host, %.1f GB needed" % (_host_available_bytes() / 1e9, need / 1e9))
    _lockstep(rlm, oracle, "M=2^22 B=64", _cfg("q_learn", 1 << 22, 64), 600, 0.97, min_k=2)


def test_lockstep_c3_kernels_by_auto_selection(rlm, oracle):
    """16 385 envs: rlm_create sends a shared batch above 16 384 envs to the three-warp learner (shared handles are never
    staged, rlm_api.cu) and to the thread-per-env tick kernel, with no switch set.  M = 2048, Q-learning, 300 ticks."""
    for k in ("RLM_AGENT_VARIANT", "RLM_ENV_VARIANT", "RLM_STAGED"):
        assert k not in os.environ, k
    B = 16385
    need = B * (600 << 10) + (4 << 30)
    if _host_available_bytes() < need:
        pytest.skip("%.1f GB available on the host, %.1f GB needed" % (_host_available_bytes() / 1e9, need / 1e9))
    _lockstep(rlm, oracle, "C3 auto B=16385", _cfg("q_learn", 2048, B, cap=120, record_envs=1024), 300, 0.97)


def test_lockstep_stream_source(rlm, oracle):
    """The stream source: the oracle's messages uploaded with load_ticks, one tick per accumulate"""
    n_ticks = 600
    cfg = _cfg("q_learn", 4096, 64, seed=77, source=abi.SOURCE_STREAM)
    msgs = _generated(rlm, cfg, n_ticks)

    def setup(m, first, n):
        part = np.ascontiguousarray(msgs[:, first:first + n, :])
        keep = (C.c_uint8 * part.size).from_buffer_copy(part.tobytes())
        m.load_ticks(C.addressof(keep), n_ticks)
        m._keep = keep

    _lockstep(rlm, oracle, "stream", cfg, n_ticks, 0.99, msgs=msgs, setup=setup)


def test_lockstep_tape_source(rlm, oracle):
    """The tape source: five synthetic days for 64 envs (env b replays day b % 5), each longer than the run"""
    n_ticks, n_days, day_len = 600, 5, 700
    cfg = _cfg("sarsa", 4096, 64, seed=55, source=abi.SOURCE_TAPE)
    days = [rlm.flow_generate(cfg.flow, 100 + d, 0, day_len) for d in range(n_days)]
    lib = (abi.TickMsg * (n_days * day_len))()
    for d, a in enumerate(days):
        C.memmove(C.addressof(lib) + d * day_len * MSG, a, day_len * MSG)
    offs = [d * day_len for d in range(n_days + 1)]
    msgs = np.empty((n_ticks, cfg.n_envs, MSG), dtype=np.uint8)
    for b in range(cfg.n_envs):
        msgs[:, b, :] = np.frombuffer(days[b % n_days], dtype=np.uint8).reshape(day_len, MSG)[:n_ticks]

    def setup(m, first, n):
        m.load_days(lib, offs)
        m.assign_days([(first + i) % n_days for i in range(n)])

    _lockstep(rlm, oracle, "tape", cfg, n_ticks, 0.99, msgs=msgs, setup=setup)


def test_lockstep_two_replicas(rlm, oracle):
    """Two handles own the halves of 64 envs and a replica of theta each (what two ranks do); the sum of their dtheta
    is what both apply and what the oracle takes -- one more tree of additions, so the same bound holds"""
    _lockstep(rlm, oracle, "two replicas", _cfg("q_learn", 4096, 64), 600, 0.99, halves=2)
