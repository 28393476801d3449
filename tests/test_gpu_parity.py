"""CUDA path vs the CPU oracle, through the C ABI (rlm_create / rlm_run_ticks / rlm_read_records).

Bar (BASELINE.json north_star): bit-exact integer book state, <= 1e-5 relative on TD deltas.
This implementation keeps the reference's fp64 operation order, so every field of the step
record -- fp64 included -- is compared BITWISE, and so is theta.
"""
import ctypes as C

import pytest

from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu


def _mk(algo, M, n_envs, flow_seed, rec_cap, source=abi.SOURCE_GENERATOR, **over):
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo, **over})
    cfg = config.from_dict(y, n_envs=n_envs, flow_seed=flow_seed, source=source)
    cfg.record_envs = n_envs
    cfg.record_cap = rec_cap
    return y, cfg


def _compare_env(rlm_records, port, label):
    n = min(len(rlm_records), port["steps"])
    assert n > 0, label + ": no steps to compare"
    for i in range(n):
        bad = abi.record_fields_equal(rlm_records[i], port["records"][i])
        if bad:
            det = []
            for f in bad:
                a, b = getattr(rlm_records[i], f), getattr(port["records"][i], f)
                if hasattr(a, "_fields_"):
                    det.append((f, [(k, getattr(a, k), getattr(b, k)) for k, _ in a._fields_]))
                elif hasattr(a, "__len__"):
                    det.append((f, list(a), list(b)))
                else:
                    det.append((f, a, b))
            raise AssertionError("%s: step %d differs (cuda, oracle): %r" % (label, i, det))
    return n


_BOLTZ = {"policy.type": "boltzmann", "policy.tau_init": 0.1, "policy.tau_floor": 0.01, "policy.tau_T": 10}


@pytest.mark.parametrize("algo,M,over", [
    ("q_learn", 65536, {}), ("sarsa", 16384, {}), ("double_q_learn", 65536, {}), ("q_learn", 4096, {}),
    # R-learning agents (agent.cpp:357-467) and the Boltzmann policy (policy.cpp:85-122; libm exp on the CPU side,
    # CUDA exp here: an action can differ only if a uniform draw lands within an ulp of a cumulative probability)
    ("r_learn", 16384, {"policy.eps_init": 0.3}), ("online_r_learn", 16384, {"policy.eps_init": 0.3}),
    ("double_r_learn", 8209, {"policy.eps_init": 0.3, "learning.alpha_start": 0.01}),
    ("q_learn", 8192, _BOLTZ), ("double_r_learn", 4096, dict(_BOLTZ, **{"learning.alpha_start": 0.01})),
    # another venue's tick table and hours (NasdaqNordic, 17 bands, market.cpp:151-172,289-291)
    ("sarsa", 8192, {"data.symbols": ["ERIC.ST"]}),
])
def test_generator_mode_matches_oracle(rlm, oracle, algo, M, over):
    n_envs, n_ticks = 8, 3000
    y, cfg = _mk(algo, M, n_envs, flow_seed=11, rec_cap=1500, **over)
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(1000)
    m.run_ticks(2000)  # chunked launches must not change anything
    m.sync()
    cnt = m.counters()
    rew, act, st, rho = m.rewards(), m.actions(), m.state(), m.rho()
    total = 0
    for b in range(n_envs):
        ticks = oracle.generate_ticks(cfg, b, n_ticks)
        port = oracle.run_port(cfg, b, ticks)
        recs, keep = m.records(b)
        assert len(recs) == port["steps"], "env %d: step count cuda %d oracle %d" % (b, len(recs), port["steps"])
        total += _compare_env(recs, port, "%s env %d" % (algo, b))
        # packed column getters (env.getReward / state->toVector of the last completed step)
        last = recs[-1]
        assert C.c_double(rew[b]).value == last.reward and 0 <= act[b] < cfg.n_actions
        assert list(st[b * cfg.n_state_vars:(b + 1) * cfg.n_state_vars]) == list(last.state[:cfg.n_state_vars])
        th = m.theta(b, 0)
        assert bytes(th) == bytes((C.c_double * M)(*port["theta"])), "%s env %d: theta differs" % (algo, b)
        assert rho[b] == port["rho"] and (port["rho"] != 0.0) == (algo.endswith("r_learn")), (algo, b, rho[b], port["rho"])
    assert cnt.steps == total
    assert cnt.ticks == sum([n_ticks - 1] * n_envs)  # the first row only opens the market (intraday.cpp:111-116)
    m.close()


def test_stream_mode_equals_generator_mode(rlm, oracle):
    n_envs, n_ticks = 4, 1500
    y, cfg = _mk("q_learn", 8192, n_envs, flow_seed=5, rec_cap=800, source=abi.SOURCE_STREAM)
    msgs = (abi.TickMsg * (n_ticks * n_envs))()
    for b in range(n_envs):
        one = rlm.flow_generate(cfg.flow, b, 0, n_ticks)
        for t in range(n_ticks):
            msgs[t * n_envs + b] = one[t]
    ms = rlm.BatchedMarket(cfg)
    # three chunks, uploads pipelined against the running kernels (rlm_load_ticks double-buffers):
    # load(k+1) is issued while run(k) is still executing, without any host sync in between
    base, per_tick = C.addressof(msgs), n_envs * C.sizeof(abi.TickMsg)
    ms.load_ticks(base, 500)
    ms.run_ticks(200)
    ms.run_ticks(300)
    ms.load_ticks(base + 500 * per_tick, 500)
    ms.run_ticks(500)
    ms.load_ticks(base + 1000 * per_tick, 500)
    ms.run_ticks(500)
    ms.sync()
    y2, cfg2 = _mk("q_learn", 8192, n_envs, flow_seed=5, rec_cap=800, source=abi.SOURCE_GENERATOR)
    mg = rlm.BatchedMarket(cfg2)
    mg.run_ticks(n_ticks)
    mg.sync()
    for b in range(n_envs):
        rs, _k1 = ms.records(b)
        rg, _k2 = mg.records(b)
        assert len(rs) == len(rg) and len(rs) > 50
        for i in range(len(rs)):
            assert not abi.record_fields_equal(rs[i], rg[i]), "env %d step %d" % (b, i)
        assert bytes(ms.theta(b)) == bytes(mg.theta(b))
    with pytest.raises(rlm.RlmError) as ei:
        ms.run_ticks(1)  # stream exhausted: performAction would return false (base.cpp:289)
    assert ei.value.code == abi.RLM_ERR_END_OF_DATA
    ms.close()
    mg.close()


def test_run_calls_of_mixed_lengths_switch_engines_without_a_trace(rlm):
    """Short calls run tick by tick, long ones round by round (rlm_run_ticks picks per call): any split of the same ticks
    must leave the same records, weights and counters."""
    n_envs, M = 7, 8192
    res = []
    for split in ([1200], [100, 300, 64, 536, 200], [127, 128, 129, 816]):
        y, cfg = _mk("sarsa", M, n_envs, flow_seed=31, rec_cap=700)
        m = rlm.BatchedMarket(cfg)
        for n in split:
            m.run_ticks(n)
        m.sync()
        c = m.counters()
        recs = [m.records(b) for b in range(n_envs)]  # (list, backing array) per env
        res.append((c.steps, c.ticks, [bytes(m.theta(b)) for b in range(n_envs)], recs))
        m.close()
    assert res[0][0] > 100
    for other in res[1:]:
        assert other[:3] == res[0][:3]
        for b in range(n_envs):
            ra, rb = res[0][3][b][0], other[3][b][0]
            assert len(ra) == len(rb) > 10
            for i in range(len(ra)):
                assert not abi.record_fields_equal(ra[i], rb[i]), "env %d step %d" % (b, i)


@pytest.mark.parametrize("env_vars,call_ticks", [({}, 50), ({"RLM_ENV_VARIANT": "1"}, 50), ({"RLM_ROUNDS": "0"}, 250), ({}, 125)])
def test_stream_mode_in_short_run_calls(rlm, monkeypatch, env_vars, call_ticks):
    """Run calls shorter than 128 ticks stay tick-synchronous and -- from the second call on -- replay ONE CUDA graph per
    chunk length whose stream pointer / offset / length live in device memory: many calls per loaded chunk, chunk swaps
    (double-buffered uploads) in between, both tick kernels.  Must equal the generator run bit for bit."""
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    n_envs, n_ticks, chunk = 6, 1500, 500
    y, cfg = _mk("q_learn", 8192, n_envs, flow_seed=11, rec_cap=800, source=abi.SOURCE_STREAM)
    msgs = (abi.TickMsg * (n_ticks * n_envs))()
    for b in range(n_envs):
        one = rlm.flow_generate(cfg.flow, b, 0, n_ticks)
        for t in range(n_ticks):
            msgs[t * n_envs + b] = one[t]
    ms = rlm.BatchedMarket(cfg)
    base, per_tick = C.addressof(msgs), n_envs * C.sizeof(abi.TickMsg)
    for c0 in range(0, n_ticks, chunk):
        ms.load_ticks(base + c0 * per_tick, chunk)
        for _ in range(chunk // call_ticks):
            ms.run_ticks(call_ticks)
    ms.sync()
    y2, cfg2 = _mk("q_learn", 8192, n_envs, flow_seed=11, rec_cap=800, source=abi.SOURCE_GENERATOR)
    mg = rlm.BatchedMarket(cfg2)
    mg.run_ticks(n_ticks)
    mg.sync()
    assert ms.counters().steps == mg.counters().steps > 0
    for b in range(n_envs):
        rs, _k1 = ms.records(b)
        rg, _k2 = mg.records(b)
        assert len(rs) == len(rg) and len(rs) > 50
        for i in range(len(rs)):
            assert not abi.record_fields_equal(rs[i], rg[i]), "env %d step %d" % (b, i)
        assert bytes(ms.theta(b)) == bytes(mg.theta(b))
    ms.close()
    mg.close()


@pytest.mark.parametrize("env_vars,algo", [
    ({"RLM_ENV_VARIANT": "1"}, "q_learn"),        # thread-per-env tick kernel (default for B > 16384)
    ({"RLM_AGENT_VARIANT": "1"}, "q_learn"),      # one-warp-per-env learner kernel
    ({"RLM_AGENT_VARIANT": "1"}, "double_r_learn"),
    ({"RLM_ENGINE": "p"}, "sarsa"),               # persistent queue engine
    ({"RLM_ENGINE": "f"}, "double_q_learn"),      # fused warp-per-env engine
    ({"RLM_ENGINE": "f"}, "r_learn"),
    ({"RLM_ENGINE": "F"}, "q_learn"),             # fused persistent engine, round 2 (rlm_fused2_kernel)
    ({"RLM_ENGINE": "F"}, "sarsa"),
    ({"RLM_ENGINE": "F"}, "double_q_learn"),
    ({"RLM_ENGINE": "s"}, "q_learn"),             # tick-synchronous engine (two launches per tick)
    ({"RLM_ENGINE": "s", "RLM_AGENT_VARIANT": "3"}, "sarsa"),  # ... with the round-1 three-warp learner kernel
    ({"RLM_ROUNDS": "1"}, "q_learn"),             # round-paced engine (rlm_env_round_kernel): every env ticks to its step end
    ({"RLM_ROUNDS": "1"}, "double_q_learn"),
    ({"RLM_ROUNDS": "1", "RLM_ROUND_CAP": "2"}, "q_learn"),   # ... with at most two ticks per env and round
    ({"RLM_ROUNDS": "1", "RLM_ROUND_CAP": "1", "RLM_ROUND_STREAMS": "2"}, "sarsa"),
    ({"RLM_ENVW_WARPS": "2"}, "q_learn"),         # two envs per CTA of the warp-per-env tick kernel
    ({"RLM_ROUNDS": "0"}, "q_learn"),             # tick-synchronous engine for every call (long calls default to rounds)
    ({"RLM_ROUNDS": "0"}, "double_q_learn"),
    ({"RLM_ROUNDS": "1"}, "r_learn"),             # (not part of the default: R-learning stays tick-synchronous)
    ({"RLM_SUBBATCHES": "3", "RLM_ROUNDS": "0"}, "q_learn"),  # three sub-batch streams; 5 envs fill the first, two stay empty
])
def test_every_engine_variant_matches_oracle(rlm, oracle, monkeypatch, env_vars, algo):
    """The non-default kernels (selected by environment variables read in rlm_create) are held to the same bar."""
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    n_envs, n_ticks, M = 5, 1500, 8192
    y, cfg = _mk(algo, M, n_envs, flow_seed=23, rec_cap=800)
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(n_ticks)
    m.sync()
    for b in range(n_envs):
        port = oracle.run_port(cfg, b, oracle.generate_ticks(cfg, b, n_ticks))
        recs, _keep = m.records(b)
        assert len(recs) == port["steps"] > 100
        _compare_env(recs, port, "%s %r env %d" % (algo, env_vars, b))
        assert bytes(m.theta(b, 0)) == bytes((C.c_double * M)(*port["theta"]))
    m.close()


def test_sub_batches_of_one_env_match_oracle(rlm, oracle, monkeypatch):
    """RLM_SUBBATCHES=3 at 65 envs: split_batch cuts whole warps, so the sub-batches hold 32, 32 and 1 envs; the envs at
    each sub-batch's edges are held to the oracle"""
    monkeypatch.setenv("RLM_SUBBATCHES", "3")
    monkeypatch.setenv("RLM_ROUNDS", "0")
    n_envs, n_ticks, M = 65, 1500, 8192
    y, cfg = _mk("q_learn", M, n_envs, flow_seed=23, rec_cap=800)
    m = rlm.BatchedMarket(cfg)
    m.run_ticks(n_ticks)
    m.sync()
    for b in (0, 31, 32, 63, 64):
        port = oracle.run_port(cfg, b, oracle.generate_ticks(cfg, b, n_ticks))
        recs, _keep = m.records(b)
        assert len(recs) == port["steps"] > 100
        _compare_env(recs, port, "sub-batches env %d" % b)
        assert bytes(m.theta(b, 0)) == bytes((C.c_double * M)(*port["theta"]))
    m.close()


@pytest.mark.parametrize("streams", [1, 3])
def test_round_paced_engine_on_a_chunked_stream(rlm, oracle, monkeypatch, streams):
    """RLM_ROUNDS=1 with sub-batches on their own streams, several run calls per loaded chunk and a chunk swap in between
    (the engine's CUDA graphs outlive rlm_load_ticks; the stream pointer travels through device memory)."""
    monkeypatch.setenv("RLM_ROUNDS", "1")
    monkeypatch.setenv("RLM_ROUND_STREAMS", str(streams))
    n_envs, n_ticks, M = 70, 900, 4096
    y, cfg = _mk("q_learn", M, n_envs, flow_seed=29, rec_cap=500, source=abi.SOURCE_STREAM)
    check = [0, 33, 69]
    per_env = {b: oracle.generate_ticks(cfg, b, n_ticks) for b in check}
    filler = rlm.flow_generate(cfg.flow, 1, 0, n_ticks)
    msgs = (abi.TickMsg * (n_ticks * n_envs))()
    for t in range(n_ticks):
        for b in range(n_envs):
            msgs[t * n_envs + b] = per_env[b][t] if b in per_env else filler[t]
    m = rlm.BatchedMarket(cfg)
    base, per_tick = C.addressof(msgs), n_envs * C.sizeof(abi.TickMsg)
    m.load_ticks(base, 500)
    m.run_ticks(150)
    m.run_ticks(150)
    m.run_ticks(200)
    m.load_ticks(base + 500 * per_tick, 400)
    m.run_ticks(1)
    m.run_ticks(399)
    m.sync()
    assert m.counters().ticks == n_envs * (n_ticks - 1)
    for b in check:
        port = oracle.run_port(cfg, b, per_env[b])
        recs, _keep = m.records(b)
        assert len(recs) == port["steps"] > 100
        _compare_env(recs, port, "round-paced, %d streams, env %d" % (streams, b))
        assert bytes(m.theta(b, 0)) == bytes((C.c_double * M)(*port["theta"]))
    m.close()
