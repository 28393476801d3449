"""The split surface in backtest mode: rlm_act / rlm_env_step / rlm_agent_update stand for
experiment::serial::Backtester::_step (src/experiment/serial.cpp:124-137), driven in Runner::RunEpisode's order:

    env_step(None)        environment.Initialise()                       serial.cpp:21-22
    agent_update()        last_state->newState(environment)              serial.cpp:25
    repeat:
      act()               int action = m->action(*state)                 serial.cpp:131
      env_step(actions)   environment.performAction(action)              serial.cpp:133
      agent_update()      state->newState(environment) of the next step  serial.cpp:129

Held bit for bit to rlm_run_ticks in backtest mode (records, rlm_env_stats, counters, reward / terminal outputs, theta
untouched) on independent and shared policies, and through main.cpp:216-244's sequence of test days to the reference's
own records (tests/golden/eval_days.json).  External actions (env_step without act) backtest a caller's own policy."""
import ctypes as C

import pytest

import test_gpu_eval_days as EV
import test_gpu_shared_backtest as SB
from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu
T0_MS, DAY_TICKS = 57425000, 1000  # 250 ms ticks from 15:57:05: the close (16:00) and the closing ClearInventory are inside
COUNTED = ("ticks", "steps", "sum_traces", "terminal_envs")  # rlm_counters without kernel_launches (the split calls launch more)


def split_day(m, max_steps=20000):
    """Backtester::RunEpisode for every env on the split surface, until no env is at a decision point any more (every
    episode over, or its tape day run out) -> (reward_out, terminal_out) of the last env_step"""
    m.env_step(None)
    assert all(d == 0.0 for d in m.agent_update())
    for _ in range(max_steps):
        a = m.act()
        rew, term = m.env_step(a)
        assert all(d == 0.0 for d in m.agent_update()), "Backtester::_step computes no TD error"
        if all(x < 0 for x in a):
            return rew, term
    raise AssertionError("the day did not end within %d steps" % max_steps)


def _yaml(algo, M=8192):
    return config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})


def _test_flow(y, seed=34):
    flow = config.from_dict(y, flow_seed=seed).flow
    flow.t0_ms = T0_MS
    return flow


def _tables(m, policy=0):
    double = m.cfg.algorithm in (abi.ALGO["double_q_learn"], abi.ALGO["double_r_learn"])
    return [bytes(m.theta(policy, k)) for k in range(2 if double else 1)]


def _all_tables(m):
    return [_tables(m, p) for p in range(1 if m.cfg.shared_policy else m.cfg.n_envs)]


def _trained_twins(rlm, algo, B=6, train_ticks=600):
    """two handles trained alike on a short stretch of a day (fused path), then GoGreedy, Backtester and the new env
    object of main.cpp:219 on the test day.  Both train, rather than one training and the other loading its tables:
    the greedy policy breaks ties with the agent's glibc rand(), whose state travels from training into evaluation."""
    y = _yaml(algo)
    cfg = config.from_dict(y, n_envs=B, flow_seed=31, env_index0=2)
    cfg.record_envs, cfg.record_cap = B, 1200
    ms = []
    for _ in range(2):
        m = rlm.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
        m.run_ticks(train_ticks)
        m.sync()
        assert m.counters().steps > 10 * B
        m.handle_terminal(0)
        m.go_greedy()
        m.set_mode(abi.MODE_BACKTEST)
        m.new_env(_test_flow(y))
        ms.append(m)
    assert _all_tables(ms[0]) == _all_tables(ms[1])
    return ms


def _counted(m):
    c = m.counters()
    return tuple(getattr(c, k) for k in COUNTED)


def assert_same_run(a, b, tag, min_records=100):
    """records of every env, rlm_env_stats and the counters of two handles, bitwise"""
    B = a.cfg.n_envs
    for e in range(B):
        ra, rb = a.records(e)[0], b.records(e)[0]
        assert len(ra) >= min_records, (tag, e, len(ra))
        SB._assert_records(ra, rb, tag + (e,))
    assert bytes(a.stats()) == bytes(b.stats()), tag
    assert _counted(a) == _counted(b), tag


@pytest.mark.parametrize("algo,variant", [(a, 0) for a in abi.ALGO] + [("q_learn", 1), ("double_q_learn", 1)])
def test_split_backtest_equals_the_fused_backtest(rlm, monkeypatch, algo, variant):
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    fused, split = _trained_twins(rlm, algo)
    before = _all_tables(split)
    fused.run_ticks(DAY_TICKS)
    fused.sync()
    rew, term = split_day(split)
    tag = (algo, variant)
    assert_same_run(split, fused, tag)
    assert bytes(rew) == bytes(fused.rewards()), tag  # reward_out is Base::getReward, as rlm_get_reward reports it
    stats = fused.stats()
    assert all(s.terminal == 1 for s in stats) and list(term) == [1] * split.cfg.n_envs, tag
    assert _all_tables(split) == before == _all_tables(fused), (tag, "evaluation must not touch theta")
    for m in (fused, split):
        m.close()


@pytest.mark.parametrize("variant", [0, 1])
def test_run_ticks_continues_where_the_split_calls_stopped(rlm, monkeypatch, variant):
    """part of the day through the split surface, the rest through rlm_run_ticks: the fused twin's day, bit for bit"""
    monkeypatch.setenv("RLM_ENV_VARIANT", str(variant))
    fused, split = _trained_twins(rlm, "q_learn")
    fused.run_ticks(DAY_TICKS)
    split.env_step(None)
    split.agent_update()
    for k in range(60):
        split.env_step(split.act())
        split.agent_update()
    split.act()                       # an action drawn and not applied yet: rlm_run_ticks applies it
    split.run_ticks(DAY_TICKS)
    for m in (fused, split):
        m.sync()
    assert_same_run(split, fused, ("continued", variant))
    for m in (fused, split):
        m.close()


def _shared_and_independent(rlm, y, theta, B, shared):
    cfg = config.from_dict(y, n_envs=B, env_index0=3, shared_policy=shared, flow_seed=33)
    cfg.record_envs, cfg.record_cap = B, 600
    return SB._evaluator(rlm, cfg, theta, _test_flow(y))


@pytest.mark.parametrize("M", [4096, 2 * 2053])  # (a shared table has an even size: twice a prime takes the modulo path)
@pytest.mark.parametrize("algo", ["q_learn", "double_q_learn"])
def test_split_backtest_of_a_shared_policy(rlm, algo, M):
    """one table loaded into a shared handle: split = fused, env by env, and both = an independent handle that carries the
    same table in every env"""
    B = 8
    y = SB._yaml(algo, M)
    theta = SB._train_shared(rlm, y)
    split = _shared_and_independent(rlm, y, theta, B, True)
    fused = _shared_and_independent(rlm, y, theta, B, True)
    indep = _shared_and_independent(rlm, y, theta, B, False)
    before = SB._policy_bytes(split)
    rew, term = split_day(split)
    for m in (fused, indep):
        m.run_ticks(DAY_TICKS)
        m.sync()
    assert SB._policy_bytes(split) == before, "evaluation must not touch theta or dtheta"
    assert_same_run(split, fused, (algo, M, "fused"))
    assert_same_run(split, indep, (algo, M, "independent"))
    assert bytes(rew) == bytes(fused.rewards()) and list(term) == [1] * B
    for m in (split, fused, indep):
        m.close()


class SplitEvaluation(EV.Evaluation):
    """test_gpu_eval_days.Evaluation with every test day driven through the split surface (training stays fused)"""

    def _feed(self, k):
        if k < 0:
            return super()._feed(k)
        split_day(self.m)


@pytest.mark.parametrize("source", ["generator", "tape"])
def test_main_cpp_test_days_on_the_split_surface(rlm, source):
    """train, GoGreedy, rlm_new_env, then per later test day set_flow + reset (generator) or assign_days + reset (tape,
    with the AAL.L / BAES.L days under their own markets): env 0 against the reference's records and day summaries, the
    other envs against the oracle"""
    for c in EV._cases(source):
        ev = SplitEvaluation(rlm, c, source, n_envs=3)
        EV._check(ev)
        ev.close()


def _fused_twin_and_actions(rlm, algo="q_learn"):
    fused, ext = _trained_twins(rlm, algo, B=4)
    fused.run_ticks(DAY_TICKS)
    fused.sync()
    return fused, ext, [[r.action for r in fused.records(b)[0]] for b in range(fused.cfg.n_envs)]


def test_external_actions_replay_the_fused_backtest(rlm):
    """the fused twin's actions supplied from outside (no Agent::action, no policy draw): the same records and stats"""
    fused, ext, acts = _fused_twin_and_actions(rlm)
    B = ext.cfg.n_envs
    before = _all_tables(ext)
    ext.env_step(None)
    ext.agent_update()
    for k in range(max(len(a) for a in acts) + 1):  # (+1: the step after the last one ends the episode, ClearInventory)
        step = (C.c_int32 * B)(*[acts[b][k] if k < len(acts[b]) else 0 for b in range(B)])
        ext.env_step(step)
        ext.agent_update()
    ext.sync()
    assert all(s.terminal == 1 for s in ext.stats())
    for b in range(B):
        SB._assert_records(ext.records(b)[0], fused.records(b)[0], ("replay", b))
    assert bytes(ext.stats()) == bytes(fused.stats())
    assert _all_tables(ext) == before
    for m in (fused, ext):
        m.close()


def test_scripted_actions_and_fused_continuation(rlm):
    """a scripted action sequence appears verbatim in the records; rlm_run_ticks then finishes the day"""
    _fused, m, _acts = _fused_twin_and_actions(rlm)
    _fused.close()
    B, n = m.cfg.n_envs, 40
    script = [(5 * k + 2 * b) % m.cfg.n_actions for k in range(n) for b in range(B)]
    m.env_step(None)
    m.agent_update()
    for k in range(n):
        m.env_step((C.c_int32 * B)(*script[k * B:(k + 1) * B]))
        m.agent_update()
    for b in range(B):
        recs = m.records(b)[0]
        assert [r.action for r in recs] == [script[k * B + b] for k in range(n)], b
        assert all(r.delta == 0.0 for r in recs)
    steps = m.counters().steps
    m.run_ticks(DAY_TICKS)
    m.sync()
    assert m.counters().steps > steps + B * 20
    assert all(s.terminal == 1 for s in m.stats())
    m.close()


def test_what_the_split_surface_still_rejects(rlm):
    """the stream source (tick-aligned) in backtest mode, and a shared handle in train mode"""
    y = _yaml("q_learn", 4096)
    m = rlm.BatchedMarket(config.from_dict(y, n_envs=2, source=abi.SOURCE_STREAM))
    m.set_mode(abi.MODE_BACKTEST)
    for call in (m.act, lambda: m.env_step(None), m.agent_update):
        with pytest.raises(rlm.RlmError) as ei:
            call()
        assert ei.value.code == abi.RLM_ERR_UNSUPPORTED
    m.close()
    m = rlm.BatchedMarket(config.from_dict(y, n_envs=2, shared_policy=True))
    for call in (m.act, lambda: m.env_step(None), m.agent_update):
        with pytest.raises(rlm.RlmError) as ei:
            call()
        assert ei.value.code == abi.RLM_ERR_UNSUPPORTED
    m.set_mode(abi.MODE_BACKTEST)  # the same handle evaluates on the split surface
    m.env_step(None)
    m.agent_update()
    m.close()


def test_agent_update_in_backtest_mode_gives_zero_deltas(rlm):
    """the TD errors of split-surface training are nonzero; after set_mode(BACKTEST) agent_update returns 0.0 for every env,
    the envs that just took their first decision state included"""
    y = _yaml("q_learn", 4096)
    cfg = config.from_dict(y, n_envs=4, flow_seed=9)
    m = rlm.BatchedMarket(cfg)
    m.env_step(None)
    m.agent_update()
    deltas = []
    for _ in range(60):
        m.env_step(m.act())
        deltas += list(m.agent_update())
    assert any(d != 0.0 for d in deltas)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    m.new_env(_test_flow(y))
    m.env_step(None)
    assert list(m.agent_update()) == [0.0] * 4
    for _ in range(20):
        m.env_step(m.act())
        assert list(m.agent_update()) == [0.0] * 4
    m.close()
