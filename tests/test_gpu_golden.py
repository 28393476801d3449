"""CUDA path vs the REFERENCE's own outputs (tests/golden, produced by the unmodified reference
compiled into oracle/_ref -- see tools/make_golden.py), plus the unit-level device entry points
against the reference's unit vectors.  All comparisons are bitwise."""
import ctypes as C

import pytest

import golden_util as G
from rl_markets_b200 import abi, config

pytestmark = pytest.mark.gpu


def test_step_records_match_the_reference(rlm):
    for case in G.manifest():
        # env `case["env"]` of a batch: local env 0 with env_index0 = case env (seeds and flow stream follow the global index)
        cfg = G.case_config(case, n_envs=3, env_index0=case["env"])
        cfg.record_envs = 1
        cfg.record_cap = 600
        m = rlm.BatchedMarket(cfg)
        m.run_ticks(case["ticks"])
        m.sync()
        recs, _keep = m.records(0)
        gold, _k2 = G.records(case["name"])
        assert len(recs) >= len(gold) > 100, (case["name"], len(recs))
        # mm_exp calls exp()/pow() (base.cpp:216-221): glibc's in the reference, CUDA's here -- both within an ulp of the
        # true value but not identical, so THIS case is held to the north star's 1e-5 relative bar on the fp64 fields that
        # depend on the reward (observed ~1e-9) and bitwise on everything else (integer book state included)
        tol = {"reward", "ep_reward", "delta", "trace_hash"} if case["yaml"]["reward"]["measure"] == "mm_exp" else set()
        for i, g in enumerate(gold):
            bad = abi.record_fields_equal(g, recs[i])
            for f in [f for f in bad if f in tol and f != "trace_hash"]:
                x, y = getattr(g, f), getattr(recs[i], f)
                assert abs(x - y) <= 1e-5 * max(abs(x), abs(y)), (case["name"], i, f, x, y)
            bad = [f for f in bad if f not in tol]
            assert not bad, "%s step %d (reference, cuda): %r" % (case["name"], i, G.describe_diff(g, recs[i], bad))
        m.close()


def test_multi_episode_records_match_the_reference(rlm):
    """N training episodes on one env + one Learner (main.cpp:45-60, serial.cpp:72-95) against the reference's own dump:
    rlm_handle_terminal(episode) + rlm_reset carry the stale State of Runner into the next episode (serial.cpp:24-25,55,60)
    and keep the window sums Base::Initialise does not clear (accumulators.cpp:60-64)."""
    for case in G.episode_manifest():
        cfg = G.case_config(case, n_envs=3, env_index0=case["env"])
        cfg.flow.t0_ms = case["t0_ms"]
        cfg.record_envs = 1
        cfg.record_cap = case["n_records"] + 16
        m = rlm.BatchedMarket(cfg)
        for ep in range(case["episodes"]):
            m.run_ticks(case["ticks"])  # more than the day holds: the env stops at the close
            m.sync()
            assert m.stats(0, 1)[0].terminal == 1
            m.handle_terminal(ep)
            m.reset()
        recs, _keep = m.records(0)
        gold, _k2 = G.records(case["name"])
        assert len(recs) == len(gold) == case["n_records"], (case["name"], len(recs), len(gold))
        for i, g in enumerate(gold):
            bad = abi.record_fields_equal(g, recs[i])
            assert not bad, "%s step %d (reference, cuda): %r" % (case["name"], i, G.describe_diff(g, recs[i], bad))
        m.close()


def test_device_to_ticks_and_to_price(rlm):
    L = rlm.load()
    for m in G.units()["market"]:
        cfg = config.from_dict(config.example_dict(), ticker=m["symbol"])
        px = [G.hex_to_double(h) for h in m["px"]]
        n = len(px)
        out = (C.c_int32 * n)()
        rlm.check(L.rlm_test_to_ticks(C.byref(cfg), (C.c_double * n)(*px), n, out))
        assert list(out) == m["ticks"], m["symbol"]
        nt = len(m["tq"])
        outp = (C.c_double * nt)()
        rlm.check(L.rlm_test_to_price(C.byref(cfg), (C.c_int32 * nt)(*m["tq"]), nt, outp))
        assert [G.double_bits(x) for x in outp] == [int(h, 16) for h in m["price"]], m["symbol"]


def _unit_states(t):
    flat = []
    for c in t["cases"]:
        flat += list(G.tile_vars(c))
    return (C.c_float * len(flat))(*flat), len(t["cases"])


def test_device_tiles(rlm, oracle):
    L = rlm.load()
    for t in G.units()["tiles"]:
        cfg = G.tile_config(t)
        arr, n = _unit_states(t)
        per = t["n_actions"] * 96
        out = (C.c_int32 * (n * per))()
        rlm.check(L.rlm_test_tiles(C.byref(cfg), arr, n, out))
        for k, c in enumerate(t["cases"]):
            assert list(out[k * per:(k + 1) * per]) == c["features"], (t["memory_size"], t["n_actions"], t["n_vars"], k)
    # a larger seeded sweep against the CPU oracle (bit-exact int32 indices)
    import random
    rnd = random.Random(3)
    cfg = config.from_dict(config.example_dict(**{"learning.memory_size": 1000003}))
    n = 2000
    flat = [C.c_float(rnd.uniform(-120, 120) if rnd.random() < 0.8 else float(rnd.randint(-100, 100))).value for _ in range(n * 8)]
    arr = (C.c_float * len(flat))(*flat)
    out = (C.c_int32 * (n * 864))()
    rlm.check(L.rlm_test_tiles(C.byref(cfg), arr, n, out))
    OL = oracle.lib()
    ref = (C.c_int32 * 864)()
    for k in range(n):
        OL.lobo_tiles(C.byref(cfg), (C.c_float * 8)(*flat[k * 8:(k + 1) * 8]), ref)
        assert list(out[k * 864:(k + 1) * 864]) == list(ref), k


def test_device_order_scripts(rlm):
    L = rlm.load()
    for o in G.units()["orders"]:
        n = len(o["ops"])
        ops = (abi.OrderOp * n)(*[abi.OrderOp(op, 0, arg) for op, arg in o["ops"]])
        out = (abi.OrderState * n)()
        rlm.check(L.rlm_test_order(o["size"], o["q_head"], ops, n, out))
        got = [[out[i].q_head, out[i].q_tail, out[i].executed, out[i].ret] for i in range(n)]
        assert got == o["out"], o
    # error behaviour of market::Order (order.cpp:22-27,56-57,86-87) maps to RLM_ERR_RUNTIME
    one = (abi.OrderOp * 1)(abi.OrderOp(1, 0, -50))
    st = (abi.OrderState * 1)()
    assert L.rlm_test_order(1, 1, one, 1, st) == abi.RLM_ERR_RUNTIME
    assert L.rlm_test_order(-100, 0, one, 0, st) == abi.RLM_ERR_RUNTIME
    assert L.rlm_test_order(100, -100, one, 0, st) == abi.RLM_ERR_RUNTIME


def test_device_rolling_mean(rlm):
    L = rlm.load()
    for r in G.units()["rolling"]:
        vals = [G.hex_to_double(h) for h in r["vals"]]
        n = len(vals)
        out = (C.c_double * (2 * n))()
        rlm.check(L.rlm_test_rolling_mean(r["window"], (C.c_double * n)(*vals), n, out))
        for i, (a, b) in enumerate(r["mean_var"]):
            assert G.double_bits(out[2 * i]) == int(a, 16), (r["window"], i)
            assert G.double_bits(out[2 * i + 1]) == int(b, 16) or out[2 * i + 1] != out[2 * i + 1], (r["window"], i)


# rlm_test_learner_tiles forms (include/rlm.h)
THREE_WARP, ONE_WARP, STAGED, TRACE_GROUP0 = 0, 1, 2, 3


def _learner_tiles(rlm, cfg, form, arr, n):
    per = cfg.n_actions * (32 if form == TRACE_GROUP0 else 96)
    out = (C.c_int32 * (n * per))()
    rlm.check(rlm.load().rlm_test_learner_tiles(C.byref(cfg), form, arr, n, out))
    return [list(out[k * per:(k + 1) * per]) for k in range(n)]


def _forms(M):
    return (THREE_WARP, ONE_WARP, TRACE_GROUP0) + ((STAGED,) if M <= 8192 else ())


def _expected(form, feats, A):
    """What a form returns for a state whose reference features are feats[a*96 + i]."""
    if form == TRACE_GROUP0:
        return [f for a in range(A) for f in feats[a * 96:a * 96 + 32]]
    return feats


def test_device_learner_tile_forms_match_the_reference(rlm):
    """Every way the learner kernels derive a tile index -- the three-warp kernel's tile_index, the one-warp learner's
    hash sums + ln_tile, the staged learner's 16-bit rows, and the trace passes' group-0 tiles rebuilt from the stored
    base -- against rl::State's own features, from tables of 1 weight up to 2^31 - 1 and for 1..9 actions, 4..13
    variables.  Above 2^30 the group-0 rebuild adds two indices below M: their sum must not wrap."""
    for t in G.units()["tiles"]:
        cfg = G.tile_config(t)
        arr, n = _unit_states(t)
        for form in _forms(t["memory_size"]):
            got = _learner_tiles(rlm, cfg, form, arr, n)
            for k, c in enumerate(t["cases"]):
                assert got[k] == _expected(form, c["features"], t["n_actions"]), (form, t["memory_size"], t["n_actions"], t["n_vars"], k)
    cfg = G.tile_config({"memory_size": 8193, "n_actions": 9, "n_vars": 8})
    out = (C.c_int32 * 864)()
    assert rlm.load().rlm_test_learner_tiles(C.byref(cfg), STAGED, (C.c_float * 8)(), 1, out) == abi.RLM_ERR_UNSUPPORTED


@pytest.mark.parametrize("M", [1, 2, 3, 97, 5003, 6000, 8190, 8192, 8194, 65536, 20000000, 1 << 27, (1 << 27) + 1,
                               (1 << 30) + 3, 3 << 29, 2 ** 31 - 1])
def test_device_learner_tile_forms_sweep(rlm, oracle, M):
    """Seeded states against the CPU oracle's tiles() for every form, action count and state size."""
    import random
    OL = oracle.lib()
    rnd = random.Random(M)
    n = 48
    for A, V in ((1, 4), (5, 13), (9, 8), (2, 11)):
        cfg = G.tile_config({"memory_size": M, "n_actions": A, "n_vars": V})
        flat = [C.c_float(rnd.uniform(-700, 700) if rnd.random() < 0.8 else float(rnd.randint(-100, 100))).value for _ in range(n * V)]
        arr = (C.c_float * len(flat))(*flat)
        ref = []
        for k in range(n):
            out = (C.c_int32 * (A * 96))()
            OL.lobo_tiles(C.byref(cfg), (C.c_float * V)(*flat[k * V:(k + 1) * V]), out)
            ref.append(list(out))
        for form in _forms(M):
            got = _learner_tiles(rlm, cfg, form, arr, n)
            for k in range(n):
                assert got[k] == _expected(form, ref[k], A), (form, M, A, V, k)
