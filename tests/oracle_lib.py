"""Test-side access to the oracle (oracle/liblob_oracle.so and oracle/_ref/*).

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this.
"""
import ctypes as C
import json
import os
import subprocess
import tempfile

import yaml

from rl_markets_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
REF_DIR = os.path.join(ORACLE_DIR, "_ref")
LIB_PATH = os.path.join(ORACLE_DIR, "liblob_oracle.so")
REF_DRIVER = os.path.join(REF_DIR, "ref_driver")
REF_UNITS = os.path.join(REF_DIR, "ref_units")
FLOW_CSV = os.path.join(REF_DIR, "flow_csv")

_lib = None


class BookOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("side", C.c_int32), ("px", C.c_double * 5), ("vol", C.c_int64 * 5),
                ("n", C.c_int32), ("pad", C.c_int32), ("a", C.c_double), ("b", C.c_int64)]


class BookResult(C.Structure):
    _fields_ = [("r_volume", C.c_int64), ("r_proxy", C.c_double), ("r_value", C.c_double), ("r_ok", C.c_int32),
                ("n_transacted", C.c_int32), ("order", abi.OrderRec), ("obs_value", C.c_double),
                ("obs_volume", C.c_int64), ("total_volume", C.c_int64)]


def build_port():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "port"])


def have_ref():
    return os.path.exists(REF_DRIVER)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build_port()
        L = C.CDLL(LIB_PATH)
        L.lobo_create.restype = C.c_void_p
        L.lobo_create.argtypes = [C.POINTER(abi.Config), C.c_int64]
        L.lobo_destroy.argtypes = [C.c_void_p]
        L.lobo_run.restype = C.c_int64
        L.lobo_run.argtypes = [C.c_void_p, C.POINTER(abi.TickMsg), C.c_int64, C.c_int64,
                               C.POINTER(abi.StepRecord), C.c_int64, C.POINTER(C.c_int64)]
        L.lobo_is_terminal.argtypes = [C.c_void_p]
        L.lobo_stats.argtypes = [C.c_void_p, C.POINTER(abi.EnvStats)]
        L.lobo_total_steps.restype = C.c_int64
        L.lobo_total_steps.argtypes = [C.c_void_p]
        L.lobo_total_ticks.restype = C.c_int64
        L.lobo_total_ticks.argtypes = [C.c_void_p]
        L.lobo_sum_traces.restype = C.c_int64
        L.lobo_sum_traces.argtypes = [C.c_void_p]
        L.lobo_theta.restype = C.POINTER(C.c_double)
        L.lobo_theta.argtypes = [C.c_void_p, C.c_int]
        L.lobo_handle_terminal.argtypes = [C.c_void_p, C.c_int]
        L.lobo_go_greedy.argtypes = [C.c_void_p]
        L.lobo_reset.argtypes = [C.c_void_p]
        L.lobo_reset_fresh_learner.argtypes = [C.c_void_p]
        L.lobo_set_backtest.argtypes = [C.c_void_p, C.c_int]
        L.lobo_new_env.argtypes = [C.c_void_p]
        L.lobo_rho.argtypes = [C.c_void_p]
        L.lobo_rho.restype = C.c_double
        L.lobo_run_batch.restype = C.c_int64
        L.lobo_run_batch.argtypes = [C.POINTER(abi.Config), C.c_int32, C.c_int64, C.c_int32,
                                     C.POINTER(C.c_int64), C.POINTER(C.c_double)]
        L.lobo_to_ticks.restype = C.c_int32
        L.lobo_to_ticks.argtypes = [C.POINTER(abi.Config), C.c_double]
        L.lobo_to_price.restype = C.c_double
        L.lobo_to_price.argtypes = [C.POINTER(abi.Config), C.c_int32]
        L.lobo_tick_size.restype = C.c_double
        L.lobo_tick_size.argtypes = [C.POINTER(abi.Config), C.c_double]
        L.lobo_tiles.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_float), C.POINTER(C.c_int32)]
        L.lobo_order_script.argtypes = [C.c_int64, C.c_int64, C.POINTER(abi.OrderOp), C.c_int32,
                                        C.POINTER(abi.OrderState)]
        L.lobo_rolling_mean.argtypes = [C.c_int32, C.POINTER(C.c_double), C.c_int32, C.POINTER(C.c_double)]
        L.lobo_mt19937_64.restype = C.c_uint64
        L.lobo_mt19937_64.argtypes = [C.c_uint64, C.c_int32]
        L.lobo_glibc_rand.restype = C.c_int32
        L.lobo_glibc_rand.argtypes = [C.c_uint32, C.c_int32]
        L.lobo_uniform_real.restype = C.c_double
        L.lobo_uniform_real.argtypes = [C.c_uint64, C.c_int32]
        L.lobo_uniform_int.restype = C.c_uint32
        L.lobo_uniform_int.argtypes = [C.c_uint64, C.c_uint32, C.c_int32]
        L.lobo_book_script.argtypes = [C.POINTER(BookOp), C.c_int32, C.POINTER(BookResult)]
        _lib = L
    return _lib


def lib_generate(cfg, env_index, n_ticks):
    """Synthetic flow through the product's host entry point rlm_flow_generate (no GPU needed)."""
    from rl_markets_b200 import lib as rlm
    return rlm.flow_generate(cfg.flow, env_index, 0, n_ticks)


def generate_ticks(cfg, env_index, n_ticks):
    """Synthetic flow for one env as a ctypes array of TickMsg (via oracle/_ref/flow_csv --packed)."""
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "t.bin")
        subprocess.check_call([FLOW_CSV, "--seed", str(cfg.flow.seed), "--env", str(env_index), "--ticks",
                               str(n_ticks), "--dt-ms", str(cfg.flow.dt_ms), "--t0-ms", str(cfg.flow.t0_ms), "--packed", p])
        raw = open(p, "rb").read()
    arr = (abi.TickMsg * n_ticks).from_buffer_copy(raw)
    return arr


def run_port(cfg, env_index, ticks, max_steps=-1, rec_cap=None, theta_at=None):
    """Run the CPU restatement for one env; returns (records list, steps, consumed, handle-free stats).
    theta: the whole table up to 2^20 weights, None above.  theta_nz: (indices, values) of the nonzero weights as
    numpy arrays, at any size.  theta_at: optional int64 indices whose weights come back as "theta_at"."""
    L = lib()
    h = L.lobo_create(C.byref(cfg), env_index)
    assert h, "lobo_create failed"
    n = len(ticks)
    cap = rec_cap if rec_cap is not None else n
    recs = (abi.StepRecord * cap)()
    used = C.c_int64(0)
    steps = L.lobo_run(h, ticks, n, max_steps, recs, cap, C.byref(used))
    assert steps >= 0, "lobo_run raised"
    st = abi.EnvStats()
    L.lobo_stats(h, C.byref(st))
    out = {"records": [recs[i] for i in range(min(steps, cap))], "steps": steps, "consumed": used.value, "stats": st,
           "sum_traces": L.lobo_sum_traces(h), "ticks": L.lobo_total_ticks(h), "rho": L.lobo_rho(h), "_keep": recs}
    M = cfg.memory_size
    th = L.lobo_theta(h, 0)
    out["theta"] = [th[i] for i in range(M)] if M <= (1 << 20) else None
    import numpy as np
    view = np.ctypeslib.as_array(th, shape=(M,))
    nz = np.flatnonzero(view)
    out["theta_nz"] = (nz, view[nz].copy())
    if theta_at is not None:
        out["theta_at"] = view[np.asarray(theta_at, dtype=np.int64)].copy()
    del view
    L.lobo_destroy(h)
    return out


def _emit(d, indent, out):
    for k, v in d.items():
        pad = " " * indent
        if isinstance(v, dict):
            out.append("%s%s:" % (pad, k))
            _emit(v, indent + 4, out)
        elif isinstance(v, (list, tuple)):
            items = ", ".join(('"%s"' % x) if isinstance(x, str) else repr(x) for x in v)
            out.append("%s%s: [%s]" % (pad, k, items))
        elif isinstance(v, bool):
            out.append("%s%s: %s" % (pad, k, "true" if v else "false"))
        else:
            out.append("%s%s: %s" % (pad, k, v))


def write_ref_yaml(path, ydict):
    """Block-style yaml in the dialect of config/example.yaml (what oracle/shim parses)."""
    out = []
    _emit(ydict, 0, out)
    with open(path, "w") as f:
        f.write("\n".join(out) + "\n")


def run_ref(ydict, flow_seed, env_index, n_ticks, dt_ms=250, max_steps=-1, algo=None, want_theta=False, t0_ms=None,
            test=None, episodes=1, tests=None):
    """Run the UNMODIFIED reference (oracle/_ref/ref_driver) on the CSV rendering of the same flow.
    test = dict(flow_seed, env, ticks, t0_ms): also run main.cpp's evaluation phase (greedy agent, new env,
    Backtester) on a second stream; its records come back as "test_records".
    tests = [day, ...]: main.cpp's evaluation phase over several test days on ONE env object (main.cpp:216-244); a day is
    dict(flow_seed, env, ticks, t0_ms) for a synthetic stream or dict(md, tas) for a CSV pair, each optionally with
    "symbol" (default: the yaml's).  The records of day d come back as "test_days"[d]; logs=True on the first day
    collects the evaluation logs of all days."""
    assert not (test and tests), "test= and tests= are two spellings of the evaluation phase"
    assert have_ref(), "oracle/_ref/ref_driver not built"
    with tempfile.TemporaryDirectory() as d:
        md, tas = os.path.join(d, "x_md_1.csv"), os.path.join(d, "x_tas_1.csv")
        t0 = [] if t0_ms is None else ["--t0-ms", str(t0_ms)]
        subprocess.check_call([FLOW_CSV, "--seed", str(flow_seed), "--env", str(env_index), "--ticks", str(n_ticks),
                               "--dt-ms", str(dt_ms), "--md", md, "--tas", tas] + t0)
        cfgp = os.path.join(d, "cfg.yaml")
        write_ref_yaml(cfgp, ydict)
        dump = os.path.join(d, "steps.bin")
        thp = os.path.join(d, "theta.bin")
        cmd = [REF_DRIVER, "--config", cfgp, "--symbol", ydict["data"]["symbols"][0], "--md", md, "--tas", tas,
               "--dump", dump, "--steps", str(max_steps)]
        if algo:
            cmd += ["--algo", algo]
        if episodes != 1:  # one Intraday + one Learner-equivalent reused over N episodes (main.cpp:45-60)
            cmd += ["--episodes", str(episodes)]
        if want_theta:
            cmd += ["--theta", thp]
        dump2 = os.path.join(d, "test_steps.bin")
        if test:
            md2, tas2 = os.path.join(d, "y_md_1.csv"), os.path.join(d, "y_tas_1.csv")
            t02 = [] if test.get("t0_ms") is None else ["--t0-ms", str(test["t0_ms"])]
            subprocess.check_call([FLOW_CSV, "--seed", str(test["flow_seed"]), "--env", str(test["env"]), "--ticks",
                                   str(test["ticks"]), "--dt-ms", str(dt_ms), "--md", md2, "--tas", tas2] + t02)
            cmd += ["--test-md", md2, "--test-tas", tas2, "--dump-test", dump2]
            if test.get("logs"):
                os.makedirs(os.path.join(d, "logs"))
                cmd += ["--log-dir", os.path.join(d, "logs")]
        day_dumps = []
        for k, t in enumerate(tests or []):
            if "md" in t:
                mdk, task = t["md"], t["tas"]
            else:
                mdk, task = os.path.join(d, "t%d_md_1.csv" % k), os.path.join(d, "t%d_tas_1.csv" % k)
                t0k = [] if t.get("t0_ms") is None else ["--t0-ms", str(t["t0_ms"])]
                subprocess.check_call([FLOW_CSV, "--seed", str(t["flow_seed"]), "--env", str(t["env"]), "--ticks", str(t["ticks"]),
                                       "--dt-ms", str(dt_ms), "--md", mdk, "--tas", task] + t0k)
            day_dumps.append(os.path.join(d, "test_steps_%d.bin" % k))
            cmd += ["--test-md", mdk, "--test-tas", task, "--dump-test", day_dumps[-1]]
            if t.get("symbol"):
                cmd += ["--test-symbol", t["symbol"]]
        want_logs = bool((test or {}).get("logs") or (tests and tests[0].get("logs")))
        if tests and want_logs:
            os.makedirs(os.path.join(d, "logs"))
            cmd += ["--log-dir", os.path.join(d, "logs")]
        out = subprocess.check_output(cmd)
        summary = json.loads(out.decode().strip().splitlines()[-1])
        raw = open(dump, "rb").read()
        n = len(raw) // C.sizeof(abi.StepRecord)
        recs = (abi.StepRecord * n).from_buffer_copy(raw)
        theta = None
        if want_theta:
            import struct
            tr = open(thp, "rb").read()
            theta = {}
            for i in range(0, len(tr), 16):
                idx, val = struct.unpack("<qd", tr[i:i + 16])
                theta[idx] = val
        test_records, logs = None, None
        if want_logs:
            logs = {n: open(os.path.join(d, "logs", n)).read() for n in ("profit_log.csv", "test_stats.csv", "order_log.csv")}
        test_days = [_read_records(p) for p in day_dumps] if tests else None
        if test:
            raw2 = open(dump2, "rb").read()
            n2 = len(raw2) // C.sizeof(abi.StepRecord)
            recs2 = (abi.StepRecord * n2).from_buffer_copy(raw2)
            test_records = [recs2[i] for i in range(n2)]
    return {"records": [recs[i] for i in range(n)], "summary": summary, "theta": theta, "_keep": recs,
            "test_records": test_records, "logs": logs, "test_days": test_days}


def _read_records(path):
    raw = open(path, "rb").read()
    arr = (abi.StepRecord * (len(raw) // C.sizeof(abi.StepRecord))).from_buffer_copy(raw)
    return [arr[i] for i in range(len(arr))]
