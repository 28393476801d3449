"""Cost of day markets (rlm_set_day_markets) at bench.py's C1 shape on the tape source, as in tools/bench_tape.py: 4096 envs,
Q-learning, memory_size 2^16, a one-day pretrain, a library of 64 synthetic days (rlm_flow_generate, env b on day b % 64).
Prints one JSON line.

Three arms, run one after the other in one process, the sequence twice:
  none   no day markets: the tick kernels read the config's market from the __constant__ block;
  same   every day under a copy of the config's market: the MKT tick kernels read each env's VenueD from global memory,
         with the same results -- theta of sampled envs must equal arm `none` bit for bit;
  split  even days under LSE group A (the config's, AAL.L), odd days under LSE group B (BAES.L): the synthetic prices
         lie in [1000, 5000), where the two tables quote 0.5 against 1.0.
Env steps/s from CUDA events around the timed run calls; per-kernel times from rlm_set_profiling in a second pass of
the timed calls.  The card's name and power limit are read in the same call.

    python tools/bench_markets.py [--steps 20] [--warmup 3] [--days 64]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _smi(field):
    """one read-only nvidia-smi query of GPU 0 (None where nvidia-smi is unavailable)"""
    import subprocess
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=" + field, "--format=csv,noheader,nounits"], timeout=10)
        return float(out.decode().strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--days", type=int, default=64)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--memory-size", dest="memory_size", type=int, default=65536)
    ap.add_argument("--pretrain", type=int, default=108000)
    ap.add_argument("--ticks", type=int, default=1024, help="ticks per timed run call (bench.py C1: 1024)")
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch
    from rl_markets_b200 import abi, config, lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_markets.py: no CUDA device; the hot path has no CPU fallback")
    B, D, M, K = args.envs, min(args.days, args.envs), args.memory_size, args.ticks
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": "q_learn", "data.symbols": ["AAL.L"]})

    def make_cfg():  # bench.py make_cfg: flow seed 2024, 1 ms rows (no env reaches the close)
        return config.from_dict(y, n_envs=B, env_index0=0, source=abi.SOURCE_TAPE, flow_seed=2024, dt_ms=1)

    day_len = args.pretrain + 2 * (args.warmup + args.steps) * K
    L = lib.load()
    flow = make_cfg().flow
    lib_msgs = (abi.TickMsg * (D * day_len))()
    size = C.sizeof(abi.TickMsg)
    for d in range(D):
        dst = C.cast(C.addressof(lib_msgs) + d * day_len * size, C.POINTER(abi.TickMsg))
        lib.check(L.rlm_flow_generate(C.byref(flow), d, 0, day_len, dst))
    offsets = [d * day_len for d in range(D + 1)]
    sample = sorted({0, 1, D // 2, D - 1, B - 1})
    stream = torch.cuda.Stream()
    arms = {
        "none": None,
        "same": ([config.config_market(make_cfg())], [0] * D),
        "split": ([config.market("AAL.L"), config.market("BAES.L")], [d % 2 for d in range(D)]),
    }

    def timed(m):
        ev_a, ev_b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        c0 = m.counters()
        with torch.cuda.stream(stream):
            ev_a.record(stream)
            for _ in range(args.steps):
                m.run_ticks(K)
            ev_b.record(stream)
        torch.cuda.synchronize()
        m.sync()
        c1 = m.counters()
        return (c1.steps - c0.steps) / (ev_a.elapsed_time(ev_b) * 1e-3)

    def run(arm):
        m = lib.BatchedMarket(make_cfg())
        m.set_stream(stream.cuda_stream)
        m.load_days(lib_msgs, offsets)
        if arms[arm] is not None:
            m.set_day_markets(*arms[arm])
        left = args.pretrain
        while left > 0:
            m.run_ticks(min(left, 512))
            left -= 512
        for _ in range(args.warmup):
            m.run_ticks(K)
        m.sync()
        sps = timed(m)
        m.set_profiling(1)
        timed(m)
        kt = m.kernel_times()
        m.set_profiling(0)
        out = {"steps_per_s": sps, "kernel_times": kt, "theta": [bytes(m.theta(b)) for b in sample]}
        m.close()
        return out

    res = {a: [] for a in arms}
    for _r in range(args.rounds):
        for a in arms:
            res[a].append(run(a))
    out = {
        "workload": "C1 shape on the tape source: %d envs, q_learn + tile coding (32 tilings, memory_size %d per env), %d days, "
                    "%d-tick pretrain, %d timed run calls of %d ticks" % (B, M, D, args.pretrain, args.steps, K),
        "gpu": torch.cuda.get_device_name(0), "power_limit_w": _smi("power.limit"),
        "unit": "env_steps/s",
        "steps_per_s": {a: [r["steps_per_s"] for r in rs] for a, rs in res.items()},
        "kernel_times": {a: [r["kernel_times"] for r in rs] for a, rs in res.items()},
        "same_theta_equals_none": all(r["theta"] == res["none"][0]["theta"] for r in res["same"] + res["none"]),
        "theta_sampled_envs": sample,
        "order": "arms none, same, split in turn, %d times, one process" % args.rounds,
        "timing": "CUDA events around the timed run calls on the launching stream; kernel times from rlm_set_profiling in a "
                  "second pass of the timed calls",
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
