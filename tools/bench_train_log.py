#!/usr/bin/env python3
"""Cost of the model_log (rlm_set_model_log) at C1's shape: 4096 independent Q-learning policies, memory_size 2^16,
after bench.py's one-day pretrain (108 000 ticks), run in 1024-tick calls (the round-paced engine, CUDA graphs on).

Two handles of the same seed in one process, one with the log on from rlm_create, one without; after the warm-ups the
timed windows alternate between them (log off, log on, log off, ...).  A window is >= --seconds of 1024-tick calls
closed by a device synchronise; env steps/s = learner steps (rlm_counters.steps) over the host clock.  The log-on
handle's rows are drained after each window, outside the timed region.  The accumulation kernel's own time per launch
comes from torch.profiler (CUDA activities) in a separate pass.  The card's name and power limit are read in the same
call.  Prints one JSON line and writes it to --out.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"])
    name, limit = [s.strip() for s in out.decode().strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(limit)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pretrain", type=int, default=108000)
    ap.add_argument("--ticks", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    from rl_markets_b200 import abi, config, lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_log.py needs a CUDA device: there is nothing to fall back to")
    y = config.example_dict(**{"learning.memory_size": 1 << 16, "learning.algorithm": "q_learn"})
    hs = {}
    for key in ("off", "on"):
        cfg = config.from_dict(y, n_envs=4096, source=abi.SOURCE_GENERATOR, flow_seed=2024, dt_ms=1)
        m = lib.BatchedMarket(cfg)
        if key == "on":
            m.set_model_log(4096)
        left = args.pretrain
        while left > 0:
            m.run_ticks(min(left, 512))
            left -= 512
        m.sync()
        for _ in range(args.warmup):
            m.run_ticks(args.ticks)
        m.sync()
        if key == "on":
            m.model_log()
        hs[key] = m

    def window(m):
        c0, t0, calls = m.counters(), time.perf_counter(), 0
        while True:
            m.run_ticks(args.ticks)
            calls += 1
            if calls % 4 == 0:
                m.sync()
                if time.perf_counter() - t0 >= args.seconds:
                    break
        dt = time.perf_counter() - t0
        return (m.counters().steps - c0.steps) / dt

    rates = {"off": [], "on": []}
    rows = 0
    for _ in range(args.windows):
        for key in ("off", "on"):
            rates[key].append(window(hs[key]))
            if key == "on":
                rows += sum(len(v) for v in hs["on"].model_log())
    assert rows > 0
    # the accumulation kernel alone: device time per launch from torch.profiler, in a pass of its own
    from torch.profiler import ProfilerActivity, profile
    m = hs["on"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(4):
            m.run_ticks(args.ticks)
        m.sync()
    m.model_log()
    k_us, k_n = 0.0, 0
    for ev in prof.key_averages():
        if ev.key.startswith("rlm_model_log_kernel") or "rlm_model_log_kernel" in ev.key:
            k_us += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
            k_n += ev.count
    med = {k: sorted(v)[len(v) // 2] for k, v in rates.items()}
    res = dict(card(), workload="C1 (4096 envs, q_learn, M=2^16, after a one-day pretrain), %d-tick calls" % args.ticks,
               env_steps_per_s_log_off=rates["off"], env_steps_per_s_log_on=rates["on"],
               median_off=med["off"], median_on=med["on"], overhead_frac=1.0 - med["on"] / med["off"],
               model_log_kernel_us_per_launch=(k_us / k_n) if k_n else None, model_log_kernel_launches_profiled=k_n,
               rows_logged_in_windows=rows)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
