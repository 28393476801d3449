#!/usr/bin/env python3
"""Throughput of Q-value queries (rlm_eval_q: Agent::getQ / DoubleAgent::getQb on any state) on one GPU; prints one JSON
line and writes it to --out.

  Q1  4096 independent Q-learning policies, memory_size 2^16, after bench.py's one-day pretrain (C1's tables)
  Q2  one shared Q-learning table of 2^22 weights (32 MB: resident in an H100's 50 MB L2)
  Q3  Q1 with Double-Q (two tables per policy, 54 gathers per lane and query)

Each case queries 2^22 random states (8 variables, uniform in [-8, 8)) spread over random policies.
  end-to-end   host clock around BatchedMarket.q_values calls: numpy in, numpy out (chunks of RLM_EVAL_Q_CHUNK through
               the handle's staging area), over a window of >= 1 s after a warm-up call
  kernel       device time of rlm_q_kernel alone, summed by torch.profiler (CUDA activities) over >= 1 s of calls
               in a separate pass
The card's name and power limit are read in the same call.  A query gathers 27 weights per lane (54 for Double-Q):
864 (1 728) random 8-byte loads; the bound quoted beside each case is the DRAM random-gather ceiling of
profiles/h100_ubench_gather.txt (32.5 G loads/s) over those loads.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    "Q1": dict(envs=4096, memory_size=1 << 16, shared=False, algo="q_learn", pretrain=108000),
    "Q2": dict(envs=4096, memory_size=1 << 22, shared=True, algo="q_learn", pretrain=4000),
    "Q3": dict(envs=4096, memory_size=1 << 16, shared=False, algo="double_q_learn", pretrain=108000),
}
N_QUERIES = 1 << 22
GATHER_CEILING = 32.5e9  # random 8-byte loads/s from DRAM, profiles/h100_ubench_gather.txt


def card():
    out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"])
    name, limit = [s.strip() for s in out.decode().strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(limit)}


def measure(name, min_seconds):
    import numpy as np
    import torch
    from rl_markets_b200 import abi, config, lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_q.py needs a CUDA device: there is nothing to fall back to")
    w = CASES[name]
    y = config.example_dict(**{"learning.memory_size": w["memory_size"], "learning.algorithm": w["algo"]})
    cfg = config.from_dict(y, n_envs=w["envs"], source=abi.SOURCE_GENERATOR, flow_seed=2024, dt_ms=1, shared_policy=w["shared"])
    m = lib.BatchedMarket(cfg)
    left = w["pretrain"]
    t0 = time.perf_counter()
    while left > 0:
        m.run_ticks(min(left, 512))
        left -= 512
    m.sync()
    pretrain_s = time.perf_counter() - t0
    if w["shared"]:
        fill = float(np.count_nonzero(np.frombuffer(m.theta(0, 0), dtype=np.float64))) / cfg.memory_size
    else:
        o = m.occupancy()
        fill = sum(o) / len(o) / float(cfg.memory_size)
    rng = np.random.default_rng(2024)
    vars_ = rng.uniform(-8.0, 8.0, size=(N_QUERIES, cfg.n_state_vars)).astype(np.float32)
    pol = None if w["shared"] else rng.integers(0, w["envs"], size=N_QUERIES).astype(np.int32)
    q = m.q_values(vars_, pol)  # warm-up (and the staging area's allocation)
    assert np.isfinite(q).all()
    calls, t0 = 0, time.perf_counter()
    while True:
        m.q_values(vars_, pol)
        calls += 1
        e2e_s = time.perf_counter() - t0
        if e2e_s >= min_seconds:
            break
    from torch.profiler import ProfilerActivity, profile
    kcalls, kernel_us = 0, 0.0
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        while kcalls < 2 or time.perf_counter() - t0 < min_seconds:
            m.q_values(vars_, pol)
            kcalls += 1
        torch.cuda.synchronize()
    launches = 0
    for e in prof.events():
        if "rlm_q_kernel" in e.name:
            kernel_us += e.device_time_total
            launches += 1
    m.close()
    gathers = 27 * 32 * (2 if w["algo"] == "double_q_learn" else 1)
    kq = kcalls * N_QUERIES / (kernel_us * 1e-6)
    return {"envs": w["envs"], "memory_size": w["memory_size"], "shared_policy": w["shared"], "algorithm": w["algo"],
            "pretrain_ticks": w["pretrain"], "pretrain_s": pretrain_s, "theta_nonzero_fraction": fill,
            "queries_per_call": N_QUERIES, "e2e_calls": calls, "e2e_s": e2e_s, "e2e_queries_per_s": calls * N_QUERIES / e2e_s,
            "kernel_calls": kcalls, "kernel_launches": launches, "kernel_s": kernel_us * 1e-6, "kernel_queries_per_s": kq,
            "gathers_per_query": gathers, "kernel_gathers_per_s": kq * gathers,
            "dram_gather_bound_queries_per_s": GATHER_CEILING / gathers}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--cases", default="Q1,Q2,Q3")
    ap.add_argument("--min-seconds", dest="min_seconds", type=float, default=1.0)
    ap.add_argument("--out", default=None, help="also write the JSON here")
    args = ap.parse_args()
    cases = [c for c in args.cases.split(",") if c]
    for c in cases:
        if c not in CASES:
            raise SystemExit("unknown case %r (known: %s)" % (c, ", ".join(CASES)))
    res = card()
    res["cases"] = {c: measure(c, args.min_seconds) for c in cases}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
