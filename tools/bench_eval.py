#!/usr/bin/env python3
"""Throughput of greedy evaluation (backtest mode) on one GPU; prints one JSON line.

  E1      C1's shape -- 4096 envs, independent Q-learning policies, memory_size 2^16 -- after bench.py's one-day pretrain
  E2      the same 4096 envs under ONE shared table of 2^22 weights (32 MB: resident in an H100's 50 MB L2)
  E2_32k  32 768 envs (C3's per-GPU shard, thread-per-env tick kernel) under one shared table of 2^22 weights

Every case: train, GoGreedy, backtest mode, a new env; >= 3 warm-up calls; then CUDA events around calls of rlm_run_ticks
until the timed window is >= 1 s, ended by rlm_sync; then a separate profiled pass (rlm_set_profiling) for the per-kernel
averages.  dt_ms = 1, so no env reaches the close inside the run.  The card's name and power limit are read in the same
call.  --lib PATH measures another build of librlm.so; --alternate-with PATH runs E1 in child processes alternately on
this tree's library and on PATH (a build of the parent commit, say), so that the two share the machine's state.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    "E1": dict(envs=4096, memory_size=1 << 16, shared=False, pretrain=108000),
    "E2": dict(envs=4096, memory_size=1 << 22, shared=True, pretrain=4000),
    "E2_32k": dict(envs=32768, memory_size=1 << 22, shared=True, pretrain=1000),
}
TICKS_PER_CALL = 1024


def card():
    out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"])
    name, limit = [s.strip() for s in out.decode().strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(limit)}


def measure(name, min_seconds):
    import numpy as np
    import torch
    from rl_markets_b200 import abi, config, lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device: there is nothing to fall back to")
    w = CASES[name]
    y = config.example_dict(**{"learning.memory_size": w["memory_size"], "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=w["envs"], source=abi.SOURCE_GENERATOR, flow_seed=2024, dt_ms=1, shared_policy=w["shared"])
    stream = torch.cuda.Stream()
    m = lib.BatchedMarket(cfg)
    m.set_stream(stream.cuda_stream)
    left = w["pretrain"]
    while left > 0:
        m.run_ticks(min(left, 512))
        left -= 512
    m.sync()
    if w["shared"]:
        fill = float(np.count_nonzero(np.frombuffer(m.theta(0, 0), dtype=np.float64))) / cfg.memory_size
    else:
        o = m.occupancy()
        fill = sum(o) / len(o) / float(cfg.memory_size)
    m.go_greedy()
    m.set_mode(abi.MODE_BACKTEST)
    m.new_env(None)
    for _ in range(3):
        m.run_ticks(TICKS_PER_CALL)
    m.sync()
    c0 = m.counters()
    ms, calls = 0.0, 0
    while ms < 1000.0 * min_seconds:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            a.record(stream)
            for _ in range(8):
                m.run_ticks(TICKS_PER_CALL)
            b.record(stream)
        m.sync()
        ms += a.elapsed_time(b)
        calls += 8
    c1 = m.counters()
    m.set_profiling(True)
    for _ in range(2):
        m.run_ticks(TICKS_PER_CALL)
    m.sync()
    k = m.kernel_times()
    m.close()
    steps, ticks = c1.steps - c0.steps, c1.ticks - c0.ticks
    return {"envs": w["envs"], "memory_size": w["memory_size"], "shared_policy": w["shared"], "pretrain_ticks": w["pretrain"],
            "theta_nonzero_fraction": fill, "timed_ms": ms, "calls": calls, "ticks_per_call": TICKS_PER_CALL,
            "eval_steps": int(steps), "eval_steps_per_s": steps / (ms * 1e-3), "env_ticks_per_s": ticks / (ms * 1e-3),
            "tick_kernel_us": 1e3 * k["env_ms"] / max(k["env_launches"], 1),
            "eval_kernel_us": 1e3 * k["agent_ms"] / max(k["agent_launches"], 1),
            "steps_per_eval_launch": steps / float(calls * TICKS_PER_CALL)}


def child(case, lib_path, min_seconds):
    env = dict(os.environ)
    if lib_path:
        env["RLM_LIB_PATH"] = os.path.abspath(lib_path)
    out = subprocess.check_output([sys.executable, os.path.abspath(__file__), "--cases", case, "--raw", "--min-seconds", str(min_seconds)], env=env)
    return json.loads(out.decode().strip().splitlines()[-1])[case]


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--cases", default="E1,E2,E2_32k")
    ap.add_argument("--lib", default=None, help="measure this librlm.so instead of the tree's")
    ap.add_argument("--alternate-with", dest="other", default=None, help="E1 alternately on the tree's library and on this one")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of --alternate-with")
    ap.add_argument("--min-seconds", dest="min_seconds", type=float, default=1.0)
    ap.add_argument("--raw", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.lib:
        os.environ["RLM_LIB_PATH"] = os.path.abspath(args.lib)
    cases = [c for c in args.cases.split(",") if c]
    for c in cases:
        if c not in CASES:
            raise SystemExit("unknown case %r (known: %s)" % (c, ", ".join(CASES)))
    if args.raw:
        print(json.dumps({c: measure(c, args.min_seconds) for c in cases}))
        return
    res = card()
    res["library"] = os.environ.get("RLM_LIB_PATH") or "rl_markets_b200/librlm.so"
    res["cases"] = {}
    for c in cases:
        if c == "E1" and args.other:
            runs = {"this": [], "other": []}
            for _ in range(args.rounds):
                runs["this"].append(child("E1", args.lib, args.min_seconds))
                runs["other"].append(child("E1", args.other, args.min_seconds))
            res["cases"]["E1"] = runs["this"][0]
            res["cases"]["E1_alternating"] = {
                "other_library": args.other,
                "this_eval_steps_per_s": [r["eval_steps_per_s"] for r in runs["this"]],
                "other_eval_steps_per_s": [r["eval_steps_per_s"] for r in runs["other"]],
                "this_eval_kernel_us": [r["eval_kernel_us"] for r in runs["this"]],
                "other_eval_kernel_us": [r["eval_kernel_us"] for r in runs["other"]],
                "this_tick_kernel_us": [r["tick_kernel_us"] for r in runs["this"]],
                "other_tick_kernel_us": [r["tick_kernel_us"] for r in runs["other"]]}
        else:
            res["cases"][c] = child(c, args.lib, args.min_seconds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
