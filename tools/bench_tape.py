"""Tape source vs in-kernel generator at bench.py's C1 shape (4096 envs, Q-learning, memory_size 2^16, after the same
one-day pretrain); prints one JSON line.

The tape library holds D synthetic days rendered on the host with rlm_flow_generate (day d = the flow of env index d,
long enough for the whole run); env b replays day b % D.  Envs b < D therefore see exactly the messages the generator
evaluates for them, so their weights after the run must equal the generator run's bit for bit (checked on a sample).
Three runs in one process, one after the other: generator, tape, and tape without the L2 prefetch of each env's next
message (RLM_TAPE_PREFETCH=0).  Times are CUDA events around the timed run calls on the launching stream.

    python tools/bench_tape.py [--steps 20] [--warmup 3] [--days 64]
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
    args = ap.parse_args()
    import torch
    from rl_markets_b200 import abi, config, lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_tape.py: no CUDA device; the hot path has no CPU fallback")
    B, D, M, K = args.envs, min(args.days, args.envs), args.memory_size, args.ticks
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": "q_learn"})

    def make_cfg(source):  # bench.py make_cfg: flow seed 2024, 1 ms rows (no env reaches the close)
        return config.from_dict(y, n_envs=B, env_index0=0, source=source, flow_seed=2024, dt_ms=1)

    day_len = args.pretrain + (args.warmup + args.steps) * K
    L = lib.load()
    flow = make_cfg(abi.SOURCE_TAPE).flow
    t0 = time.time()
    lib_msgs = (abi.TickMsg * (D * day_len))()
    size = C.sizeof(abi.TickMsg)
    for d in range(D):
        dst = C.cast(C.addressof(lib_msgs) + d * day_len * size, C.POINTER(abi.TickMsg))
        lib.check(L.rlm_flow_generate(C.byref(flow), d, 0, day_len, dst))
    render_s = time.time() - t0
    offsets = [d * day_len for d in range(D + 1)]
    sample = sorted({0, D // 2, D - 1})
    stream = torch.cuda.Stream()

    def run(source, prefetch=True):
        if prefetch:
            os.environ.pop("RLM_TAPE_PREFETCH", None)
        else:
            os.environ["RLM_TAPE_PREFETCH"] = "0"
        m = lib.BatchedMarket(make_cfg(source))
        os.environ.pop("RLM_TAPE_PREFETCH", None)
        m.set_stream(stream.cuda_stream)
        upload_s = None
        if source == abi.SOURCE_TAPE:
            t = time.time()
            m.load_days(lib_msgs, offsets)
            upload_s = time.time() - t
        left = args.pretrain
        while left > 0:
            m.run_ticks(min(left, 512))
            left -= 512
        for _ in range(args.warmup):
            m.run_ticks(K)
        m.sync()
        c0 = m.counters()
        ev_a, ev_b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            ev_a.record(stream)
            for _ in range(args.steps):
                m.run_ticks(K)
            ev_b.record(stream)
        torch.cuda.synchronize()
        m.sync()
        c1 = m.counters()
        ms = ev_a.elapsed_time(ev_b)
        out = {"steps_per_s": (c1.steps - c0.steps) / (ms * 1e-3), "ticks_per_s": (c1.ticks - c0.ticks) / (ms * 1e-3),
               "ms": ms, "upload_s": upload_s, "theta": [bytes(m.theta(b)) for b in sample]}
        if source == abi.SOURCE_TAPE:
            pos = m.tape_pos()
            out["all_envs_at_day_end"] = pos == [day_len] * B
        m.close()
        return out

    gen = run(abi.SOURCE_GENERATOR)
    tape = run(abi.SOURCE_TAPE)
    tape_nopf = run(abi.SOURCE_TAPE, prefetch=False)
    res = {
        "workload": "C1 shape: %d envs, q_learn + tile coding (32 tilings, memory_size %d per env), %d-tick pretrain, %d timed run "
                    "calls of %d ticks" % (B, M, args.pretrain, args.steps, K),
        "gpu": torch.cuda.get_device_name(0),
        "unit": "env_steps/s",
        "generator": gen["steps_per_s"],
        "tape": tape["steps_per_s"],
        "tape_no_l2_prefetch": tape_nopf["steps_per_s"],
        "tape_over_generator": tape["steps_per_s"] / gen["steps_per_s"],
        "ticks_per_s": {"generator": gen["ticks_per_s"], "tape": tape["ticks_per_s"], "tape_no_l2_prefetch": tape_nopf["ticks_per_s"]},
        "days": D, "messages_per_day": day_len, "library_mb": D * day_len * size / 1e6,
        "render_s": render_s, "upload_s": tape["upload_s"],
        "theta_equal": all(a == b for a, b in zip(gen["theta"], tape["theta"])) and all(a == b for a, b in zip(gen["theta"], tape_nopf["theta"])),
        "theta_sampled_envs": sample,
        "tape_envs_at_day_end": tape["all_envs_at_day_end"] and tape_nopf["all_envs_at_day_end"],
        "timing": "CUDA events around the timed run calls on the launching stream",
        "power_limit_w": _smi("power.limit"), "sm_mhz_after": _smi("clocks.sm"),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
