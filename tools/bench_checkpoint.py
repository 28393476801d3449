#!/usr/bin/env python3
"""Cost and size of a checkpoint (rlm_save / rlm_load) at two shapes:
  K1  C1: 4096 independent Q-learning policies of 2^16 weights after bench.py's one-day pretrain (108 000 ticks)
  K2  one shared Q-learning table of 2^22 weights over 4096 envs after a 4000-tick pretrain

For each: the wall time of rlm_save and of rlm_load into a second handle of the same config, each closed by a device
synchronise (host clock, median of --reps), the file's bytes and its packed weight tables' bytes against the tables' dense size, and the
device time of the pack and unpack kernels per call from torch.profiler (CUDA activities) in a pass of its own.  The
loaded handle's weight tables are checked against the saved handle's.  Files go to a temporary directory, removed at
the end.  The card's name and power limit are read in the same call.  Prints one JSON line and writes it to --out.
"""
import argparse
import json
import os
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = {
    "K1": dict(envs=4096, memory_size=1 << 16, shared=False, pretrain=108000),
    "K2": dict(envs=4096, memory_size=1 << 22, shared=True, pretrain=4000),
}
PACK = ("rlm_pack_count_kernel", "rlm_ck_scan_kernel", "rlm_pack_kernel")
UNPACK = ("rlm_unpack_count_kernel", "rlm_ck_scan_kernel", "rlm_unpack_kernel")


def card():
    out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"])
    name, limit = [s.strip() for s in out.decode().strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit_w": float(limit)}


def kernel_us(prof, names):
    out = {}
    for ev in prof.key_averages():
        for n in names:
            if n in ev.key:
                t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
                out[n] = out.get(n, 0.0) + t
    return out


def table_bytes(path):
    """bytes of the packed weight-table sections (ids 64..66) of a checkpoint's section table"""
    with open(path, "rb") as f:
        head = f.read(28)
        n_sec, header_bytes = struct.unpack_from("<I", head, 12)[0], struct.unpack_from("<I", head, 24)[0]
        f.seek(header_bytes - 32 * n_sec)
        secs = [struct.unpack("<IIQQQ", f.read(32)) for _ in range(n_sec)]
    return sum(s[3] for s in secs if s[0] >= 64)


def run_case(key, w, reps, tmp):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from rl_markets_b200 import abi, config, lib
    y = config.example_dict(**{"learning.memory_size": w["memory_size"], "learning.algorithm": "q_learn"})
    cfg = config.from_dict(y, n_envs=w["envs"], source=abi.SOURCE_GENERATOR, flow_seed=2024, dt_ms=1, shared_policy=w["shared"])
    m = lib.BatchedMarket(cfg)
    left = w["pretrain"]
    while left > 0:
        m.run_ticks(min(left, 512))
        left -= 512
    m.sync()
    n = lib.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
    path = os.path.join(tmp, key + ".rlm")
    save_s, load_s = [], []
    for _ in range(reps + 1):  # (the first pair warms up)
        t0 = time.perf_counter()
        m.save(path)
        m.sync()
        save_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        n.load(path)
        n.sync()
        load_s.append(time.perf_counter() - t0)
    save_s, load_s = save_s[1:], load_s[1:]
    policies = 1 if w["shared"] else w["envs"]
    for p in sorted({0, policies // 2, policies - 1}):
        assert bytes(n.theta(p)) == bytes(m.theta(p)), p
    size, tables = os.path.getsize(path), table_bytes(path)
    dense = policies * w["memory_size"] * 8 + (w["memory_size"] * 8 if w["shared"] else 0)  # (+ dtheta of a shared policy)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.save(path)
        torch.cuda.synchronize()
    pk = kernel_us(prof, PACK)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        n.load(path)
        torch.cuda.synchronize()
    uk = kernel_us(prof, UNPACK + ("rlm_fingerprint_kernel",))
    n.close()
    m.close()
    os.remove(path)
    med = lambda v: sorted(v)[len(v) // 2]
    return {"envs": w["envs"], "memory_size": w["memory_size"], "shared_policy": w["shared"], "pretrain_ticks": w["pretrain"],
            "save_s": save_s, "load_s": load_s, "save_s_median": med(save_s), "load_s_median": med(load_s),
            "file_bytes": size, "packed_table_bytes": tables, "dense_table_bytes": dense, "tables_over_dense": tables / dense,
            "other_section_bytes": size - tables,
            "pack_kernels_us_per_save": sum(pk.values()), "pack_kernels_us": pk,
            "unpack_kernels_us_per_load": sum(uk.values()), "unpack_kernels_us": uk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="K1,K2")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=None, help="where the checkpoint files go (default: a temporary directory)")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpoint.py needs a CUDA device: there is nothing to fall back to")
    res = card()
    with tempfile.TemporaryDirectory(dir=args.dir) as tmp:
        for key in args.cases.split(","):
            res[key] = run_case(key, CASES[key], args.reps, tmp)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
