#!/usr/bin/env python3
"""Per-warp phase timeline of rlm_learn_kernel (the RLM_TIMING build: see rl_markets_b200/csrc/Makefile).

    RLM_LIB_PATH=rl_markets_b200/librlm_timing.so python tools/phase_probe_learn.py [pretrain_ticks] [envs] [M] [algo] [ticks]

Trains `pretrain_ticks` ticks per env (default 108000: C1's one-day pretrain), then runs calls of `ticks` ticks (default
256: the round-paced engine at C1) and reads the LPH marks of the learner's last launches.  The marks of one launch are
told apart from older ones by time, SM by SM (clock64 is a per-SM counter): launches on one stream do not overlap, so
an SM's warps are split where a warp starts after every earlier one has ended, and each SM's largest launch is shown.
Then, on the same trained state, the launch times of both kernels under the what-if switches of D.debug_flags
(rlm_debug_set_flags; 1 = every env gathers from ONE table, L2-resident; 4 = no patch of the second evaluation;
5 = both).  The switches make results wrong: they run last.
"""
import ctypes as C, sys, numpy as np
sys.path.insert(0, '.')
from rl_markets_b200 import config, lib
pre = int(sys.argv[1]) if len(sys.argv) > 1 else 108000
B = int(sys.argv[2]) if len(sys.argv) > 2 else 4096
M = int(sys.argv[3]) if len(sys.argv) > 3 else 65536
algo = sys.argv[4] if len(sys.argv) > 4 else "q_learn"
T = int(sys.argv[5]) if len(sys.argv) > 5 else 256
y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
cfg = config.from_dict(y, n_envs=B, flow_seed=1, dt_ms=1)
m = lib.BatchedMarket(cfg)
left = pre
while left > 0:
    m.run_ticks(min(left, 512)); left -= 512
m.sync()
L = m.L
L.rlm_debug_read_phases.argtypes = [C.c_void_p, C.c_void_p]
L.rlm_debug_set_flags.argtypes = [C.c_void_p, C.c_int32]
# marks in the order a stage-0 step writes them (ln_step)
order = [0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 14, 10, 11, 12]
names = ["stage AgentD", "hash", "gather issue", "tile table (under the gathers)", "gather wait + store", "sums", "TD",
         "trace pass", "threadfence", "advance state", "patch", "syncwarp", "sums 2", "write-back"]


def last_launch(a, sm):
    # clock64 is a per-SM counter: the launches are told apart on each SM, and each SM's largest launch is kept
    ok = (np.diff(a[:, order], axis=1) >= 0).all(axis=1) & (a[:, 12] > a[:, 0])
    out, spans = [], []
    for s in np.unique(sm[ok]):
        b = a[ok & (sm == s)]
        b = b[np.argsort(b[:, 0])]
        cut = np.nonzero(b[1:, 0] > np.maximum.accumulate(b[:-1, 12]))[0] + 1
        b = max(np.split(b, cut), key=len)
        out.append(b)
        spans.append(b[:, 12].max() - b[:, 0].min())
    return np.concatenate(out), np.array(spans)


def timeline(tag):
    clk = (C.c_longlong * (4096 * 16))(); sm = (C.c_uint * 4096)()
    assert L.rlm_debug_read_phases(clk, sm) == 0
    a, spans = last_launch(np.frombuffer(clk, dtype=np.int64).reshape(4096, 16).copy(), np.frombuffer(sm, dtype=np.uint32).copy())
    d = np.diff(a[:, order], axis=1)
    dur = a[:, 12] - a[:, 0]
    print("%s: stage-0 steps %d on %d SMs  mean step %.0f cycles (max %d)  SM span of the launch mean %.0f max %d cycles" % (
        tag, len(a), len(spans), dur.mean(), dur.max(), spans.mean(), spans.max()))
    for i, n in enumerate(names):
        print("  %-32s mean %8.0f  p50 %8.0f  p90 %8.0f  max %8.0f  (%4.1f %%)" % (
            n, d[:, i].mean(), np.percentile(d[:, i], 50), np.percentile(d[:, i], 90), d[:, i].max(), 100.0 * d[:, i].mean() / dur.mean()))
    post = a[:, 12] - a[:, 7]
    print("  after the TD step (trace pass .. write-back): mean %.0f cycles (%.1f %% of a step)" % (post.mean(), 100.0 * post.mean() / dur.mean()))
    if a[:, 15].any():  # (builds that record whether the second sums ran)
        print("  second sums taken in %.1f %% of the steps" % (100.0 * a[:, 15].mean()))


for rep in range(3):
    m.run_ticks(T); m.sync()
    timeline("rep %d" % rep)
for flags in (0, 4, 1, 5):
    assert L.rlm_debug_set_flags(m.h, flags) == 0
    m.run_ticks(T); m.sync()  # (warm: the same engine, state under these switches)
    m.set_profiling(True)
    m.run_ticks(T); m.sync()
    kt = m.kernel_times()
    m.set_profiling(False)
    print("debug_flags %d: learner %.1f us/launch (%d launches)  tick kernel %.1f us/launch (%d launches)" % (
        flags, 1e3 * kt["agent_ms"] / max(kt["agent_launches"], 1), kt["agent_launches"],
        1e3 * kt["env_ms"] / max(kt["env_launches"], 1), kt["env_launches"]))
    m.run_ticks(T); m.sync()
    timeline("  timeline under debug_flags %d" % flags)
m.close()
