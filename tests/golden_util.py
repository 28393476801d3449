"""Loaders for tests/golden (fixtures generated from the compiled reference by tools/make_golden.py)."""
import ctypes as C
import hashlib
import json
import os
import struct

from rl_markets_b200 import abi, config

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _all_cases():
    with open(os.path.join(GOLD, "manifest.json")) as f:
        return json.load(f)


def manifest():
    """Single-episode training cases."""
    return [c for c in _all_cases() if not c.get("backtest") and not c.get("multi_episode") and not c.get("ingest")]


def ingest_manifest():
    """Reference runs on CSV pairs with real-data irregularities (tools/messy_csv.py); the pair is committed beside them."""
    return [c for c in _all_cases() if c.get("ingest")]


def ingest_paths(case):
    return os.path.join(GOLD, case["name"] + "_md.csv"), os.path.join(GOLD, case["name"] + "_tas.csv")


def episode_manifest():
    """N training episodes on one Intraday + one Learner-equivalent (main.cpp:45-60)."""
    return [c for c in _all_cases() if c.get("multi_episode")]


def backtest_manifest():
    """Train-until-the-close, then evaluate (main.cpp:216-241) cases."""
    return [c for c in _all_cases() if c.get("backtest")]


def units():
    with open(os.path.join(GOLD, "units.json")) as f:
        return json.load(f)


def records(name):
    raw = open(os.path.join(GOLD, "steps_%s.bin" % name), "rb").read()
    n = len(raw) // C.sizeof(abi.StepRecord)
    arr = (abi.StepRecord * n).from_buffer_copy(raw)
    return [arr[i] for i in range(n)], arr


def record_digest(r):
    """8-byte digest of a StepRecord over exactly the bytes abi.record_fields_equal compares (every field but `pad`)."""
    raw = bytes(r)
    h = hashlib.blake2b(digest_size=8)
    for name, _typ in abi.StepRecord._fields_:
        if name != "pad":
            f = getattr(abi.StepRecord, name)
            h.update(raw[f.offset:f.offset + f.size])
    return h.digest()


def digests(name):
    """Per-record digests of a stored reference run (tests/golden/digests_<name>.bin, written by tools/make_golden.py)."""
    raw = open(os.path.join(GOLD, "digests_%s.bin" % name), "rb").read()
    return [raw[i:i + 8] for i in range(0, len(raw), 8)]


def case_config(case, n_envs=1, env_index0=0, source=abi.SOURCE_GENERATOR):
    return config.from_dict(case["yaml"], n_envs=n_envs, env_index0=env_index0, flow_seed=case["flow_seed"], source=source)


_TILE_VARS = ["pos", "spd", "mpm", "imb", "svl", "vol", "rsi", "vwap", "a_dist", "a_queue", "b_dist", "b_queue", "last_action"]


def tile_config(entry):
    """Config of a units.json tile entry: its memory_size, n_actions and number of state variables (which variables
    they are does not enter tiles(): only their values do)."""
    y = config.example_dict(**{"learning.memory_size": entry["memory_size"], "learning.n_actions": entry["n_actions"],
                               "state.variables": _TILE_VARS[:entry["n_vars"]]})
    return config.from_dict(y)


def tile_vars(case):
    """The state of a units.json tile case as a ctypes float array (stored as bit patterns)."""
    return (C.c_float * len(case["vars"]))(*[C.c_float.from_buffer_copy(C.c_uint32(u)).value for u in case["vars"]])


def hex_to_double(h):
    return struct.unpack("<d", struct.pack("<Q", int(h, 16)))[0]


def double_bits(d):
    return struct.unpack("<Q", struct.pack("<d", d))[0]


def describe_diff(a, b, fields):
    det = []
    for f in fields:
        x, y = getattr(a, f), getattr(b, f)
        if hasattr(x, "_fields_"):
            det.append((f, [(k, getattr(x, k), getattr(y, k)) for k, _ in x._fields_]))
        elif hasattr(x, "__len__"):
            det.append((f, list(x), list(y)))
        else:
            det.append((f, x, y))
    return det
