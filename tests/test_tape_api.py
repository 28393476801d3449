"""The tape source's C ABI and its Python face, without a GPU: the enum and the three entry points are declared, exported
and bound; null handles are status codes; ingest.day_library concatenates rlm_ingest_csv outputs with the right offsets."""
import ctypes as C
import os
import re

import golden_util as G
from rl_markets_b200 import abi, ingest, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_tape_enum_and_entry_points():
    header = open(os.path.join(ROOT, "include", "rlm.h")).read()
    assert int(re.search(r"RLM_SOURCE_TAPE\s*=\s*(\d+)", header).group(1)) == abi.SOURCE_TAPE == 2
    assert (abi.SOURCE_GENERATOR, abi.SOURCE_STREAM) == (0, 1)
    L = lib.load()
    assert L.rlm_abi_version() == 4
    for name in ("rlm_load_days", "rlm_assign_days", "rlm_get_tape_pos"):
        assert name in lib.EXPORTS and hasattr(L, name), name
    out = (C.c_int64 * 1)()
    offs = (C.c_int64 * 2)(0, 1)
    assert L.rlm_load_days(None, None, offs, 1) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_assign_days(None, 0, 1, (C.c_int32 * 1)(0)) == abi.RLM_ERR_INVALID_ARGUMENT
    assert L.rlm_get_tape_pos(None, out) == abi.RLM_ERR_INVALID_ARGUMENT


def test_day_library_concatenates_the_ingested_pairs():
    samples = [("AAL.L",) + G.ingest_paths(c) for c in G.ingest_manifest()]
    assert len(samples) >= 2
    msgs, offs = ingest.day_library(samples + samples[:1])  # a day may appear twice
    parts = [lib.ingest_csv(md, tas) for _s, md, tas in samples + samples[:1]]
    assert offs[0] == 0 and len(offs) == len(parts) + 1
    for d, (m, n, _t) in enumerate(parts):
        assert offs[d + 1] - offs[d] == n > 300
        size = n * C.sizeof(abi.TickMsg)
        got = (C.c_char * size).from_address(C.addressof(msgs) + offs[d] * C.sizeof(abi.TickMsg)).raw
        assert got == (C.c_char * size).from_address(C.addressof(m)).raw, d
    assert len(msgs) == offs[-1]
