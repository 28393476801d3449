"""Checkpoint files held to the NumPy model of their format (tests/checkpoint_format.py), at the shapes where the pack,
unpack, scan and fingerprint kernels and the two-buffer chunk pipeline of rlm_checkpoint.cu reach their edges.

Every weight table is written through write_theta with a seeded pattern; the saved file's packed bytes must be the
model's, bit for bit.  The file is then loaded into a handle whose tables hold nonzero junk: every table must come back
exactly (so clear bits must be written as +0.0), and that handle saves the same bytes again.  Corrupt files are refused
and leave the loading handle as it was.  Then a resume across 16 chunks, and one saved under sub-batches."""
import ctypes as C
import shutil

import numpy as np
import pytest

import checkpoint_format as ckf
from rl_markets_b200 import abi, config, lib
from test_gpu_checkpoint import Setup, _assert_same, _code, _do, _observe
from test_gpu_checkpoint import _cfg as _ck_cfg

pytestmark = pytest.mark.gpu

CHUNK = 1 << 22  # RLM_CK_CHUNK: the most words of one chunk of the pipeline, and the slice length of a larger table
THETA, THETA_B, DTHETA = ckf.THETA, ckf.THETA_B, ckf.DTHETA

# -0.0, quiet and signalling NaNs of both signs with payloads, +-inf, the smallest and the largest denormal
SPECIAL = np.array([0x8000000000000000, 0x7FF80000DEADBEEF, 0xFFF80000000000FF, 0x7FF0000000000001, 0xFFF4000000C0FFEE,
                    0x7FF0000000000000, 0xFFF0000000000000, 0x0000000000000001, 0x800FFFFFFFFFFFFF], dtype=np.uint64)
PATTERNS = ("zero", "dense", "first", "last", "edges", "sparse", "half")

# id: (algorithm, n_envs, memory_size, shared policy, the patterns its tables take in turn)
SHAPES = {
    # 4096 one-word tables per chunk: 4096 blocks, 4 per scan thread; then a chunk of one table; 31 padding bits per table
    "a-q-B4097-M1": ("q_learn", 4097, 1, False, PATTERNS),
    # 4096 + 1 tables of theta and of theta_b: 4 chunks, both buffers reused; 7 padding bits in the last file byte
    "b-double-B4097-M1001": ("double_q_learn", 4097, 1001, False, PATTERNS),
    # a tile one word short, an exact tile, one word into a second tile (511 tables per chunk, 2 chunks)
    "c-q-B600-M8191": ("q_learn", 600, 8191, False, PATTERNS),
    "c-q-B600-M8192": ("q_learn", 600, 8192, False, PATTERNS),
    "c-q-B600-M8193": ("q_learn", 600, 8193, False, PATTERNS),
    # the largest table that is not sliced, a table of exactly one chunk, a table with a one-word second slice
    "d-double-B2-M4194303": ("double_q_learn", 2, CHUNK - 1, False, ("edges", "dense", "last", "half")),
    "d-double-B2-M4194304": ("double_q_learn", 2, CHUNK, False, ("edges", "dense", "last", "half")),
    "d-double-B2-M4194305": ("double_q_learn", 2, CHUNK + 1, False, ("edges", "dense", "last", "half")),
    # three full slices and a partial one, for theta and for dtheta: value offsets carried from slice to slice
    "e-shared-B8-M12591106": ("q_learn", 8, 3 * CHUNK + 8194, True, ("half",)),
}


def _cfg(case, flow_seed=7, source=abi.SOURCE_GENERATOR, n_envs=None, mem=None):
    algo, B, M, shared, _kinds = SHAPES[case] if case else ("q_learn", n_envs, mem, False, None)
    y = config.example_dict(**{"learning.memory_size": M, "learning.algorithm": algo})
    cfg = config.from_dict(y, n_envs=B, flow_seed=flow_seed, shared_policy=shared, source=source)
    cfg.record_envs, cfg.record_cap = 2, 1000
    return cfg


def _edges(M):
    e = {31, 32, 1023, 1024, 8191, 8192}
    for k in range(1, M // CHUNK + 1):
        e |= {k * CHUNK - 1, k * CHUNK}
    return sorted(i for i in e if i < M)


def _rand(rng, n):
    v = rng.integers(0, 2**64 - 1, size=n, dtype=np.uint64, endpoint=True)
    v[v == 0] = 1
    return v


def _pattern(kind, M, rng):
    w = np.zeros(M, np.uint64)
    if kind == "dense":
        w[:] = _rand(rng, M)
        w[rng.integers(0, M, size=M // 64)] = 0
        at = rng.integers(0, M, size=min(M, 4 * len(SPECIAL)))
        w[at] = SPECIAL[np.arange(len(at)) % len(SPECIAL)]
    elif kind == "first":
        w[0] = _rand(rng, 1)[0]
    elif kind == "last":
        w[M - 1] = _rand(rng, 1)[0]
    elif kind == "edges":
        e = _edges(M)
        w[e] = _rand(rng, len(e))
    elif kind in ("sparse", "half"):
        at = np.flatnonzero(rng.random(M) < (1e-3 if kind == "sparse" else 0.5))
        w[at] = _rand(rng, len(at))
    else:
        assert kind == "zero", kind
    return w


def _junk(k, M):
    """nonzero finite words, different from table to table"""
    return np.random.default_rng([99, k]).uniform(0.5, 1.5, M) * np.where(np.arange(M) % 3 == 0, -1.0, 1.0)


def _order(m):
    """(section id, policy) of every written table, in file order"""
    pol = 1 if m.cfg.shared_policy else m.cfg.n_envs
    return [(sid, p) for sid in (THETA, THETA_B)[:m.n_tables] for p in range(pol)]


def _write(m, sid, p, w):
    m.write_theta((C.c_double * len(w)).from_buffer(w), p, sid - THETA)


def _read(m, sid, p):
    return np.frombuffer(m.theta(p, sid - THETA), np.uint64)


def _accumulate_a_step(m):
    """rlm_shared_tick_accumulate until a tick's learner updates add traces to dtheta, so that it is not empty (the
    step counter moves in rlm_apply_dtheta, the trace sum in the accumulation)"""
    for _ in range(1000):
        s0 = m.counters().sum_traces
        m.shared_tick_accumulate()
        if m.counters().sum_traces > s0:
            return
        m.apply_dtheta()
    raise AssertionError("no learner update in 1000 ticks")


def _junk_handle(case):
    """a handle of the case's config (another flow) with junk in every table; on a shared policy, a dtheta of its own"""
    m = lib.BatchedMarket(_cfg(case, flow_seed=11))
    for k, (sid, p) in enumerate(_order(m)):
        _write(m, sid, p, _junk(k, m.cfg.memory_size))
    if m.cfg.shared_policy:
        _accumulate_a_step(m)
    return m


def _assert_junk(m, case):
    for k, (sid, p) in enumerate(_order(m)):
        assert _read(m, sid, p).tobytes() == _junk(k, m.cfg.memory_size).tobytes(), (case, sid, p)


class Saved:
    def __init__(self, case, path, tables, theta_after):
        self.case, self.path, self.tables, self.theta_after = case, path, tables, theta_after


@pytest.fixture(scope="module")
def saved(tmp_path_factory):
    """the file of each case (built once per module): every table written with its pattern, then rlm_save.  A shared
    policy saves between rlm_shared_tick_accumulate and rlm_apply_dtheta, and keeps theta after that apply."""
    done = {}

    def get(case):
        if case not in done:
            _algo, _B, M, shared, kinds = SHAPES[case]
            m = lib.BatchedMarket(_cfg(case))
            if shared:
                _write(m, THETA, 0, _junk(0, M))  # (weights that are not all zero: the step's update is not zero)
                _accumulate_a_step(m)
            tables = {}
            for k, (sid, p) in enumerate(_order(m)):
                w = _pattern(kinds[k % len(kinds)], M, np.random.default_rng([list(SHAPES).index(case), k]))
                _write(m, sid, p, w)
                tables[(sid, p)] = w
            path = str(tmp_path_factory.mktemp("ck") / (case + ".rlm"))
            m.save(path)
            after = None
            if shared:
                m.apply_dtheta()
                after = _read(m, THETA, 0).copy()
            m.close()
            done[case] = Saved(case, path, tables, after)
        return done[case]

    return get


def _first_diff(a, b):
    d = np.flatnonzero(np.frombuffer(a, np.uint8)[:min(len(a), len(b))] != np.frombuffer(b, np.uint8)[:min(len(a), len(b))])
    return int(d[0]) if len(d) else min(len(a), len(b))


@pytest.mark.parametrize("case", list(SHAPES))
def test_file_matches_the_model_and_loads_over_junk(rlm, saved, tmp_path, case):
    s = saved(case)
    M = SHAPES[case][2]
    f = ckf.File.read(s.path)
    assert f.magic == ckf.MAGIC and f.file_bytes == len(f.data)
    pos = f.header_bytes
    for sec in f.sections:
        assert sec[2] == pos, (case, sec)
        pos += sec[3]
    assert pos == f.file_bytes
    tabs = f.tables()
    assert f.sections[-len(tabs):] == tabs and all(sec[0] < THETA for sec in f.sections[:-len(tabs)])
    want_ids = list(s.tables) + ([(DTHETA, 0)] if s.theta_after is not None else [])
    assert [(sec[0], sec[1]) for sec in tabs] == want_ids
    for sec in tabs:
        body = f.body(sec)
        if sec[0] == DTHETA:
            dtheta = ckf.unpack(body, M)
            assert 0 < sec[4] == np.count_nonzero(dtheta), (case, sec)
            continue
        w = s.tables[(sec[0], sec[1])]
        want = ckf.packed(w)
        assert sec[4] == np.count_nonzero(w) and sec[3] == len(want), (case, sec)
        if body != want:
            at = _first_diff(body, want)
            raise AssertionError("%s: table %r differs from the model at byte %d of %d (bitmap: %d bytes)" % (case, sec[:2], at, len(want), (M + 7) // 8))
    if s.theta_after is not None:
        # the saved dtheta is the one rlm_apply_dtheta added: theta_after = theta + dtheta, word by word (NaNs as NaNs)
        with np.errstate(all="ignore"):
            want = s.tables[(THETA, 0)].view(np.float64) + dtheta.view(np.float64)
        got = s.theta_after.view(np.float64)
        nan = np.isnan(want)
        assert np.array_equal(nan, np.isnan(got)), case
        assert np.array_equal(want[~nan].view(np.uint64), got[~nan].view(np.uint64)), case
    j = _junk_handle(case)
    j.load(s.path)
    for (sid, p), w in s.tables.items():
        got = _read(j, sid, p)
        if got.tobytes() != w.tobytes():
            bad = np.flatnonzero(got != w)
            raise AssertionError("%s: table %r after the load differs at %d words, first %d" % (case, (sid, p), len(bad), bad[0]))
    again = str(tmp_path / "again.rlm")
    j.save(again)
    with open(again, "rb") as g:
        assert g.read() == f.data, case
    if s.theta_after is not None:
        j.apply_dtheta()
        assert _read(j, THETA, 0).tobytes() == s.theta_after.tobytes(), case
    j.close()


# ---- corrupt files ---------------------------------------------------------------------------------------------------
def _index(f, sid, p):
    return next(k for k, sec in enumerate(f.sections) if (sec[0], sec[1]) == (sid, p))


def _flipped(f, k, *bits, extra=b"", more=0):
    """section k's bytes with the given bitmap bits flipped (and `extra` value bytes appended, `more` values counted)"""
    b = bytearray(f.body(f.sections[k]))
    for i in bits:
        b[i // 8] ^= 1 << (i % 8)
    return bytes(b) + extra, f.sections[k][4] + more


def _words(f, k, case):
    return ckf.unpack(f.body(f.sections[k]), SHAPES[case][2])


def _padding_bit(f, case):
    """a padding bit set in the last byte of table theta[4096] (the second chunk) -- with one more value, so that the
    bitmap's population, padding bit included, equals the stored count: only the padding check can refuse it"""
    M, k = SHAPES[case][2], _index(f, THETA, 4096)
    return {k: _flipped(f, k, 8 * ((M + 7) // 8) - 1, extra=b"\x00\x00\x00\x00\x00\x00\xf0\x3f", more=1)}


def _cleared_in_two_chunks(f, case):
    """one set bit cleared in a table of chunk 0 (theta) and in one of chunk 2 (theta_b)"""
    out = {}
    for sid in (THETA, THETA_B):
        k = next(k for p in range(1, 4096) for k in [_index(f, sid, p)] if f.sections[k][4] > 0)
        out[k] = _flipped(f, k, int(np.flatnonzero(_words(f, k, case))[0]))
    return out


def _moved_bit(f, case):
    """a set bit of theta[1] cleared and a clear bit of theta[2] set: the chunk's total population is right, the two
    tables' are not"""
    k1, k2 = _index(f, THETA, 1), _index(f, THETA, 2)
    return {k1: _flipped(f, k1, int(np.flatnonzero(_words(f, k1, case))[0])),
            k2: _flipped(f, k2, int(np.flatnonzero(_words(f, k2, case) == 0)[0]))}


def _slice_bit(f, case):
    """one bitmap bit flipped in the second slice of the last table (dtheta)"""
    k = len(f.sections) - 1
    return {k: _flipped(f, k, CHUNK + 12345)}


REJECT = {
    "padding-bit": ("b-double-B4097-M1001", _padding_bit),
    "cleared-bits-two-chunks": ("b-double-B4097-M1001", _cleared_in_two_chunks),
    "moved-bit-one-chunk": ("b-double-B4097-M1001", _moved_bit),
    "slice-bit": ("e-shared-B8-M12591106", _slice_bit),
}


@pytest.mark.parametrize("what", list(REJECT))
def test_corrupt_tables_are_refused_and_leave_the_handle_untouched(rlm, saved, tmp_path, what):
    case, corrupt = REJECT[what]
    f = ckf.File.read(saved(case).path)
    path = str(tmp_path / "bad.rlm")
    with open(path, "wb") as g:
        g.write(f.rebuilt(corrupt(f, case)))
    m = _junk_handle(case)
    assert _code(m.load, path) == abi.RLM_ERR_INVALID_ARGUMENT, what
    _assert_junk(m, case)
    ref = _junk_handle(case)
    shared = SHAPES[case][3]
    ops = [("apply",), ("shared", 30)] if shared else [("run", 200)]
    _do(ref, ops)
    _do(m, ops)
    _assert_same(_observe(ref), _observe(m), what, shared=shared)
    m.close()
    ref.close()


# ---- the fingerprint of the day library ------------------------------------------------------------------------------
def _days(cfg, ticks, seed0=100):
    parts = [lib.flow_generate(cfg.flow, seed0 + d, 0, n) for d, n in enumerate(ticks)]
    buf = (abi.TickMsg * sum(ticks))()
    offs = [0]
    for p, n in zip(parts, ticks):
        C.memmove(C.addressof(buf) + offs[-1] * C.sizeof(abi.TickMsg), p, C.sizeof(p))
        offs.append(offs[-1] + n)
    return buf, offs


def _tape_handle(cfg, buf, offs):
    m = lib.BatchedMarket(abi.Config.from_buffer_copy(bytes(cfg)))
    m.load_days(buf, offs)
    m.assign_days([b % (len(offs) - 1) for b in range(cfg.n_envs)])
    m.reset()
    return m


def _grid_stride_ticks():
    import torch
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    limit = n_sms * 8 * 256  # words one pass of rlm_fingerprint_kernel's largest grid covers
    return max(40000, limit // 16 + 1001)


@pytest.mark.parametrize("ticks", ["2", "1001", "grid-stride"])
def test_library_fingerprint(rlm, tmp_path, ticks):
    """2 ticks = 32 words (less than a warp); 1001 ticks = 16016 words (not a multiple of 256); more words than one pass
    of the fingerprint kernel's grid"""
    n = _grid_stride_ticks() if ticks == "grid-stride" else int(ticks)
    cfg = _cfg(None, source=abi.SOURCE_TAPE, n_envs=4, mem=4096)
    day_ticks = [n] if n < 1000 else [n // 2, n - n // 2]
    buf, offs = _days(cfg, day_ticks)
    m = _tape_handle(cfg, buf, offs)
    path = str(tmp_path / "ck.rlm")
    m.save(path)
    m.close()
    words = np.frombuffer(bytes(buf), np.uint64)
    assert len(words) == 16 * n
    assert ckf.File.read(path).library_fp == ckf.fingerprint(words)


def test_swapped_days_are_refused(rlm, tmp_path):
    """two days of equal length in the other order, under the same offsets: the same words at other indices"""
    cfg = _cfg(None, source=abi.SOURCE_TAPE, n_envs=4, mem=4096)
    buf, offs = _days(cfg, [1500, 1500])
    half = 1500 * C.sizeof(abi.TickMsg)
    swapped = (abi.TickMsg * 3000).from_buffer_copy(bytes(buf)[half:] + bytes(buf)[:half])
    assert ckf.fingerprint(bytes(swapped)) != ckf.fingerprint(bytes(buf))
    m = _tape_handle(cfg, buf, offs)
    path = str(tmp_path / "ck.rlm")
    m.save(path)
    m.close()
    other = _tape_handle(cfg, swapped, offs)
    assert _code(other.load, path) == abi.RLM_ERR_INVALID_ARGUMENT
    other.close()
    same = _tape_handle(cfg, buf, offs)
    same.load(path)
    same.close()


# ---- resumes ---------------------------------------------------------------------------------------------------------
def test_resume_across_16_chunks(rlm, monkeypatch, tmp_path):
    """C1's table of 2^16 weights per env at 1024 envs: 64 tables per chunk, 16 chunks through both buffers"""
    import torch
    B, M = 1024, 1 << 16
    assert B * M // CHUNK == 16
    dense = B * M * 8
    if shutil.disk_usage(str(tmp_path)).free < 2 * dense:
        pytest.skip("needs %d MB free for the checkpoint file" % (2 * dense >> 20))
    if torch.cuda.mem_get_info()[0] < 4 * dense:
        pytest.skip("needs %d MB of free device memory" % (4 * dense >> 20))
    setup = Setup(_ck_cfg("q_learn", n_envs=B, mem=M))
    path = str(tmp_path / "ck.rlm")
    a = setup.make(monkeypatch, fresh=True)
    _do(a, [("run", 1500)])
    a.save(path)
    _do(a, [("run", 1000)])
    want = _observe(a)
    a.close()
    assert len(ckf.File.read(path).tables()) == B
    b = setup.make(monkeypatch)
    b.load(path)
    _do(b, [("run", 1000)])
    _assert_same(want, _observe(b), "16 chunks")
    b.close()
    assert want["counters"][1] > 0


def test_resume_saved_under_sub_batches(rlm, monkeypatch, tmp_path):
    """saved under RLM_SUBBATCHES=3 (70 envs: sub-batches of 32, 32 and 6 envs on their own streams), continued under
    the default engine"""
    setup = Setup(_ck_cfg("q_learn", n_envs=70), {"RLM_SUBBATCHES": "3", "RLM_ROUNDS": "0"})
    path = str(tmp_path / "ck.rlm")
    after = [("run", 137), ("run", 260), ("term", 1), ("reset",), ("run", 300)]
    a = setup.make(monkeypatch, fresh=True)
    _do(a, [("run", 300)])
    a.save(path)
    _do(a, after)
    want = _observe(a)
    a.close()
    b = setup.make(monkeypatch, env={})
    b.load(path)
    _do(b, after)
    _assert_same(want, _observe(b), "sub-batches")
    b.close()
