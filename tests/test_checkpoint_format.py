"""The checkpoint format model (tests/checkpoint_format.py) on tables and files worked out by hand, without a GPU."""
import ctypes as C
import struct

import numpy as np
import pytest

import checkpoint_format as ckf
from rl_markets_b200 import abi

ONE = 0x3FF0000000000000  # 1.0
NEG_ZERO = 0x8000000000000000
QNAN = 0x7FF80000DEADBEEF  # a quiet NaN with a payload
SNAN = 0xFFF0000000000001  # a signalling NaN


def _w(*words):
    return np.array(words, dtype=np.uint64)


def _le(*words):
    return b"".join(struct.pack("<Q", w) for w in words)


def test_empty_tables():
    assert ckf.pack(_w()) == (b"", b"", 0)
    assert ckf.pack(np.zeros(16, np.uint64)) == (b"\0\0", b"", 0)
    assert ckf.pack(np.zeros(3, np.float64)) == (b"\0", b"", 0)


def test_one_word():
    assert ckf.pack(_w(0)) == (b"\x00", b"", 0)
    assert ckf.pack(_w(ONE)) == (b"\x01", b"\x00\x00\x00\x00\x00\x00\xf0\x3f", 1)
    assert ckf.pack(np.array([1.0])) == (b"\x01", b"\x00\x00\x00\x00\x00\x00\xf0\x3f", 1)


def test_nine_words_one_bit_in_the_second_byte():
    w = np.zeros(9, np.uint64)
    w[8] = 0x0123456789ABCDEF
    assert ckf.pack(w) == (b"\x00\x01", b"\xef\xcd\xab\x89\x67\x45\x23\x01", 1)
    w[0], w[3] = ONE, 5
    assert ckf.pack(w) == (b"\x09\x01", _le(ONE, 5, 0x0123456789ABCDEF), 3)


def test_negative_zero_and_nans_are_set():
    w = _w(0, NEG_ZERO, 0, QNAN, SNAN, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1)
    bits, vals, n = ckf.pack(w)
    assert bits == b"\x1a\x00\x01" and n == 4
    assert vals == _le(NEG_ZERO, QNAN, SNAN, 1)
    assert ckf.packed(w) == bits + vals
    assert ckf.unpack(bits + vals, len(w)).tobytes() == w.tobytes()


def test_unpack_rejects_what_load_must_reject():
    w = _w(0, ONE, 0, 0, 0, 0, 0, 0, 0)  # 9 words: 2 bitmap bytes, 7 padding bits
    sec = ckf.packed(w)
    assert sec[:2] == b"\x02\x00"
    with pytest.raises(ValueError):
        ckf.unpack(b"\x02\x80" + sec[2:], 9)  # a padding bit
    with pytest.raises(ValueError):
        ckf.unpack(b"\x03\x00" + sec[2:], 9)  # one more bit than values
    with pytest.raises(ValueError):
        ckf.unpack(sec[:-1], 9)  # not whole words
    assert ckf.unpack(sec, 9).tobytes() == w.tobytes()


def _mix_int(x):
    x = (x + 0x9E3779B97F4A7C15) & (2**64 - 1)
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & (2**64 - 1)
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & (2**64 - 1)
    return x ^ (x >> 31)


def test_fingerprint():
    assert ckf.fingerprint(_w()) == 0
    assert ckf.fingerprint(_w(0)) == 0xE220A8397B1DCDAF  # splitmix64's first output from state 0
    rng = np.random.default_rng(5)
    w = rng.integers(0, 2**64 - 1, size=300, dtype=np.uint64, endpoint=True)
    want = sum(_mix_int(int(x) ^ ((i * 0xD6E8FEB86659FD93) & (2**64 - 1))) for i, x in enumerate(w)) % 2**64
    assert ckf.fingerprint(w) == want
    # the index mixing tells two equal halves apart when they swap places
    swapped = np.concatenate([w[150:], w[:150]])
    assert ckf.fingerprint(swapped) != ckf.fingerprint(w)


def test_file_reader():
    assert ckf.LIBRARY_FP_OFFSET % 8 == 0
    cfg = abi.Config()
    cfg.n_envs, cfg.memory_size = 3, 9
    t0 = ckf.packed(_w(0, ONE, 0, 0, 0, 0, 0, 0, NEG_ZERO))
    n_sec = 2
    header_bytes = ckf.LIBRARY_FP_OFFSET + 8 + 16 + n_sec * ckf.SECTION.size
    raw = b"\x11" * 24
    head = bytearray(header_bytes - n_sec * ckf.SECTION.size)
    head[:8] = ckf.MAGIC
    struct.pack_into("<II", head, 8, 1, n_sec)
    struct.pack_into("<Q", head, 16, header_bytes + len(raw) + len(t0))
    struct.pack_into("<I", head, 24, header_bytes)
    struct.pack_into("<q", head, abi.CKPT_MODEL_LOG_CAP_OFFSET, 12)
    head[abi.CKPT_CONFIG_OFFSET:abi.CKPT_CONFIG_OFFSET + C.sizeof(cfg)] = bytes(cfg)
    struct.pack_into("<Q", head, ckf.LIBRARY_FP_OFFSET, 0xFEEDFACECAFEBEEF)
    secs = ckf.SECTION.pack(1, 0, header_bytes, len(raw), 0) + ckf.SECTION.pack(ckf.THETA, 0, header_bytes + len(raw), len(t0), 2)
    f = ckf.File(bytes(head) + secs + raw + t0)
    assert f.magic == ckf.MAGIC and f.version == 1 and f.n_sections == 2
    assert f.file_bytes == len(f.data) and f.header_bytes == header_bytes and f.model_log_cap == 12
    assert f.config.n_envs == 3 and f.config.memory_size == 9
    assert f.library_fp == 0xFEEDFACECAFEBEEF
    assert f.tables() == [(ckf.THETA, 0, header_bytes + len(raw), len(t0), 2)]
    assert f.body(f.sections[0]) == raw
    assert ckf.unpack(f.body(f.tables()[0]), 9).tolist() == [0, ONE, 0, 0, 0, 0, 0, 0, NEG_ZERO]


def test_rebuilt_file_moves_the_sections_after_a_changed_one():
    w = _w(ONE, 0, 2)
    head = bytearray(ckf.LIBRARY_FP_OFFSET + 8)
    head[:8] = ckf.MAGIC
    header_bytes = len(head) + 2 * ckf.SECTION.size
    struct.pack_into("<II", head, 8, 1, 2)
    struct.pack_into("<I", head, 24, header_bytes)
    t0, t1 = ckf.packed(w), ckf.packed(_w(0, 0, 0))
    secs = ckf.SECTION.pack(ckf.THETA, 0, header_bytes, len(t0), 2) + ckf.SECTION.pack(ckf.THETA, 1, header_bytes + len(t0), len(t1), 0)
    struct.pack_into("<Q", head, 16, header_bytes + len(t0) + len(t1))
    f = ckf.File(bytes(head) + secs + t0 + t1)
    g = ckf.File(f.rebuilt({0: (t0 + _le(7), 3)}))
    assert g.sections == [(ckf.THETA, 0, header_bytes, len(t0) + 8, 3), (ckf.THETA, 1, header_bytes + len(t0) + 8, len(t1), 0)]
    assert g.file_bytes == len(g.data) == len(f.data) + 8
    assert g.body(g.sections[1]) == t1
    assert ckf.File(f.rebuilt({})).data == f.data
