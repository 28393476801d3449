"""A NumPy statement of the checkpoint file that rlm_save writes (include/rlm.h, rl_markets_b200/csrc/rlm_checkpoint.cu),
written from the documented format and not from the kernels, so the tests can hold the packed bytes to it.

  header     magic "RLMCKPT\\0", version (u32 at 8), n_sections (u32 at 12), file_bytes (u64 at 16), header_bytes (u32 at 24),
             model_log_cap (i64 at 40), the saved rlm_config (at 48), then alpha, eps, tau, launches and six int32 fields,
             then library_fp (u64)
  sections   n_sections entries of <IIQQQ (id, table, offset, bytes, count) ending at header_bytes; the sections follow in
             table order, back to back, and the last one ends at file_bytes
  a table    of M 64-bit words: a bitmap with bit i set when word i is not +0.0 bitwise, (M + 7) / 8 little-endian bytes
             (bit i in byte i / 8, bit i % 8), then the words that are set, in index order; count = their number
  library_fp the sum modulo 2^64 of mix(w[i] ^ i * 0xD6E8FEB86659FD93) over the day library's words (mix: the splitmix64
             finaliser)
"""
import ctypes as C
import struct

import numpy as np

from rl_markets_b200 import abi

MAGIC = b"RLMCKPT\0"
SECTION = struct.Struct("<IIQQQ")
THETA, THETA_B, DTHETA = 64, 65, 66
# after the config: three doubles (alpha, eps, tau), int64 launches and six int32 (run_seq .. has_env_market)
LIBRARY_FP_OFFSET = abi.CKPT_CONFIG_OFFSET + C.sizeof(abi.Config) + 3 * 8 + 8 + 6 * 4


def words_of(a):
    """the 64-bit words of a table: a uint64 / float64 array, or anything with the buffer protocol"""
    if isinstance(a, np.ndarray):
        return np.ascontiguousarray(a).view(np.uint64).reshape(-1)
    return np.frombuffer(bytes(a), np.uint64)


def pack(words):
    """-> (bitmap bytes, value bytes, count) of one table"""
    w = words_of(words)
    nz = w != 0
    return np.packbits(nz, bitorder="little").tobytes(), w[nz].tobytes(), int(nz.sum())


def packed(words):
    """the section bytes of one table: bitmap, then values"""
    bits, vals, _n = pack(words)
    return bits + vals


def unpack(section, m):
    """the M words of a packed table section; ValueError on set padding bits or a count that does not match the bitmap"""
    nb = (m + 7) // 8
    if len(section) < nb or (len(section) - nb) % 8:
        raise ValueError("a packed table of %d words cannot be %d bytes" % (m, len(section)))
    bits = np.unpackbits(np.frombuffer(section[:nb], np.uint8), bitorder="little")
    if bits[m:].any():
        raise ValueError("padding bits set")
    nz = bits[:m].astype(bool)
    vals = np.frombuffer(section[nb:], np.uint64)
    if len(vals) != int(nz.sum()):
        raise ValueError("bitmap population %d, %d values" % (int(nz.sum()), len(vals)))
    out = np.zeros(m, np.uint64)
    out[nz] = vals
    return out


_U = np.uint64


def _mix(x):
    x = x + _U(0x9E3779B97F4A7C15)
    x = (x ^ (x >> _U(30))) * _U(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> _U(27))) * _U(0x94D049BB133111EB)
    return x ^ (x >> _U(31))


def fingerprint(words):
    """library_fp of a day library's bytes (uint64 words)"""
    w = words_of(words)
    i = np.arange(len(w), dtype=np.uint64)
    return int(np.sum(_mix(w ^ (i * _U(0xD6E8FEB86659FD93))), dtype=np.uint64))


class File:
    """the header fields and the section table of a checkpoint file's bytes"""

    def __init__(self, data):
        self.data = bytes(data)
        d = self.data
        self.magic = d[:8]
        self.version, self.n_sections = struct.unpack_from("<II", d, 8)
        self.file_bytes = struct.unpack_from("<Q", d, 16)[0]
        self.header_bytes = struct.unpack_from("<I", d, 24)[0]
        self.model_log_cap = struct.unpack_from("<q", d, abi.CKPT_MODEL_LOG_CAP_OFFSET)[0]
        self.config = abi.Config.from_buffer_copy(d, abi.CKPT_CONFIG_OFFSET)
        self.library_fp = struct.unpack_from("<Q", d, LIBRARY_FP_OFFSET)[0]
        first = self.header_bytes - self.n_sections * SECTION.size
        self.sections = [SECTION.unpack_from(d, first + k * SECTION.size) for k in range(self.n_sections)]

    @classmethod
    def read(cls, path):
        with open(path, "rb") as f:
            return cls(f.read())

    def body(self, section):
        """the bytes of one section table entry's section"""
        _id, _table, off, n, _count = section
        return self.data[off:off + n]

    def tables(self):
        """the packed weight-table sections, in file order"""
        return [s for s in self.sections if s[0] >= THETA]

    def rebuilt(self, bodies):
        """this file's bytes with some sections replaced ({section index: (bytes, count)}), and the offsets, the section
        table and file_bytes recomputed to fit them"""
        secs, parts, pos = [], [], self.header_bytes
        for k, sec in enumerate(self.sections):
            body, count = bodies.get(k, (self.body(sec), sec[4]))
            secs.append((sec[0], sec[1], pos, len(body), count))
            parts.append(body)
            pos += len(body)
        head = bytearray(self.data[:self.header_bytes - self.n_sections * SECTION.size])
        struct.pack_into("<Q", head, 16, pos)
        return bytes(head) + b"".join(SECTION.pack(*s) for s in secs) + b"".join(parts)
