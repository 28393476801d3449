"""Test-side oracle support for day markets: lobo_set_market / lobo_batch_set_market (tests/oracle_market.cpp, the
reference's LoadData market replacement restated on the oracle's own source), compiled once per session into a
temporary directory with the flags of oracle/Makefile.

The library holds a whole copy of the oracle; only its two market functions are called, on envs and batches that
oracle_lib's library created.  Both are built from the same lob_oracle.cpp with the same compiler and flags, so the
structs they share have one layout."""
import ctypes as C
import os
import subprocess
import tempfile

from rl_markets_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None
_dir = None


def lib():
    global _lib, _dir
    if _lib is None:
        _dir = tempfile.TemporaryDirectory()
        out = os.path.join(_dir.name, "liblob_oracle_market.so")
        subprocess.check_call(["g++", "-std=c++14", "-O3", "-DNDEBUG", "-ffp-contract=off", "-fPIC", "-shared", "-w",
                               "-I" + os.path.join(_ROOT, "include"), "-I" + os.path.join(_ROOT, "oracle"),
                               os.path.join(_HERE, "oracle_market.cpp"), "-o", out, "-lpthread"])
        L = C.CDLL(out)
        L.lobo_set_market.argtypes = [C.c_void_p, C.POINTER(abi.Market)]
        L.lobo_batch_set_market.argtypes = [C.c_void_p, C.c_int32, C.POINTER(abi.Market)]
        _lib = L
    return _lib


def set_market(h, market):
    """oracle env h (oracle_lib.lib().lobo_create) now runs under `market` (abi.Market)"""
    lib().lobo_set_market(h, C.byref(market))


def batch_set_market(b, env, market):
    lib().lobo_batch_set_market(b, env, C.byref(market))
