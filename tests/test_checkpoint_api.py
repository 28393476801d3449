"""rlm_save / rlm_load without a GPU: the binding carries the header's types, the ABI version is unchanged, and a null
handle or path is refused before anything touches a device or the file system."""
import ctypes as C
import os

from rl_markets_b200 import abi, lib


def test_binding_and_abi_version():
    L = lib.load()
    for name in ("rlm_save", "rlm_load"):
        assert name in lib.EXPORTS and hasattr(L, name), name
        assert getattr(L, name).argtypes == [C.c_void_p, C.c_char_p], name
    assert L.rlm_abi_version() == 4
    assert hasattr(lib.BatchedMarket, "save") and hasattr(lib.BatchedMarket, "load")


def test_header_offsets_fit_the_config():
    # lib.BatchedMarket.load reads the model_log capacity (int64) and the saved rlm_config at these offsets
    assert abi.CKPT_MODEL_LOG_CAP_OFFSET + 8 == abi.CKPT_CONFIG_OFFSET
    assert abi.CKPT_CONFIG_OFFSET % C.alignment(abi.Config) == 0


def test_null_arguments_are_refused(tmp_path):
    L = lib.load()
    path = str(tmp_path / "ck.rlm").encode()
    for fn in (L.rlm_save, L.rlm_load):
        assert fn(None, path) == abi.RLM_ERR_INVALID_ARGUMENT
        assert fn.__name__ in L.rlm_last_error().decode()
        assert fn(None, None) == abi.RLM_ERR_INVALID_ARGUMENT
    assert not os.path.exists(path)
