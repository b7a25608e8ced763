"""The C-ABI library loads and exports every symbol include/fastfp_b200.h declares (no compute
calls: this runs without a GPU)."""
import ctypes
import os
import re

from fastfp_b200 import _cabi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "fastfp_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(fastfp_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    lib = ctypes.CDLL(_cabi.lib_path())
    names = _declared()
    assert len(names) >= 15
    for name in names:
        assert hasattr(lib, name), f"{name} is declared in the header but missing from the library"


def test_binding_table_matches_header():
    assert sorted(_cabi.SYMBOLS) == _declared()


def test_library_answers_metadata_calls_without_a_gpu():
    lib = _cabi.load()
    assert lib.fastfp_version() >= 100
    assert lib.fastfp_device_count() >= 0
    assert lib.fastfp_kernel_launches() >= 0
    assert lib.fastfp_device_bytes() >= 0
    if lib.fastfp_device_count() == 0:  # with a device, packs of earlier tests may still be cached
        assert lib.fastfp_device_bytes() == 0
    assert lib.fastfp_pack_bytes(None) == 0 and lib.fastfp_pack_num_pulsars(None) == 0


def test_null_arguments_are_rejected_not_dereferenced():
    lib = _cabi.load()
    h = ctypes.c_void_p()
    rc = lib.fastfp_pack_create(0, 0, None, None, None, None, None, None, None, None, ctypes.byref(h))
    assert rc == -1 and b"null" in lib.fastfp_last_error()
    assert lib.fastfp_fp_sweep(None, None, 4, None, 0, None) == -1
    assert lib.fastfp_xcy(0, 0, 0, None, None, None, None, None, None, None) == -1
