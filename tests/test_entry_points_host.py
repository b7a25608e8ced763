"""Entry points that must fail or resolve before any device work: null arguments of the pack constructors, a NULL
pack handed to every call that takes one, and the device / path resolution of the front ends (CPU)."""
import ctypes
import os
import re

import pytest

import fastfp_b200
from fastfp_b200 import _cabi, synth
from fastfp_b200.nmfp import NMFP, RN_container

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_DEVICE = 1 << 20  # an ordinal no machine has: selecting it would fail with FASTFP_ERR_CUDA (-2)


def _null_args(name, **fixed):
    """Arguments for ``name``: None for every pointer, 1 for every integer (sizes), ``fixed`` by position."""
    args = [None if a not in (ctypes.c_int, ctypes.c_int64) else 1 for a in _cabi.SYMBOLS[name][1]]
    for i, v in fixed.items():
        args[int(i[1:])] = v
    return args


@pytest.mark.parametrize("name", ["fastfp_pack_create", "fastfp_nmfp_pack_create", "fastfp_pack_create_blockn"])
@pytest.mark.parametrize("P", [0, 1])
def test_pack_constructors_reject_null_arguments_before_selecting_a_device(name, P):
    lib = _cabi.load()
    h = ctypes.c_void_p(1)
    nargs = len(_cabi.SYMBOLS[name][1])
    args = _null_args(name, a0=NO_DEVICE, a1=P)
    args[nargs - 1] = ctypes.byref(h)
    assert getattr(lib, name)(*args) == -1
    assert lib.fastfp_last_error().decode() == f"{name}: null argument or P < 1"


def _pack_calls():
    """Every function of the header whose first parameter is a pack."""
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "fastfp_b200.h")).read(), flags=re.S)
    return sorted(set(re.findall(r"\b(fastfp_[a-z0-9_]+)\s*\(\s*(?:const\s+)?fastfp_pack_t\s*\*", text)))


SIZE_GETTERS = {"fastfp_pack_bytes", "fastfp_pack_num_pulsars", "fastfp_pack_mvar_total"}


def test_every_call_on_a_null_pack_is_rejected():
    lib = _cabi.load()
    names = _pack_calls()
    assert len(names) >= 17 and SIZE_GETTERS <= set(names) and "fastfp_fp_sweep" in names
    for name in names:
        rc = getattr(lib, name)(*_null_args(name))
        if name == "fastfp_pack_destroy":
            assert rc is None
        elif name in SIZE_GETTERS:
            assert rc == 0, name
        else:
            assert rc == -1, name


def _psrs(P=2):
    return synth.make_pta(P, 24, n_tm=3, ncomps=2).psrs


def _front_ends():
    psrs = _psrs()
    return [
        lambda **kw: fastfp_b200.FastFp(psrs, **kw),
        lambda **kw: fastfp_b200.FastFe(psrs, **kw),
        lambda **kw: NMFP(psrs, [RN_container(q, ncomps=2) for q in psrs], **kw),
    ]


@pytest.mark.parametrize("which", [0, 1, 2], ids=["FastFp", "FastFe", "NMFP"])
def test_front_ends_resolve_device_and_path_alike(which, monkeypatch):
    make = _front_ends()[which]
    monkeypatch.delenv("LOCAL_RANK", raising=False)
    monkeypatch.delenv("FASTFP_B200_PATH", raising=False)
    obj = make()
    assert (obj.device, obj.path) == (0, "auto")
    monkeypatch.setenv("LOCAL_RANK", "5")
    monkeypatch.setenv("FASTFP_B200_PATH", "prefer-i8")
    obj = make()  # no device is touched: ordinal 5 need not exist
    assert (obj.device, obj.path) == (5, "prefer-i8")
    obj = make(device=3, path="fp64")  # arguments win over the environment
    assert (obj.device, obj.path) == (3, "fp64")
    assert isinstance(obj.device, int) and make(device="2").device == 2
    with pytest.raises(ValueError, match="path must be"):
        make(path="tensor")
    monkeypatch.setenv("FASTFP_B200_PATH", "bogus")
    with pytest.raises(ValueError, match="path must be"):
        make()
    assert make(path="i8").path == "i8"
