"""CPU tier: the product library builds, loads, exports exactly the symbols include/lyra_b200.h declares,
and refuses to run without a GPU (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import pytest

from conftest import ROOT
from lyra_b200 import _capi


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "lyra_b200.h")).read()
    return sorted(set(re.findall(r"\b(lyra_b200_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    assert declared_symbols() == sorted(_capi.CApi.EXPORTS)


def test_product_library_exports_declared_abi():
    import __graft_entry__ as g
    so = g.build_product()
    lib = ctypes.CDLL(so)
    for name in declared_symbols():
        assert hasattr(lib, name), name
    out = subprocess.check_output(["nm", "-D", "--defined-only", so]).decode()
    exported = sorted(set(re.findall(r"\bT (lyra_b200_[a-z0-9_]+)\b", out)))
    assert exported == declared_symbols()


def test_product_library_is_sm90a_only():
    import __graft_entry__ as g
    out = subprocess.check_output([os.path.join(os.path.dirname(g.NVCC), "cuobjdump"), "-lelf", g.build_product()]).decode()
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_create_without_gpu_fails_loudly():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    api = _capi.load()
    with pytest.raises(_capi.LyraB200Error) as e:
        _capi.Context(4, capi=api)
    assert e.value.code == _capi.ENODEV


def test_product_never_touches_the_oracle():
    """No file under lyra_b200/ or include/ may include, import, link or load anything of oracle/ or the emulator
    (comments citing the oracle for the arithmetic contract are fine)."""
    bad = []
    for base in ("lyra_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".py", ".cc", ".cu", ".cuh", ".h")):
                    text = open(os.path.join(dirpath, f), errors="ignore").read()
                    if re.search(r"#include[^\n]*(oracle|cuda_emu\.cc)|liblyra_oracle|oracle/_build|import oracle|from oracle|liblyra_b200_emu", text):
                        bad.append(os.path.join(dirpath, f))
    assert not bad, bad
