import os
import subprocess
import sys
import wave

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODEL_DIR = os.path.join(ROOT, "lyra_b200", "model_coeffs")
DATA_DIR = os.path.join(ROOT, "tests", "data")
GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")
EMU_DIR = os.path.join(ROOT, "tests", "cuda_emu")
EMU_SO = os.path.join(EMU_DIR, "_build", "liblyra_b200_emu.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def read_wav(name):
    with wave.open(os.path.join(DATA_DIR, name)) as w:
        assert w.getframerate() == 16000 and w.getnchannels() == 1 and w.getsampwidth() == 2
        return np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).copy()


def read_wav_any(name, rate):
    with wave.open(os.path.join(DATA_DIR, name)) as w:
        assert w.getframerate() == rate and w.getnchannels() == 1 and w.getsampwidth() == 2
        return np.frombuffer(w.readframes(w.getnframes()), dtype=np.int16).copy()


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle as O
    O.build()
    return O


@pytest.fixture(scope="session")
def sample1():
    return read_wav("sample1_16kHz.wav")


@pytest.fixture(scope="session")
def sample2():
    return read_wav("sample2_16kHz.wav")


def build_emu():
    """g++ -DLYRA_EMU build of the product kernels against tests/cuda_emu (test infrastructure only)."""
    csrc = os.path.join(ROOT, "lyra_b200", "csrc")
    srcs = [os.path.join(csrc, f) for f in os.listdir(csrc)] + [os.path.join(EMU_DIR, f) for f in ("cuda_emu.h", "cuda_emu.cc")]
    if os.path.exists(EMU_SO) and all(os.path.getmtime(s) <= os.path.getmtime(EMU_SO) for s in srcs):
        return EMU_SO
    os.makedirs(os.path.dirname(EMU_SO), exist_ok=True)
    subprocess.check_call(
        ["g++", "-std=c++17", "-O2", "-DLYRA_EMU", "-fPIC", "-shared", "-x", "c++", "-I" + EMU_DIR, "-I" + csrc,
         "-Wno-unknown-pragmas", os.path.join(csrc, "engine.cu"), os.path.join(csrc, "model_spec.cc"),
         os.path.join(csrc, "tflite_model.cc"), os.path.join(EMU_DIR, "cuda_emu.cc"), "-o", EMU_SO])
    return EMU_SO


@pytest.fixture(scope="session")
def emu_api():
    from lyra_b200 import _capi
    return _capi.CApi(build_emu())


@pytest.fixture(scope="session")
def gpu_api():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from lyra_b200 import _capi
    return _capi.load()
