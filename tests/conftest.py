import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EPS = 2.220446049250313e-16


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100; run with -m gpu)")


@pytest.fixture(params=["auto", "fp64"])
def sweep_path(request, monkeypatch):
    """Run a plain-Fp GPU test on both sweep kernels: "auto" = the INT8 tensor-core kernel wherever the pack can take
    it (else the fp64 DMMA kernel; the library's AUTO is the DMMA kernel, so this parameter asks for "prefer-i8"),
    "fp64" = the DMMA kernel always. FastFp reads FASTFP_B200_PATH at construction."""
    path = request.param
    monkeypatch.setenv("FASTFP_B200_PATH", "prefer-i8" if path == "auto" else path)
    return path


class Psr:
    """Duck-typed pulsar: all the hot path reads (reference fastfp/fastfp.py:44-45)."""

    def __init__(self, toas, residuals, name="J0000+0000", Mmat=None, backend_flags=None):
        self.toas, self.residuals, self.name = toas, residuals, name
        self.Mmat = Mmat
        self.backend_flags = backend_flags


class Golden:
    """A committed fixture of tests/golden/ (inputs + outputs of the reference source)."""

    def __init__(self, name):
        self.g = np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"))
        self.P = int(self.g["P"])

    def lst(self, key):
        return [self.g[f"{key}_{p}"] for p in range(self.P)]

    def __getitem__(self, k):
        return self.g[k]

    @property
    def psrs(self):
        return [
            Psr(t, r, name=str(self.g[f"name_{p}"]), Mmat=np.zeros((len(t), int(self.g[f"ntm_{p}"]))))
            for p, (t, r) in enumerate(zip(self.lst("toas"), self.lst("res")))
        ]


@pytest.fixture(scope="session")
def golden():
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Golden(name)
        return cache[name]

    return get


def term_tolerance(tt, cond, ora, k_oracle=4.0, rel=1e-10):
    """Per-(pulsar, frequency) absolute tolerance for the terms 0.5 N^T M^-1 N.

    ``rel`` is the north-star tolerance (1e-10 relative). Near a red-noise Fourier frequency the
    reference formula is a difference of numbers up to ~1e9 times larger than the result and its
    own float64 output is only defined to eps*kappa (SURVEY.md section 7.3 H1); the allowance is
    therefore ``rel*|truth| + k_oracle * E_p * eps * cond`` with ``cond`` the first-order
    conditioning figure of oracle/truth.py and ``E_p >= 1`` the oracle's own worst normalised
    distance from the longdouble truth for that pulsar -- i.e. "within 1e-10, or within
    k_oracle times the reference formula's own error at that conditioning"."""
    tt, cond, ora = np.asarray(tt, float), np.asarray(cond, float), np.asarray(ora, float)
    E = np.maximum(1.0, (np.abs(ora - tt) / (EPS * cond)).max(axis=1, keepdims=True))
    return rel * np.abs(tt) + k_oracle * E * EPS * cond
