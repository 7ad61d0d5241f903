"""Host cost of one CudaBackend kernel call (run on the CPU: python tests/backend_call_bench.py [--calls N]).

Times ``lloyd_chunk``, ``assign_chunk`` and ``glm_pass_chunk`` against a library whose entry points are Python
functions that return 0 at once, so what is timed is the Python side of a call: building the arguments, the size query,
the scratch lookup, the device context and the status check (not the ctypes conversion, which the library's prototypes
fix).  Prints one JSON line of microseconds per call.
"""
import argparse
import json
import os
import sys
import time

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dask_ml_b200 import _lib, engine  # noqa: E402


class _Stream(object):
    cuda_stream = 0x5EA0


class _NoDevice(object):
    def __init__(self, device):
        pass

    def __enter__(self):
        pass

    def __exit__(self, *exc):
        pass


class _NullLib(object):
    """Every entry point returns 0 at once; a size query reports 4096 bytes."""

    def __init__(self):
        for name in _lib.SIGNATURES:
            setattr(self, name, self._sizer if name.endswith("_bytes") else self._ok)

    @staticmethod
    def _ok(*args):
        return 0

    @staticmethod
    def _sizer(*args):
        args[-1]._obj.value = 4096
        return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100000)
    a = ap.parse_args()
    lib = _NullLib()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(torch.cuda, "is_available", lambda: True)
        mp.setattr(torch.cuda, "device", _NoDevice)
        mp.setattr(torch.cuda, "current_stream", lambda device=None: _Stream())
        mp.setattr(_lib, "load", lambda: lib)
        mp.setattr(_lib, "_lib", lib)
        mp.delenv("BKM_FLAGS", raising=False)
        be = engine.CudaBackend(device="cpu")
        n, d, k = 64, 16, 8
        x = torch.zeros((n, d), dtype=torch.float32)
        pack = torch.zeros(4096, dtype=torch.uint8)
        labels, min_d2 = torch.zeros(n, dtype=torch.int32), torch.zeros(n, dtype=torch.float32)
        sums, counts, inertia = torch.zeros(k * d, dtype=torch.float64), torch.zeros(k, dtype=torch.float64), \
            torch.zeros(1, dtype=torch.float64)
        y, beta, grad = torch.zeros(n, dtype=torch.float64), torch.zeros(d + 1, dtype=torch.float64), \
            torch.zeros(d + 2, dtype=torch.float64)
        cases = {
            "lloyd_chunk": lambda: be.lloyd_chunk(x, pack, k, labels, min_d2, sums, counts, inertia, first=True),
            "assign_chunk": lambda: be.assign_chunk(x, pack, k, labels, min_d2, True, inertia),
            "glm_pass_chunk": lambda: be.glm_pass_chunk(x, y, beta, 0, 0, grad=grad, first=True),
        }
        out = {}
        for name, fn in cases.items():
            for _ in range(1000):
                fn()
            best = None
            for _ in range(3):
                t0 = time.perf_counter()
                for _ in range(a.calls):
                    fn()
                dt = (time.perf_counter() - t0) / a.calls * 1e6
                best = dt if best is None else min(best, dt)
            out[name + "_us"] = round(best, 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
