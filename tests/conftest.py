import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: the library is built for sm_90a)")


def _cuda_device_count() -> int:
    try:
        import ctypes as C
        from duckpgq_extension_b200 import _native
        if _native.needs_build():
            return 0
        c = C.c_int(0)
        _native.load().pgq_device_count(C.byref(c))
        return c.value
    except Exception:
        return 0


def pytest_collection_modifyitems(config, items):
    """A bare `pytest` on a box without a CUDA device skips the gpu-marked tests instead of failing them
    (`-m gpu` / `-m "not gpu"` select as before)."""
    if _cuda_device_count() > 0:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible: gpu-marked tests need an H100")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


def golden_names():
    return sorted(f[4:-4] for f in os.listdir(GOLDEN) if f.startswith("ref_") and f.endswith(".npz"))


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, f"ref_{name}.npz"))
    g = {k: z[k] for k in z.files}
    for k in ("src", "dst", "psrc", "pdst", "csr_v", "csr_e", "length", "path_flat", "path_off"):
        g[k] = g[k].astype(np.int64)
    g["n"] = int(g["n"])
    g["has_paths"] = bool(int(g["has_paths"]))
    off = g["path_off"]
    g["paths"] = [g["path_flat"][off[i]:off[i + 1]].tolist() if g["path_valid"][i] else None
                  for i in range(len(g["psrc"]))] if g["has_paths"] else None
    return g


@pytest.fixture(scope="session")
def gpu_ctx():
    from duckpgq_extension_b200 import pgq
    return pgq.default_context(0)
