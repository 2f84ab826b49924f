"""The C-ABI library builds for sm_90a without a GPU, loads, and exports every symbol include/evok.h declares."""

import ctypes
import os
import re

import pytest

from evotorch_b200 import _native as nat
from evotorch_b200 import build as evok_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libpath():
    return evok_build.build()


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "evok.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(evok_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert declared_symbols() == sorted(nat.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol(libpath):
    handle = ctypes.CDLL(libpath)
    for name in declared_symbols():
        assert hasattr(handle, name), name
    lib = nat.lib()
    assert lib.evok_abi_version() == 1
    assert lib.evok_error_string(0) == b"ok" and b"workspace" in lib.evok_error_string(-4)


def test_host_side_argument_checks_need_no_gpu(libpath):
    lib = nat.lib()
    assert lib.evok_rank_workspace_bytes(1_000_000) >= 16_000_000
    assert lib.evok_grad_workspace_bytes(1000, 10_000) > 0
    assert lib.evok_sample_eval(2, None, 0, None, None, 0, 4, 4, 1, 0, 0, None, None, None) == -1  # null pointers
    assert lib.evok_rank(9, 1, 4, 0, 1, None, 1, 0, None) == -3  # bad enum (pointers are never dereferenced on the host)
    assert lib.evok_clipup_step(None, 4, None, 0.1, 0.9, 0.2, None, None, None) == -1


def test_shared_forward_eligibility_needs_no_gpu(libpath):
    """evok_mlp_forward_shared_supported: the nets the shared-minibatch forward takes.  Its second kernel stages two [width][33]
    activation tiles and the largest later layer in at most 200 KB of shared memory; the pairs below sit on either side of that."""
    from evotorch_b200 import ops

    def ok(*dims):
        return bool(nat.lib().evok_mlp_forward_shared_supported(len(dims) - 1, (ctypes.c_int32 * len(dims))(*dims)))

    assert ok(376, 256, 17) and ok(6, 16, 3) and ok(33, 40, 24, 5) and ok(8, 512, 2) and ok(2048, 508, 32)
    assert ok(8, 512, 33) and not ok(8, 512, 34)  # 202 884 B / 204 936 B
    assert ok(8, 195, 195, 2) and not ok(8, 196, 196, 2)  # 204 360 B / 206 192 B
    assert not ok(8, 256, 256, 2) and not ok(8, 512, 40) and not ok(8, 200, 200, 2)
    assert not ok(8, 513, 2) and not ok(2049, 16, 2) and not ok(8, 0, 2)  # widths
    assert not ok(8, 16) and ok(*([8] * 9)) and not ok(*([8] * 10))  # 2 .. 8 layers
    assert not nat.lib().evok_mlp_forward_shared_supported(2, None)
    assert ops.mlp_forward_shared_supported([8, 512, 33]) and not ops.mlp_forward_shared_supported([8, 512, 34])


def test_kernels_are_sm90a_sass(libpath):
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", libpath], capture_output=True, text=True).stdout
    assert "sm_90a" in out
