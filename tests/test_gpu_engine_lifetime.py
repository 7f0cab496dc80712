"""GPU: an engine gives back its device memory when it is destroyed, and when its create fails part-way.

A full-size engine (at least 16 GiB of device memory) is created and destroyed 8 times in a row.  Then 8 times a create
that allocates the same arenas and fails with E_NOMEM on a chunk table no H100 can hold alternates with the full-size
create.  Every full-size create must succeed: memory that a destroy or a failed create kept would make one of them fail.

The loop runs in a fresh process (python -m tests.test_gpu_engine_lifetime): a failed cudaMalloc leaves its error as
the thread's last CUDA error, and a later test's first kernel launch in the same process would report it."""
import ctypes
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FULL = dict(device=0, device_arena_bytes=4 << 30, n_device_slots=4, max_extents=1 << 16)  # 4 slots of 4 GiB
TOO_MANY_CHUNKS = 1 << 40   # 8 TiB of chunk starts alone: allocated after the arenas, fails on every H100
ROUNDS = 8
E_NOMEM = -3
SKIP_EXIT = 77


def _device_free_bytes(cu):
    free, total = ctypes.c_size_t(), ctypes.c_size_t()
    rc = cu.cuMemGetInfo_v2(ctypes.byref(free), ctypes.byref(total))
    assert rc == 0, f"cuMemGetInfo_v2: {rc}"
    return free.value


def _child():
    from makisu_b200.abi import Engine, MksnapError
    cu = ctypes.CDLL("libcuda.so.1")
    ctx = ctypes.c_void_p()
    # the primary context, which the engine's runtime calls use too: free memory can be read before the first create
    assert cu.cuInit(0) == 0 and cu.cuDevicePrimaryCtxRetain(ctypes.byref(ctx), 0) == 0 and cu.cuCtxSetCurrent(ctx) == 0
    free0 = _device_free_bytes(cu)
    try:
        e = Engine(**FULL)
    except MksnapError as x:
        if x.code != E_NOMEM:
            raise
        print(f"the full-size engine does not fit: {free0 / 2**30:.1f} GiB free ({x})")
        sys.exit(SKIP_EXIT)
    used = free0 - _device_free_bytes(cu)
    e.close()
    print(f"full-size engine: {used / 2**30:.2f} GiB of device memory")
    assert used >= 16 << 30, used
    for _ in range(ROUNDS - 1):
        Engine(**FULL).close()
    for _ in range(ROUNDS):
        with pytest.raises(MksnapError, match="E_NOMEM"):
            Engine(**FULL, max_chunks=TOO_MANY_CHUNKS)
        Engine(**FULL).close()
    print(f"free device memory before the first create {free0 / 2**30:.2f} GiB, after the last destroy "
          f"{_device_free_bytes(cu) / 2**30:.2f} GiB")


def test_create_destroy_and_failed_create_give_memory_back():
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_engine_lifetime"], cwd=ROOT, capture_output=True, text=True)
    print(r.stdout)
    if r.returncode == SKIP_EXIT:
        pytest.skip(r.stdout.strip())
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]


if __name__ == "__main__":
    _child()
