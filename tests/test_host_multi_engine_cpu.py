"""CPU: the multi-engine calls of libmkhost (mkhost_context_crc32_multi, mkhost_memfs_commit_layers_multi) over several
handles of the CPU mock engine in one process.  Each scenario of tests/mock_engine/multi_engine_cases.py compares 1, 2,
3 and 5 engines with the single-engine call.  Every scenario runs once more with libmkhost built with ThreadSanitizer:
the engines are driven from threads of their own, each with its own reader pool.  Each runs in a fresh process that
loads the mock (with mksnap_get_table, tests/mock_engine/mock_table.cpp) with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_multi_engine_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import functools
import os
import subprocess
import sys

import pytest

from tests import mock_engine
from tests.mock_engine import multi_engine_cases as cases


@functools.cache
def _mock() -> str:
    """The mock with mksnap_get_table, built once per process outside the tree."""
    d = mock_engine._out_dir()
    so = os.path.join(d, "libmock_table.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wl,-Bsymbolic",
                           os.path.join(mock_engine.HERE, "mock_table.cpp"), os.path.join(d, "mkoracle.o"), "-o", so])
    return so


@functools.cache
def _tsan_host() -> str:
    """libmkhost built as tests/run_host_tsan.sh builds it (ThreadSanitizer), once per process, outside the tree."""
    so = os.path.join(mock_engine._out_dir(), "libmkhost_tsan.so")
    lib = os.path.join(mock_engine.ROOT, "makisu_b200", "lib")
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-shared", "-pthread", "-fsanitize=thread",
                           "-fno-omit-frame-pointer", "-I", os.path.join(mock_engine.ROOT, "include"), "-o", so,
                           os.path.join(mock_engine.ROOT, "makisu_b200", "host", "mkhost.cpp"), "-L", lib, "-lmksnap",
                           "-Wl,-rpath," + lib, "-ldl"])
    return so


def _run(scenario, tmp, env=None):
    r = subprocess.run([sys.executable, "-m", "tests.test_host_multi_engine_cpu", _mock(), scenario, str(tmp)],
                       cwd=mock_engine.ROOT, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    return r


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_engine_mock(tmp_path, scenario):
    assert scenario + " ok" in _run(scenario, tmp_path).stdout


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_engine_under_tsan(tmp_path, scenario):
    tsan = subprocess.check_output(["gcc", "-print-file-name=libtsan.so"], text=True).strip()
    if not os.path.isabs(tsan):
        pytest.skip("no ThreadSanitizer runtime")
    env = dict(os.environ, LD_PRELOAD=tsan, TSAN_OPTIONS="report_signal_unsafe=0 exitcode=0")
    env[mock_engine.SANITIZED_HOST] = _tsan_host()
    r = _run(scenario, tmp_path, env)
    assert scenario + " ok" in r.stdout
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-8000:]


# ---------------------------------------------------------------------------------------------------------------
class _Engine:
    def __init__(self, mock, arena, max_extents=1 << 12, max_chunks=0, cdc=None):
        from makisu_b200 import abi
        self.mock = mock
        cfg = abi.Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.device_arena_bytes = 2, arena, arena
        cfg.max_extents, cfg.max_chunks = max_extents, max_chunks
        if cdc is not None:
            cfg.cdc = cdc
        self.h = C.c_void_p()
        mock.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        assert mock.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0
        mock.mock_submits.restype = C.c_uint64
        mock.mock_submits.argtypes = [C.c_void_p]

    def work(self):
        return int(self.mock.mock_submits(self.h))

    def __del__(self):
        self.mock.mksnap_destroy(self.h)


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=True)
    seen = C.CDLL(None)
    assert C.cast(mock.mksnap_get_table, C.c_void_p).value == C.cast(seen.mksnap_get_table, C.c_void_p).value, \
        "libmkhost is not bound to the mock engine (mksnap_get_table)"
    mock.mksnap_destroy.argtypes = [C.c_void_p]

    def make(arena, **kw):
        return _Engine(mock, arena, **kw)
    getattr(cases, scenario)(make, tmp)


if __name__ == "__main__":
    main()
