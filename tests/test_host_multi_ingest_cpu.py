"""CPU: the sharded layer ingest of libmkhost (mkhost_memfs_update_from_tars_multi) over several handles of the CPU mock
engine in one process.  Each scenario of tests/mock_engine/multi_ingest_cases.py compares 1, 2, 3 and 5 engines with
update_from_tars_cached on one engine.  Every scenario runs once more with libmkhost built with ThreadSanitizer: the
engines ingest from threads of their own while the calling thread only waits.  Each runs in a fresh process that loads
the mock (with mksnap_get_table, and its gunzip opens ordered by a lock: tests/mock_engine/mock_threads.cpp) with
RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_multi_ingest_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import functools
import os
import subprocess
import sys

import pytest

from tests import mock_engine
from tests.mock_engine import multi_ingest_cases as cases
from tests.test_host_multi_engine_cpu import _Engine, _tsan_host


@functools.cache
def _mock() -> str:
    """The mock of mock_threads.cpp, built once per process outside the tree."""
    d = mock_engine._out_dir()
    so = os.path.join(d, "libmock_threads.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wl,-Bsymbolic",
                           os.path.join(mock_engine.HERE, "mock_threads.cpp"), os.path.join(d, "mkoracle.o"), "-o", so])
    return so


def _run(scenario, tmp, env=None):
    os.makedirs(os.path.join(tmp, "run"))
    r = subprocess.run([sys.executable, "-m", "tests.test_host_multi_ingest_cpu", _mock(), scenario, os.path.join(tmp, "run")],
                       cwd=mock_engine.ROOT, capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    return r


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_ingest_mock(tmp_path, scenario):
    assert scenario + " ok" in _run(scenario, tmp_path).stdout


@pytest.mark.parametrize("scenario", cases.ALL)
def test_multi_ingest_under_tsan(tmp_path, scenario):
    tsan = subprocess.check_output(["gcc", "-print-file-name=libtsan.so"], text=True).strip()
    if not os.path.isabs(tsan):
        pytest.skip("no ThreadSanitizer runtime")
    env = dict(os.environ, LD_PRELOAD=tsan, TSAN_OPTIONS="report_signal_unsafe=0 exitcode=0")
    env[mock_engine.SANITIZED_HOST] = _tsan_host()
    r = _run(scenario, tmp_path, env)
    assert scenario + " ok" in r.stdout
    assert "WARNING: ThreadSanitizer" not in r.stderr, r.stderr[-8000:]


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
