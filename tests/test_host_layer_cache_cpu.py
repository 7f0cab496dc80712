"""CPU: the incremental layer ingest (mkhost_memfs_update_from_tars_cached, mkhost_layer_cache) under the CPU mock engine
(tests/mock_engine/mock_mksnap.cpp).  Each scenario of tests/layer_cache_cases.py compares the cached run with
update_from_tars_indexed on a fresh tree: cold and warm runs, a mixed run, misses (touch, same-size rewrite, wrong key),
what an entry holds, other CDC parameters, MKHOST_UNTAR (as root), a pipe, save / load and damaged files, no cache, and
a damaged layer in the middle of a run.  Every scenario runs once more with libmkhost and the mock built with
AddressSanitizer and UndefinedBehaviorSanitizer.  Each runs in a fresh process that loads the mock with RTLD_GLOBAL
before libmkhost:
    python -m tests.test_host_layer_cache_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import os
import sys

import pytest

from tests import layer_cache_cases as cases
from tests import mock_engine


@pytest.mark.parametrize("scenario", cases.ALL + ["untar"])
def test_layer_cache_mock(tmp_path, scenario):
    if scenario == "untar" and os.geteuid() != 0:
        pytest.skip("MKHOST_UNTAR applies owners (chown)")
    r = mock_engine.run("tests.test_host_layer_cache_cpu", scenario, tmp_path)
    assert scenario + " ok" in r.stdout


def test_layer_cache_under_asan_ubsan(tmp_path, monkeypatch):
    monkeypatch.setenv(mock_engine.SANITIZED_HOST, mock_engine.sanitized_host())
    r = mock_engine.run("tests.test_host_layer_cache_cpu", "every", tmp_path, sanitize=True)
    assert "every ok" in r.stdout


# ---------------------------------------------------------------------------------------------------------------
class _Engine:
    def __init__(self, mock, arena, cdc=None, max_chunks=0, max_extents=1 << 12):
        from makisu_b200 import abi
        cfg = abi.Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.device_arena_bytes = 2, arena, arena
        cfg.max_extents, cfg.max_chunks = max_extents, max_chunks
        if cdc is not None:
            cfg.cdc = cdc
        self.h = C.c_void_p()
        mock.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        assert mock.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0


def every(make, tmp):
    for name in cases.ALL + (["untar"] if os.geteuid() == 0 else []):
        d = os.path.join(tmp, name)
        os.mkdir(d)
        getattr(cases, name)(make, d)
    print("every ok")


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=True)

    def make(arena, **kw):
        return _Engine(mock, arena, **kw)
    (every if scenario == "every" else getattr(cases, scenario))(make, tmp)


if __name__ == "__main__":
    main()
