"""CPU: the batched incremental layer commit (mkhost_memfs_commit_layers_cached) under the CPU mock engine
(tests/mock_engine/mock_mksnap.cpp).  Each scenario of tests/commit_layers_cases.py compares a batch with one
commit_copy_ops_cached call per layer on a fresh tree: cold, warm and edited caches, MKHOST_NO_TAR_DIGEST with and
without a tar, MKHOST_FILE_DIGESTS with and without a cache, one-entry arena shares, other CDC parameters, too few
stream slots, and a content-aware scan after a batch.  Every scenario runs once more with libmkhost and the mock built
with AddressSanitizer and UndefinedBehaviorSanitizer.  Each runs in a fresh process that loads the mock with
RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_commit_layers_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import os
import sys

import pytest

from tests import commit_layers_cases as cases
from tests import mock_engine


@pytest.mark.parametrize("scenario", cases.ALL)
def test_commit_layers_mock(tmp_path, scenario):
    r = mock_engine.run("tests.test_host_commit_layers_cpu", scenario, tmp_path)
    assert scenario + " ok" in r.stdout


def test_commit_layers_under_asan_ubsan(tmp_path, monkeypatch):
    monkeypatch.setenv(mock_engine.SANITIZED_HOST, mock_engine.sanitized_host())
    r = mock_engine.run("tests.test_host_commit_layers_cpu", "every", tmp_path, sanitize=True)
    assert "every ok" in r.stdout


# ---------------------------------------------------------------------------------------------------------------
class _Engine:
    def __init__(self, mock, arena, cdc=None, max_extents=1 << 12):
        from makisu_b200 import abi
        self.mock = mock
        cfg = abi.Config()
        cfg.n_host_arenas, cfg.host_arena_bytes, cfg.device_arena_bytes = 2, arena, arena
        cfg.max_extents = max_extents
        if cdc is not None:
            cfg.cdc = cdc
        self.h = C.c_void_p()
        mock.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        assert mock.mksnap_create(C.byref(cfg), C.byref(self.h)) == 0
        mock.mock_submits.restype = C.c_uint64
        mock.mock_submits.argtypes = [C.c_void_p]
        mock.mock_chunk_log.restype = C.c_size_t
        mock.mock_chunk_log.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]

    def work(self):
        return int(self.mock.mock_submits(self.h))

    def mark(self):
        pass

    def uploaded(self):
        """Arena bytes of the last session's submits: the spans of a sparse submit, else everything used."""
        n = self.mock.mock_chunk_log(self.h, None, 0)
        buf = C.create_string_buffer(n)
        self.mock.mock_chunk_log(self.h, buf, n)
        total = 0
        for line in buf.value.decode().split("\n"):
            if not line.startswith("submit"):
                continue
            head, _, spans = line.partition(" spans")
            if " spans" in line:
                total += sum(int(s.split("+")[1]) for s in spans.split())
            else:
                total += int(dict(x.split("=") for x in head.split()[1:])["used"])
        return total


def every(make, tmp):
    for name in cases.ALL:
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
