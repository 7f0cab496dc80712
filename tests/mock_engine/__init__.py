"""The CPU mock of libmksnap (mock_mksnap.cpp) from Python: build it, run a scenario in a fresh process bound to it,
and, in that process, load it ahead of libmkhost.

A scenario runs in its own process because libmkhost's mksnap_* references must bind to the mock: the mock is loaded
with RTLD_GLOBAL before anything loads libmksnap or libmkhost, which a process that ran other tests cannot promise."""
import atexit
import ctypes as C
import functools
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
# every entry point the mock implements: after host.load() libmkhost must see the mock's
ENTRY_POINTS = ("mksnap_begin", "mksnap_arena_submit", "mksnap_finish", "mksnap_get_stream_digests",
                "mksnap_arena_submit_spans", "mksnap_chunks_add", "mksnap_get_chunks", "mksnap_crc_fold",
                "mksnap_get_crc_streams", "mksnap_reserve_stream_log", "mksnap_gunzip_open",
                "mksnap_gunzip_open_indexed", "mksnap_gunzip_read", "mksnap_gunzip_get_index")


@functools.cache
def _out_dir() -> str:
    d = tempfile.mkdtemp(prefix="mock_mksnap_")
    atexit.register(shutil.rmtree, d, True)
    obj = os.path.join(d, "mkoracle.o")
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-c", os.path.join(ROOT, "oracle", "mkoracle.c"), "-o", obj])
    return d


def build(sanitize: bool = False) -> str:
    """Path of the mock library, built once per process (with ASan/UBSan when `sanitize`), outside the tree."""
    return _build(bool(sanitize))


@functools.cache
def _build(sanitize: bool) -> str:
    d = _out_dir()
    so = os.path.join(d, "libmock_mksnap%s.so" % ("_asan" if sanitize else ""))
    flags = (["-O1", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer"]
             if sanitize else ["-O2"])
    # -Bsymbolic: the mock's own calls bind inside it even when libmksnap or the oracle is loaded globally
    subprocess.check_call(["g++", *flags, "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wl,-Bsymbolic",
                           os.path.join(HERE, "mock_mksnap.cpp"), os.path.join(d, "mkoracle.o"), "-o", so])
    return so


def run(module: str, scenario: str, tmp, sanitize: bool = False) -> subprocess.CompletedProcess:
    """python -m <module> <mock.so> <scenario> <tmp> in a fresh process; it must exit 0 with no sanitizer report."""
    env = dict(os.environ)
    if sanitize:
        env["LD_PRELOAD"] = " ".join(subprocess.check_output(["gcc", "-print-file-name=" + l], text=True).strip()
                                     for l in ("libasan.so", "libubsan.so"))
        env["ASAN_OPTIONS"] = "detect_leaks=0"
    r = subprocess.run([sys.executable, "-m", module, build(sanitize), scenario, str(tmp)], cwd=ROOT,
                       capture_output=True, text=True, env=env)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-6000:]
    assert "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-6000:]
    return r


def load_for_child(path: str, host: bool = False) -> C.CDLL:
    """In the scenario's process: load the mock with RTLD_GLOBAL, and with `host` load libmkhost after it and check
    that libmkhost's mksnap_* references bind to the mock."""
    mock = C.CDLL(path, mode=C.RTLD_GLOBAL)  # BEFORE anything loads libmksnap / libmkhost
    if host:
        from makisu_b200 import host as mkhost
        mkhost.load()
        seen = C.CDLL(None)
        for name in ENTRY_POINTS:
            assert C.cast(getattr(mock, name), C.c_void_p).value == C.cast(getattr(seen, name), C.c_void_p).value, \
                "libmkhost is not bound to the mock engine (%s)" % name
    return mock
