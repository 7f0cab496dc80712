"""CPU: gunzip (mksnap_gunzip_*) and update_from_tar(MKHOST_GUNZIP) under the CPU mock of the engine.

The mock (tests/mock_engine/mock_mksnap.cpp) runs the engine's own candidate rule, decoder, link and resolve code
(makisu_b200/csrc/mksnap_inflate_core.h) step for step as the device does, so these tests check the code that runs on
the GPU against Go's gzip reader (tests/gzip_corpus.py):
  - the generated corpus, bit-exact, with Go's acceptance where Python's gzip differs;
  - a few thousand truncated or bit-flipped blobs through a mock built with ASan/UBSan: zlib's output or MKSNAP_E_DATA;
  - the work of the speculative decodes of a blob full of 00 00 FF FF stays linear in its size;
  - update_from_tar(MKHOST_GUNZIP) against the uncompressed ingest of zlib's output.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_gunzip_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import os
import sys

import pytest

from tests import mock_engine


@pytest.mark.parametrize("scenario", ["corpus", "linear_work", "ingest"])
def test_gunzip_mock(tmp_path, scenario):
    mock_engine.run("tests.test_host_gunzip_cpu", scenario, tmp_path)


def test_fuzz_under_asan_ubsan(tmp_path):
    r = mock_engine.run("tests.test_host_gunzip_cpu", "fuzz", tmp_path, sanitize=True)
    assert "fuzz ok" in r.stdout


def test_describe_refuses_gunzip(tmp_path):
    from makisu_b200 import host
    from tests import gzip_corpus as gc
    blob = gc.layer_blobs()[1][1]
    path = tmp_path / "layer.gz"
    path.write_bytes(blob)
    (tmp_path / "root").mkdir()
    with open(path, "rb") as f, pytest.raises(host.HostError, match="uncompressed tars only"):
        host.MemFS(str(tmp_path / "root")).describe_update_from_tar(0, f.fileno(), flags=host.MKHOST_GUNZIP)


# ---------------------------------------------------------------------------------------------------------------
def _engine(mock):
    from makisu_b200 import abi
    cfg = abi.Config()
    cfg.max_extents = 64
    h = C.c_void_p()
    mock.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
    assert mock.mksnap_create(C.byref(cfg), C.byref(h)) == 0
    return h


def corpus(mock, tmp):
    from tests import gzip_corpus as gc
    h = _engine(mock)
    for name, blob in gc.corpus():
        want = gc.go_gunzip(blob)
        for chunk in (1 << 20, 4097):
            rc, got, info = gc.engine_gunzip(mock, h, blob, chunk)
            if want is None:
                assert rc == gc.MKSNAP_E_DATA, name
            else:
                assert rc == 0 and got == want, name
                assert (info.gz_bytes, info.out_bytes) == (len(blob), len(want))
                assert info.n_segments >= info.n_members >= 1
        if name.startswith("pgzip") or name in ("full_flush", "sync_flush_one_stream"):
            assert info.n_segments > 3, name  # decoded in pieces, references across segment boundaries resolved
    # where Python's gzip and Go part ways, the engine is Go
    import gzip
    zero_padded = dict(gc.corpus())["zero_padding"]
    assert gzip.decompress(zero_padded) and gc.go_gunzip(zero_padded) is None
    # an error leaves the handle usable; a second open without close is refused
    info = gc.GunzipInfo()
    good = dict(gc.corpus())["multi_member"]
    assert mock.mksnap_gunzip_open(h, good, len(good), C.byref(info)) == 0
    assert mock.mksnap_gunzip_open(h, good, len(good), C.byref(info)) == -5
    assert mock.mksnap_gunzip_close(h) == 0
    assert gc.engine_gunzip(mock, h, good)[1] == gc.go_gunzip(good)


def fuzz(mock, tmp):
    from tests import gzip_corpus as gc
    h = _engine(mock)
    n_bad = 0
    for blob in gc.fuzz_cases(3000, seed=11):
        want = gc.go_gunzip(blob)
        rc, got, _ = gc.engine_gunzip(mock, h, blob, 5000)
        if want is None:
            assert rc == gc.MKSNAP_E_DATA, blob[:64].hex()
            n_bad += 1
        else:
            assert rc == 0 and got == want, blob[:64].hex()
    assert n_bad >= 1000, n_bad
    print("fuzz ok", n_bad)


def linear_work(mock, tmp):
    """Every byte after a 00 00 FF FF is a candidate start; a stored block full of them would make unlimited
    speculative decodes quadratic.  With the K limit the input all decodes go through stays a small multiple of the
    blob, and the same multiple at 4x the size."""
    from tests import gzip_corpus as gc
    mock.mock_gunzip_consumed.restype = mock.mock_gunzip_candidates.restype = C.c_uint64
    h = _engine(mock)
    ratios = []
    for n in (50_000, 200_000):
        pat = b"\x00\x00\xff\xff" * n
        blob = gc.gzip_member(gc.deflate(pat, 0), pat)
        rc, got, _ = gc.engine_gunzip(mock, h, blob)
        assert rc == 0 and got == pat
        assert mock.mock_gunzip_candidates() >= n
        ratios.append(mock.mock_gunzip_consumed() / len(blob))
    assert max(ratios) <= 4 * 6, ratios  # each decode stops within K + 1 candidates of 4 bytes, K = 4
    assert abs(ratios[1] - ratios[0]) < 1.0, ratios


def ingest(mock, tmp):
    from tests import gzip_corpus as gc
    from tests.mock_engine.scenarios import MockEngineFactory
    from makisu_b200 import host
    make = MockEngineFactory(mock)
    untar = [host.MKHOST_UNTAR, host.MKHOST_UNTAR | host.MKHOST_FILE_DIGESTS] if os.geteuid() == 0 else []  # chown
    for flags in [0, host.MKHOST_FILE_DIGESTS, host.MKHOST_NO_TAR_DIGEST] + untar:
        for name, blob in gc.layer_blobs():
            if flags & host.MKHOST_UNTAR and name == "big_member_multi":
                continue  # MKHOST_UNTAR needs every member inside one arena, compressed or not
            gc.check_ingest(make, tmp, name, blob, flags)
    # a damaged blob fails the call; the engine handle (a fresh one per call here) is not left with an open gunzip
    good = gc.layer_blobs()[1][1]
    bad = bytearray(good)
    bad[-6] ^= 1
    path = os.path.join(tmp, "bad.gz")
    open(path, "wb").write(bytes(bad))
    root = os.path.join(tmp, "bad_root")
    os.mkdir(root)
    eng = make(1 << 20)
    try:
        with open(path, "rb") as f:
            host.MemFS(root).update_from_tar(eng, 0, f.fileno(), flags=host.MKHOST_GUNZIP)
        raise AssertionError("expected a gunzip error")
    except host.HostError as e:
        assert "CRC-32 or length mismatch" in str(e), str(e)
    info = gc.GunzipInfo()
    assert mock.mksnap_gunzip_open(eng.h, good, len(good), C.byref(info)) == 0
    assert mock.mksnap_gunzip_close(eng.h) == 0


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=scenario == "ingest")
    from tests import gzip_corpus as gc
    gc.bind(mock)
    globals()[scenario](mock, tmp)


if __name__ == "__main__":
    main()
