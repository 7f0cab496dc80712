"""CPU: gunzip of multi-member blobs (bgzip / BGZF, eStargz, concatenated members) under the CPU mock of the engine.

Every member body start is a candidate segment start, next to the flush points, so the members of such a blob are
count-decoded in parallel and the link needs no decode of its own per member.  The mock
(tests/mock_engine/mock_mksnap.cpp) runs the engine's candidate rule, decoder and link
(makisu_b200/csrc/mksnap_inflate_core.h); expectations come from Go's reader restated over zlib (tests/gzip_corpus.py):
  - BGZF, eStargz, every header-flag combination, empty members, false candidates, members with flushes, headers across
    a scan-chunk edge, trailing garbage, zero padding, bad trailers and truncated headers (tests/gzip_members.py);
  - the candidate table: sorted, every member body start tagged as one, flush points tagged as such;
  - a stored block full of valid member headers keeps the speculative work linear in the blob;
  - a few thousand fuzzed multi-member blobs through the mock built with ASan/UBSan;
  - update_from_tar(MKHOST_GUNZIP) of BGZF and eStargz layers against the uncompressed ingest.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_gunzip_members_cpu <mock.so> <scenario> <tmpdir>"""
import ctypes as C
import sys

import pytest

from tests import mock_engine
from tests.test_host_gunzip_cpu import _engine


@pytest.mark.parametrize("scenario", ["cases", "candidates", "linear_work", "ingest"])
def test_members_mock(tmp_path, scenario):
    mock_engine.run("tests.test_host_gunzip_members_cpu", scenario, tmp_path)


def test_members_fuzz_under_asan_ubsan(tmp_path):
    r = mock_engine.run("tests.test_host_gunzip_members_cpu", "fuzz", tmp_path, sanitize=True)
    assert "fuzz ok" in r.stdout


# ---------------------------------------------------------------------------------------------------------------
def _candidates(mock):
    mock.mock_gunzip_candidate.restype = C.c_uint32
    mock.mock_gunzip_candidate.argtypes = [C.c_uint64, C.POINTER(C.c_uint64)]
    out, off, i = [], C.c_uint64(), 0
    while True:
        k = mock.mock_gunzip_candidate(i, C.byref(off))
        if not k:
            return out
        out.append((off.value, k))
        i += 1


def cases(mock, tmp):
    from tests import gzip_members as gm
    h = _engine(mock)
    n_ok = n_bad = 0
    for name, blob in gm.cases():
        for chunk in (1 << 20, 4097):
            info, _ = gm.check(mock, h, name, blob, chunk)
        if info is None:
            n_bad += 1
            continue
        n_ok += 1
        if name.startswith(("bgzf", "estargz", "concat", "empty_members")) and name != "bgzf_eof_only":
            assert info.n_members > 3, name
    assert n_bad == 13 and n_ok > 60, (n_ok, n_bad)  # gm.malformed: every case is refused
    print("cases ok", n_ok, n_bad)


def candidates(mock, tmp):
    """The table the count pass and the link see: sorted, unique, kinds as the bytes say."""
    from tests import gzip_corpus as gc
    from tests import gzip_members as gm
    h = _engine(mock)
    for name, blob in gm.cases():
        gm.engine_gunzip_times(mock, h, blob)
        cand = _candidates(mock)
        offs = [o for o, _ in cand]
        assert offs == sorted(set(offs)), name
        first = gc._header_end(blob, 0)
        if first is None:
            continue
        assert cand[0] == (first, gm.CAND_MEMBER), name
        for o, k in cand[1:]:
            assert first < o <= len(blob), name
            assert bool(k & gm.CAND_FLUSH) == (blob[o - 4:o] == b"\x00\x00\xff\xff"), (name, o)
            if k & gm.CAND_MEMBER:  # some header before o ends there (the scan does not compare FHCRC)
                assert any(blob[q:q + 3] == b"\x1f\x8b\x08" for q in range(max(0, o - 66_000), o - 9)), (name, o)
        if gc.go_gunzip(blob) is not None:
            kinds = dict(cand)
            for b in gm.member_bodies(blob):
                assert kinds.get(b, 0) & gm.CAND_MEMBER, (name, b)
    # false candidates: member kinds well beyond the member count, both kinds present in one blob
    blob = dict(gm.cases())["false_candidates"]
    gm.engine_gunzip_times(mock, h, blob)
    cand = _candidates(mock)
    assert sum(1 for _, k in cand if k & gm.CAND_MEMBER) > 10 * len(gm.member_bodies(blob))
    blob = dict(gm.cases())["with_flushes"]
    gm.engine_gunzip_times(mock, h, blob)
    kinds = {k for _, k in _candidates(mock)}
    assert gm.CAND_FLUSH in kinds and gm.CAND_MEMBER in kinds
    # a body start that is also a flush end carries both bits: a header whose XFL / OS bytes are FF FF after mtime 0
    m = bytearray(gc.gzip_member(gc.deflate(b"abc"), b"abc"))
    m[8], m[9] = 0xFF, 0xFF
    blob = gc.gzip_member(gc.deflate(b"x"), b"x") + bytes(m)
    rc, got, info, extra = gm.engine_gunzip_times(mock, h, blob)
    assert rc == 0 and got == b"xabc" and extra == 0
    assert (gm.member_bodies(blob)[1], gm.CAND_FLUSH | gm.CAND_MEMBER) in _candidates(mock)
    print("candidates ok")


def fuzz(mock, tmp):
    from tests import gzip_corpus as gc
    from tests import gzip_members as gm
    h = _engine(mock)
    n_bad = 0
    for blob in gm.fuzz_cases(3000, seed=5):
        want = gc.go_gunzip(blob)
        rc, got, _ = gc.engine_gunzip(mock, h, blob, 7000)
        if want is None:
            assert rc == gc.MKSNAP_E_DATA, blob[:64].hex()
            n_bad += 1
        else:
            assert rc == 0 and got == want, blob[:64].hex()
    assert 1000 <= n_bad <= 2500, n_bad  # both outcomes are well represented
    print("fuzz ok", n_bad)


def linear_work(mock, tmp):
    """A stored block full of valid member headers makes nearly every byte run a candidate; with the K limit the input
    all speculative decodes go through stays a small multiple of the blob, the same multiple at 4x the size, and within
    the bound the 00 00 FF FF wall of test_host_gunzip_cpu asserts."""
    from tests import gzip_corpus as gc
    from tests import gzip_members as gm
    mock.mock_gunzip_consumed.restype = mock.mock_gunzip_candidates.restype = C.c_uint64
    h = _engine(mock)
    ratios = []
    for n in (200_000, 800_000):
        blob, pat = gm.header_wall(n)
        rc, got, _ = gc.engine_gunzip(mock, h, blob)
        assert rc == 0 and got == pat
        assert mock.mock_gunzip_candidates() >= n // 14
        ratios.append(mock.mock_gunzip_consumed() / len(blob))
    assert max(ratios) <= 4 * 6, ratios
    assert abs(ratios[1] - ratios[0]) < 1.0, ratios
    print("linear ok", ratios)


def ingest(mock, tmp):
    import io
    import random
    import tarfile
    from tests import gzip_corpus as gc
    from tests import gzip_members as gm
    from tests.mock_engine.scenarios import MockEngineFactory
    from makisu_b200 import host
    make = MockEngineFactory(mock)
    buf = io.BytesIO()
    r = random.Random(3)
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        for i, data in enumerate([gc.mixed(r, 1_500_000), r.randbytes(200_000), gc.mixed(r, 70_000), b""]):
            ti = tarfile.TarInfo("opt/f%d.bin" % i)
            ti.size, ti.mtime, ti.mode = len(data), 1_500_000_000, 0o644
            tf.addfile(ti, io.BytesIO(data))
    tar = buf.getvalue()
    for name, blob in (("bgzf", gm.bgzf(tar)), ("estargz", gm.estargz(tar, chunk=300_000))):
        assert len(gm.member_bodies(blob)) > 5
        for flags in (0, host.MKHOST_FILE_DIGESTS):
            gc.check_ingest(make, tmp, name, blob, flags)
    print("ingest ok")


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=scenario == "ingest")
    from tests import gzip_corpus as gc
    gc.bind(mock)
    globals()[scenario](mock, tmp)


if __name__ == "__main__":
    main()
