"""CPU: the gunzip (mksnap_gunzip_open / mksnap_gunzip_open_indexed) on hand-built DEFLATE blocks and on short
segments, under the CPU mock of the engine.

The mock (tests/mock_engine/mock_mksnap.cpp) runs the engine's decoder, link and resolve code
(makisu_b200/csrc/mksnap_inflate_core.h); the cases come from tests/deflate_blocks.py, where zlib is the judge of
every one:
  - blocks: every case through the plain open (zlib's bytes, or MKSNAP_E_DATA and then a valid blob on the same
    handle), and through the indexed open with a point at every block header, so that each block is a segment of its
    own: code lengths 1-15 on both sets, incomplete and empty sets, repeats across the lit/len and distance lengths,
    HLIT / HDIST / HCLEN at their limits, each of zlib's refusals, Go's empty final stored block and empty flush blocks,
    block headers at all 8 bit offsets;
  - short_segments: streams with a flush every 1 to 32769 bytes and empty segments mixed in, whose back-references
    reach over up to 32768 segments and, with the mock's 256 KiB windows, into the history of earlier windows;
  - the invalid cases once more through a mock built with ASan/UBSan.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL:
    python -m tests.test_host_deflate_blocks_cpu <mock.so> <scenario> <tmpdir>"""
import sys

import pytest

from tests import deflate_blocks as db
from tests import mock_engine
from tests.test_host_gunzip_cpu import _engine


@pytest.mark.parametrize("scenario", ["blocks", "short_segments"])
def test_deflate_blocks_mock(tmp_path, scenario):
    mock_engine.run("tests.test_host_deflate_blocks_cpu", scenario, tmp_path)


def test_invalid_blocks_under_asan_ubsan(tmp_path):
    r = mock_engine.run("tests.test_host_deflate_blocks_cpu", "invalid", tmp_path, sanitize=True)
    assert "invalid ok" in r.stdout


def test_zlib_agrees_with_every_declared_validity():
    cs = db.self_check()
    assert sum(c.valid for c in cs) >= 20 and sum(not c.valid for c in cs) >= 20


def test_block_headers_cover_every_bit_offset_class():
    classes = {}
    for c in db.cases():
        for p in db.points(c):
            classes.setdefault(p % 8, set()).add(c.name)
    assert sorted(classes) == list(range(8)), classes


# ---------------------------------------------------------------------------------------------------------------
def check_case(lib, h, case, good, chunk=4097):
    """One case through the plain open and the indexed open with a point at every block header."""
    from tests import gzip_corpus as gc
    from tests import gzip_index as gi
    blob, pts = db.member(case), db.points(case)
    want = gc.go_gunzip(blob)
    assert (want is not None) == case.valid, case.name
    rc, got, info = gc.engine_gunzip(lib, h, blob, chunk)
    if want is None:
        assert rc == gc.MKSNAP_E_DATA, (case.name, rc)
        rc, got, _, _, _ = gi.engine_gunzip_indexed(lib, h, blob, [p for p in pts if p < 8 * len(blob)], chunk)
        assert rc == gc.MKSNAP_E_DATA, (case.name, rc)
        rc, got, _ = gc.engine_gunzip(lib, h, good, chunk)  # the handle is still usable
        assert rc == 0 and got == gc.go_gunzip(good), case.name
        return
    assert rc == 0 and got == want, (case.name, rc, len(got), len(want))
    assert (info.gz_bytes, info.out_bytes, info.n_members) == (len(blob), len(want), 1), case.name
    rc, got, info, ix, _ = gi.engine_gunzip_indexed(lib, h, blob, pts, chunk)
    assert rc == 0 and got == want, (case.name, rc)
    assert ix.points_given == ix.points_linked == len(pts) and ix.points_recorded == 0, (case.name, ix.points_linked)
    assert info.n_segments == len(pts), (case.name, info.n_segments, len(pts))


def blocks(lib, h):
    cs = db.cases()
    good = db.member(next(c for c in cs if c.valid))
    for c in cs:
        check_case(lib, h, c, good)
    print("blocks ok", len(cs))


def invalid(lib, h):
    cs = db.cases()
    good = db.member(next(c for c in cs if c.valid))
    bad = [c for c in cs if not c.valid]
    for c in bad:
        check_case(lib, h, c, good)
    print("invalid ok", len(bad))


def check_short(lib, h, name, blob, data, segs, chunk=1 << 20):
    from tests import gzip_corpus as gc
    rc, got, info = gc.engine_gunzip(lib, h, blob, chunk)
    assert rc == 0 and info.out_bytes == len(data), (name, rc)
    assert info.n_segments == segs, (name, info.n_segments, segs)
    assert got == data, name


def short_segments(lib, h):
    from tests import gzip_corpus as gc
    for name, blob, data, segs in db.short_cases():
        assert gc.go_gunzip(blob) == data, name
        check_short(lib, h, name, blob, data, segs)
        print(name, len(blob), segs, flush=True)
    print("short_segments ok")


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path)
    from tests import gzip_index as gi
    gi.bind(mock)
    globals()[scenario](mock, _engine(mock))


if __name__ == "__main__":
    main()
