"""CPU: the files the four libmkhost caches keep between builds (mkhost_*_cache_save / _load, cache_file.inc).

tests/golden/cache_files/ holds one small file per cache, in the formats libmkhost has written since each cache was
added (an earlier libmkhost re-saves each of them byte for byte):
    crc.cache       three files, one path with a space
    chunk.cache     three files: one path with a space, one with three chunks, one with none
    gz_index.cache  three blobs: one key with spaces, one with three points, one with none
    layer.cache     three layers: with and without DiffID and file digests, a key with spaces, no members, and member
                    mtimes outside int64 (the two-word split), negative and positive
Checked: a load and a save give back each file byte for byte; every prefix of a file is either refused whole or loads
and re-saves to itself; a refused file leaves a populated cache as it was; and a loaded file merges into a crc cache and
into a chunk cache of the same CDC parameters, and replaces a chunk cache of other parameters, a gzip index cache and a
layer cache.  Everything runs once more, in a fresh process, with libmkhost built with AddressSanitizer and
UndefinedBehaviorSanitizer:
    python -m tests.test_host_cache_files_cpu <mock.so> every <tmpdir>"""
import os
import sys

import pytest

from tests import mock_engine

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cache_files")
KINDS = {"crc": "CrcCache", "chunk": "ChunkCache", "gz-index": "GzIndexCache", "layer": "LayerCache"}
LOADABLE_PREFIXES = {"crc": 4, "chunk": 4, "gz-index": 4, "layer": 1}  # the header alone, then after every entry


def _fixture(kind):
    with open(os.path.join(GOLDEN, kind.replace("-", "_") + ".cache"), "rb") as f:
        return f.read()


def _cache(kind, path=None):
    from makisu_b200 import host
    return getattr(host, KINDS[kind])(path)


def _write(tmp, name, data):
    path = os.path.join(tmp, name)
    with open(path, "wb") as f:
        f.write(data)
    return path


def _saved(cache, tmp):
    path = os.path.join(tmp, "saved.cache")
    cache.save(path)
    with open(path, "rb") as f:
        return f.read()


def _load(cache, kind, path):
    """True when the load succeeds; a refusal must say that the file is not one of this kind."""
    from makisu_b200 import host
    try:
        cache.load(path)
        return True
    except host.HostError as e:
        assert "not a mkhost-%s-cache file" % kind in str(e), str(e)
        return False


def _entries(kind):
    """A fixture in one of the line formats as its header line and its entries, each a line and its raw rows."""
    head, rest = _fixture(kind).split(b"\n", 1)
    entries = []
    while rest:
        line, rest = rest.split(b"\n", 1)
        f = line.split(b" ")
        n = 32 * int(f[5]) if kind == "chunk" else 8 * int(f[1]) if kind == "gz-index" else 0
        entries.append(line + b"\n" + rest[:n])
        rest = rest[n:]
    return head + b"\n", entries


def round_trip(tmp):
    for kind in KINDS:
        cache = _cache(kind, os.path.join(GOLDEN, kind.replace("-", "_") + ".cache"))
        assert len(cache) == 3, kind
        assert _saved(cache, tmp) == _fixture(kind), kind


def prefixes(tmp):
    for kind in KINDS:
        data, loaded = _fixture(kind), 0
        for n in range(len(data) + 1):
            cache = _cache(kind)
            if _load(cache, kind, _write(tmp, "prefix.cache", data[:n])):
                assert _saved(cache, tmp) == data[:n], (kind, n)
                loaded += 1
        assert loaded == LOADABLE_PREFIXES[kind], (kind, loaded)


# the same entries under other keys of the same length: none of them is in a cache loaded from the fixture
RENAMED = {"crc": (b"/ctx/", b"/new/"), "chunk": (b"/ctx/", b"/new/"), "gz-index": (b"spaces", b"SPACES"),
           "layer": (b"spaces", b"SPACES")}


def refused_leaves_cache(tmp):
    for kind in KINDS:
        data = _fixture(kind)
        cache = _cache(kind, _write(tmp, "good.cache", data))
        bad = data.replace(*RENAMED[kind])
        assert bad != data
        for damaged in (bad + b"garbage\n", bad + b"garbage", bad[:-1]):
            assert not _load(cache, kind, _write(tmp, "bad.cache", damaged)), kind
            assert len(cache) == 3 and _saved(cache, tmp) == data, kind


def merge_or_replace(tmp):
    # crc: merge, the loaded entry wins
    head, (a, b, z) = _entries("crc")
    b2 = b.replace(b" 00000000 ", b" 12345678 ")
    new = b"1 2 3 4 5 0badf00d /ctx/new\n"
    cache = _cache("crc", _write(tmp, "good.cache", _fixture("crc")))
    cache.load(_write(tmp, "more.cache", head + b2 + new))
    assert len(cache) == 4 and _saved(cache, tmp) == head + a + b2 + new + z
    # chunk, same CDC parameters: merge
    head, (big, empty, small) = _entries("chunk")
    empty2 = b"2049 201 64 1 1 1 /ctx/empty\n" + bytes(range(32))
    new = b"1 2 3 4 5 0 /ctx/new\n"
    cache = _cache("chunk", _write(tmp, "good.cache", _fixture("chunk")))
    cache.load(_write(tmp, "more.cache", head + empty2 + new))
    assert len(cache) == 4 and _saved(cache, tmp) == head + big + empty2 + new + small
    # chunk, other CDC parameters: replace, and take those parameters
    other = b"mkhost-chunk-cache 1 1024 4096 32768 14 10\n" + new
    cache.load(_write(tmp, "other.cache", other))
    assert len(cache) == 1 and _saved(cache, tmp) == other
    # gzip index: replace
    head, _ = _entries("gz-index")
    one = head + b"5 0 another key\n"
    cache = _cache("gz-index", _write(tmp, "good.cache", _fixture("gz-index")))
    cache.load(_write(tmp, "one.cache", one))
    assert len(cache) == 1 and _saved(cache, tmp) == one
    # layer: replace (with an empty cache's file, CDC parameters included)
    empty = _saved(_cache("layer"), tmp)
    cache = _cache("layer", _write(tmp, "good.cache", _fixture("layer")))
    cache.load(_write(tmp, "empty.cache", empty))
    assert len(cache) == 0 and _saved(cache, tmp) == empty


CHECKS = [round_trip, prefixes, refused_leaves_cache, merge_or_replace]


@pytest.mark.parametrize("check", CHECKS, ids=lambda c: c.__name__)
def test_cache_files(tmp_path, check):
    check(str(tmp_path))


def test_cache_files_under_asan_ubsan(tmp_path, monkeypatch):
    monkeypatch.setenv(mock_engine.SANITIZED_HOST, mock_engine.sanitized_host())
    r = mock_engine.run("tests.test_host_cache_files_cpu", "every", tmp_path, sanitize=True)
    assert "every ok" in r.stdout


def main():
    mock_path, _, tmp = sys.argv[1:4]
    mock_engine.load_for_child(mock_path, host=True)
    for check in CHECKS:
        check(tmp)
    print("every ok")


if __name__ == "__main__":
    main()
