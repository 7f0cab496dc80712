"""CPU: mkhost_memfs_update_from_tars (a run of layers in one engine session, DiffID chains deferred to the stream log)
under the CPU mock engine (tests/mock_engine/mock_mksnap.cpp).  In each case the run equals one
update_from_tar call per layer (tests/apply_layers.py): per-layer DiffID, entries and tar bytes, the tree (a probe layer
described against it), remembered file digests and, under MKHOST_UNTAR, the files on disk.  Layers: whiteouts and
overwrites of what an earlier layer added, a hard link to an earlier layer's file, an empty layer, gzip and plain blobs,
a member larger than the arena (without untar); a damaged layer in the middle leaves the layers before it merged.
Each scenario runs in a fresh process that loads the mock with RTLD_GLOBAL before libmkhost:
    python -m tests.test_host_update_from_tars_cpu <mock.so> <scenario> <tmpdir>"""
import os
import sys

import pytest

from tests import mock_engine


@pytest.mark.parametrize("scenario", ["run", "damaged_layer", "too_few_slots", "no_layers"])
def test_update_from_tars_mock(tmp_path, scenario):
    r = mock_engine.run("tests.test_host_update_from_tars_cpu", scenario, tmp_path)
    assert "SCENARIO-OK" in r.stdout


# ---------------------------------------------------------------------------------------------------------------
def run(make, tmp):
    from makisu_b200 import host
    from tests import apply_layers as al
    untar = [host.MKHOST_UNTAR, host.MKHOST_UNTAR | host.MKHOST_FILE_DIGESTS] if os.geteuid() == 0 else []  # chown
    for flags in [0, host.MKHOST_FILE_DIGESTS, host.MKHOST_NO_TAR_DIGEST] + untar:
        d = os.path.join(tmp, "flags%d" % flags)
        os.mkdir(d)
        # MKHOST_UNTAR writes a member from one contiguous body: no member larger than the arena there
        layers = al.layer_run(big=not flags & host.MKHOST_UNTAR)
        res = al.check_run(make, d, layers, flags)
        assert [r["n_entries"] for r in res][2] == 0 and len(res) == len(layers)


def damaged_layer(make, tmp):
    """Layer 1 of 3 fails (gzip CRC-32): the call fails; layer 0 stays merged, as after separate calls."""
    from makisu_b200 import host
    from tests import apply_layers as al
    layers = al.layer_run(big=False)
    bad = bytearray(layers[1][1])
    bad[-6] ^= 1
    run3 = [layers[0], ("damaged", bytes(bad), True), layers[3]]
    for flags in [0, host.MKHOST_FILE_DIGESTS] + ([host.MKHOST_UNTAR] if os.geteuid() == 0 else []):
        d = os.path.join(tmp, "flags%d" % flags)
        os.mkdir(d)
        paths = []
        for i, (_, blob, _) in enumerate(run3):
            paths.append(os.path.join(d, "l%d" % i))
            open(paths[-1], "wb").write(blob)
        roots = [os.path.join(d, "single"), os.path.join(d, "run")]
        for r in roots:
            os.mkdir(r)
        fs_s, fs_r = host.MemFS(roots[0]), host.MemFS(roots[1])
        for p, (_, _, z) in zip(paths, run3):
            with open(p, "rb") as f:
                try:
                    fs_s.update_from_tar(make(1 << 20), al.NOW, f.fileno(), flags=flags | (host.MKHOST_GUNZIP if z else 0))
                except host.HostError:
                    break
        fh = [open(p, "rb") for p in paths]
        try:
            fs_r.update_from_tars(make(1 << 20), al.NOW, [(f.fileno(), host.MKHOST_GUNZIP if z else 0)
                                                          for f, (_, _, z) in zip(fh, run3)], flags=flags)
            raise AssertionError("expected the damaged layer to fail the run")
        except host.HostError as e:
            assert "CRC-32 or length mismatch" in str(e), str(e)
        finally:
            for f in fh:
                f.close()
        tars = al.plain([layers[0], layers[1], layers[3]])
        names = {m for t in tars for m in al.tarfile.open(fileobj=al.io.BytesIO(t)).getnames()}
        for n in names:
            assert fs_s.file_digest("/" + n) == fs_r.file_digest("/" + n), n
        pr = os.path.join(d, "probe")
        open(pr, "wb").write(al.probe(tars))
        texts = []
        for fs in (fs_s, fs_r):
            with open(pr, "rb") as f:
                texts.append(fs.describe_update_from_tar(al.NOW, f.fileno()))
        assert texts[0] == texts[1]
        if flags & host.MKHOST_UNTAR:
            from tests.mock_engine import scenarios
            # no mtimes: the failed layer never restores its parent directories' mtimes, they hold the time of the write
            assert scenarios._tree(roots[0]) == scenarios._tree(roots[1])
            assert os.path.exists(os.path.join(roots[1], "app", "keep"))


def too_few_slots(make, tmp):
    """More layers than stream slots: refused before any layer is read (the tree stays empty)."""
    from makisu_b200 import host
    from tests import apply_layers as al
    layers = al.layer_run(big=False)
    paths = []
    for i, (_, blob, _) in enumerate(layers):
        paths.append(os.path.join(tmp, "l%d" % i))
        open(paths[-1], "wb").write(blob)
    root = os.path.join(tmp, "root")
    os.mkdir(root)
    fs = host.MemFS(root)
    fh = [open(p, "rb") for p in paths]
    try:
        fs.update_from_tars(make(1 << 20, max_extents=3), al.NOW, [(f.fileno(), host.MKHOST_GUNZIP if z else 0)
                                                                   for f, (_, _, z) in zip(fh, layers)])
        raise AssertionError("expected a stream-slot error")
    except host.HostError as e:
        assert "stream slot per layer" in str(e), str(e)
    assert all(f.tell() == 0 for f in fh)
    for f in fh:
        f.close()
    assert fs.file_digest("/app/keep") is None
    try:  # MKHOST_FILE_DIGESTS needs a slot after the layers
        fs.update_from_tars(make(1 << 20, max_extents=2), al.NOW, [os.open(paths[0], os.O_RDONLY), os.open(paths[2], os.O_RDONLY)],
                            flags=host.MKHOST_FILE_DIGESTS)
        raise AssertionError("expected a stream-slot error")
    except host.HostError as e:
        assert "per-file digests" in str(e), str(e)


def no_layers(make, tmp):
    from makisu_b200 import host
    root = os.path.join(tmp, "root")
    os.mkdir(root)
    assert host.MemFS(root).update_from_tars(make(1 << 20), 0, []) == []
    with pytest.raises(host.HostError, match="per-layer flag"):
        host.MemFS(root).update_from_tars(make(1 << 20), 0, [(0, host.MKHOST_UNTAR)])


def main():
    mock_path, scenario, tmp = sys.argv[1:4]
    mock = mock_engine.load_for_child(mock_path, host=True)
    from tests.mock_engine.scenarios import MockEngineFactory
    globals()[scenario](MockEngineFactory(mock), tmp)
    print("SCENARIO-OK", scenario)


if __name__ == "__main__":
    main()
