"""Incremental layer ingest: a run of layers applied without a cache (update_from_tars_indexed), with a cold layer cache
(every layer read, decompressed, hashed and recorded) and with a warm one (every layer replayed: the remembered members
merged, the remembered chunk digests appended, nothing read).

Workload: the layers of bench_apply_layers.py -- 16 synthetic layers whose sizes cycle through 4, 16, 32 and 8 MiB, as
plain tars and as pgzip-shaped gzip blobs -- and one 1 GiB pgzip layer, the shape whose single DiffID chain bounds an
uncached ingest.  Per leg: best of --reps after one warm-up, wall time of the whole call on a 64 MiB-arena engine,
blob_bytes_read of the layer cache's stats, and the engine's device times of that call's finish (mksnap_stats: K3 sort
and unique, Merkle root), which a warm run still pays in full.  Results of all three ways are checked to be
identical before anything is timed.  Prints the card name and power limit (read in the same process), then one JSON
line per leg and one JSON line with everything.

    python bench_ingest_cache.py [--reps 3] [--big-mib 1024]"""
import argparse
import json
import os
import shutil
import tempfile
import time

from bench_apply_layers import SIZES_MIB, card, layer_tar
from makisu_b200 import abi, host
from tests import gzip_corpus as gc


def engine():
    # a 1 GiB layer has ~65k chunks of the default CDC: more than the default table of a 64 MiB arena holds
    return abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=64 << 20,
                      max_extents=1 << 14, max_chunks=1 << 18)


def leg(eng, paths, gz, lc, tmp):
    """One application of the layers on a fresh tree -> (seconds, results, stats, device ms)."""
    root = tempfile.mkdtemp(dir=tmp)
    fs = host.MemFS(root)
    g = host.MKHOST_GUNZIP if gz else 0
    keys = [os.path.basename(p) for p in paths]
    fds = [os.open(p, os.O_RDONLY) for p in paths]
    try:
        t0 = time.perf_counter()
        if lc is None:
            res, st = fs.update_from_tars_indexed(eng, None, keys, 1_600_000_000, [(f, g) for f in fds])[0], None
        else:
            res, st, _ = fs.update_from_tars_cached(eng, lc, None, keys, 1_600_000_000, [(f, g) for f in fds])
        t = time.perf_counter() - t0
    finally:
        for f in fds:
            os.close(f)
    s = eng.stats()
    fs.close()
    shutil.rmtree(root)
    return t, res, st, {"ms_sort": round(s.ms_sort, 3), "ms_root": round(s.ms_root, 3)}


def bench(eng, name, paths, gz, reps, tmp):
    ref = leg(eng, paths, gz, None, tmp)[1]
    warm_cache = host.LayerCache()
    assert leg(eng, paths, gz, warm_cache, tmp)[1] == ref, "cold cache differs"
    assert leg(eng, paths, gz, warm_cache, tmp)[1] == ref, "warm cache differs"
    rec = {"workload": name, "layers": len(paths), "gzip": gz, "blob_bytes": sum(os.path.getsize(p) for p in paths)}
    for label, fresh in (("uncached", None), ("cold_cache", True), ("warm_cache", False)):
        best = None
        for _ in range(reps + 1):  # the first is the warm-up
            lc = None if fresh is None else (host.LayerCache() if fresh else warm_cache)
            t, _, st, ms = leg(eng, paths, gz, lc, tmp)
            if best is None or t < best[0]:
                best = (t, st, ms)
        t, st, ms = best
        rec[label] = {"wall_s": round(t, 4), "blob_bytes_read": st["blob_bytes_read"] if st else rec["blob_bytes"],
                      "layers_replayed": st["layers_replayed"] if st else 0, **ms}
    rec["warm_speedup_vs_uncached"] = round(rec["uncached"]["wall_s"] / rec["warm_cache"]["wall_s"], 2)
    print(json.dumps(rec), flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--big-mib", type=int, default=1024)
    a = ap.parse_args()
    name = card()
    print("card:", name, flush=True)
    out = {"card": name, "sizes_mib": SIZES_MIB, "legs": []}
    with tempfile.TemporaryDirectory() as tmp:
        plain, gzp = [], []
        for i in range(16):
            t = layer_tar(i, SIZES_MIB[i % len(SIZES_MIB)] << 20)
            plain.append(os.path.join(tmp, "l%02d.tar" % i))
            open(plain[-1], "wb").write(t)
            gzp.append(os.path.join(tmp, "l%02d.tar.gz" % i))
            open(gzp[-1], "wb").write(gc.pgzip(t, block=1 << 20, level=1))
        big = os.path.join(tmp, "big.tar.gz")
        open(big, "wb").write(gc.pgzip(layer_tar(99, a.big_mib << 20), block=1 << 20, level=1))
        with engine() as eng:
            out["legs"].append(bench(eng, "16_layers", plain, False, a.reps, tmp))
            out["legs"].append(bench(eng, "16_layers", gzp, True, a.reps, tmp))
            out["legs"].append(bench(eng, "1_layer_%d_mib" % a.big_mib, [big], True, a.reps, tmp))
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
