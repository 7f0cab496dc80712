"""Indexed gunzip of a single-member layer blob on the GPU (mksnap_gunzip_open_indexed) against zlib on one core.

Workload: the 1 GiB synthetic layer tar of bench_gunzip.py, compressed as one zlib level-6 gzip member: no flush
points, the shape the gzip CLI, Go's compress/gzip, containerd and docker write, and most registry layers have.
Legs, every output checked against zlib:
  - plain: mksnap_gunzip_open + reads.  The member is one segment decoded by one GPU thread, so this leg takes minutes
    at 1 GiB; it runs once on the first --plain-mib MiB of the tar (0: the whole tar);
  - record: mksnap_gunzip_open_indexed without points + reads: the open a first build pays, one serial count decode
    that records a block start about every 1 MiB of output, then parallel write decodes of the cut member; one run;
  - indexed: mksnap_gunzip_open_indexed with the recorded points + reads: what every later build pays; best of --reps
    after one warm-up;
  - zlib: zlib.decompress on one core (CPython's zlib), best of --reps;
  - layers: a run of --layers single-member layers of --layer-mib MiB each (level 6) through
    MemFS.update_from_tars_indexed with a warm gzip index cache, against zlib streaming each tar through a pipe into
    MemFS.update_from_tars, with and without MKHOST_NO_TAR_DIGEST; the cold run that fills the cache is reported too.
Prints the card name and power limit, then one JSON line.

    python bench_gunzip_index.py [--gib 1] [--plain-mib 64] [--layers 16] [--layer-mib 64] [--reps 3]"""
import argparse
import json
import os
import tempfile
import threading
import time
import zlib

import numpy as np

from bench_gunzip import best, card, layer_tar
from makisu_b200 import abi, host
from tests import gzip_corpus as gc


def gunzip_run(eng, blob, want, points=False, chunk=256 << 20):
    """One open + reads into a host buffer, checked after the clock stops: (seconds, kernel ms, info, index points,
    index info)."""
    out = np.empty(len(want) + chunk, dtype=np.uint8)
    t0 = time.perf_counter()
    if points is False:
        info = eng.gunzip_open(blob)
    else:
        info = eng.gunzip_open_indexed(blob, points)
    pos = 0
    while True:
        got = eng.gunzip_read(memoryview(out)[pos:pos + chunk])
        pos += got
        if got < chunk:
            break
    t = time.perf_counter() - t0
    times = eng.gunzip_times()
    pts, ix = eng.gunzip_index() if points is not False else (None, None)
    eng.gunzip_close()
    assert pos == len(want) and out[:pos].tobytes() == want, "gunzip output differs from zlib"
    ms = {k: round(getattr(times, k), 2) for k, _ in times._fields_}
    ixd = {k: getattr(ix, k) for k, _ in ix._fields_} if ix is not None else None
    return t, ms, {k: getattr(info, k) for k, _ in info._fields_}, pts, ixd


def layers_legs(blobs, reps, tmp):
    """(cold s, warm s, zlib-pipe s, cache stats of the warm run) for each of flags 0 and MKHOST_NO_TAR_DIGEST."""
    paths = []
    for i, b in enumerate(blobs):
        paths.append(os.path.join(tmp, "layer%02d.gz" % i))
        open(paths[-1], "wb").write(b)
    keys = ["layer%02d" % i for i in range(len(blobs))]

    def engine():
        return abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=64 << 20,
                          max_extents=1 << 14)

    def gpu(cache, flags):
        fds = [os.open(p, os.O_RDONLY) for p in paths]
        try:
            with engine() as e:
                t0 = time.perf_counter()
                res, st = host.MemFS(tempfile.mkdtemp(dir=tmp)).update_from_tars_indexed(
                    e, cache, keys, 1_600_000_000, [(f, host.MKHOST_GUNZIP) for f in fds], flags)
                return time.perf_counter() - t0, res, st
        finally:
            for f in fds:
                os.close(f)

    def cpu(flags):
        pipes = [os.pipe() for _ in blobs]

        def feed(blob, w):
            d = zlib.decompressobj(31)
            with open(w, "wb", closefd=True) as wf:
                for i in range(0, len(blob), 4 << 20):
                    wf.write(d.decompress(blob[i:i + (4 << 20)]))
                wf.write(d.flush())
        ts = [threading.Thread(target=feed, args=(b, w)) for b, (_, w) in zip(blobs, pipes)]
        with engine() as e:
            for t in ts:
                t.start()
            t0 = time.perf_counter()
            res = host.MemFS(tempfile.mkdtemp(dir=tmp)).update_from_tars(e, 1_600_000_000, [r for r, _ in pipes], flags)
            t = time.perf_counter() - t0
        for th in ts:
            th.join()
        for r, _ in pipes:
            os.close(r)
        return t, res

    out = {}
    for name, flags in (("digest", 0), ("no_tar_digest", host.MKHOST_NO_TAR_DIGEST)):
        cache = host.GzIndexCache()
        tcold, res_cold, _ = gpu(cache, flags)
        warm = [gpu(cache, flags) for _ in range(reps)]
        tw, res_w, st = min(warm, key=lambda r: r[0])
        cpu_runs = [cpu(flags) for _ in range(reps)]
        tc, res_c = min(cpu_runs, key=lambda r: r[0])
        assert res_cold == res_w == res_c, "update_from_tars_indexed differs from zlib + update_from_tars"
        out[name] = {"cold_s": round(tcold, 3), "warm_s": round(tw, 3), "zlib_pipe_s": round(tc, 3), "warm_stats": st}
        print("layers", name, json.dumps(out[name]), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--plain-mib", type=int, default=64)
    ap.add_argument("--layers", type=int, default=16)
    ap.add_argument("--layer-mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    tar = layer_tar(int(a.gib * (1 << 30)))
    blob = gc.gzip_member(gc.deflate(tar, 6), tar)
    plain_tar = tar[:a.plain_mib << 20] if a.plain_mib else tar
    plain_blob = gc.gzip_member(gc.deflate(plain_tar, 6), plain_tar) if a.plain_mib else blob
    res = {"card": card(), "tar_bytes": len(tar), "blob_bytes": len(blob), "plain_tar_bytes": len(plain_tar)}
    tz, out = best(lambda: zlib.decompress(blob, 31), a.reps)
    assert out == tar
    res["zlib"] = {"s": round(tz, 4), "GBps": round(len(tar) / tz / 1e9, 3)}
    print("zlib", json.dumps(res["zlib"]), flush=True)
    with abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=1, host_arena_bytes=8 << 20) as eng:
        t, ms, info, _, _ = gunzip_run(eng, plain_blob, plain_tar)
        tzp, _ = best(lambda: zlib.decompress(plain_blob, 31), a.reps)
        res["plain"] = {"s": round(t, 4), "zlib_s": round(tzp, 4), "kernel_ms": ms, "info": info}
        print("plain", json.dumps(res["plain"]), flush=True)
        t, ms, info, pts, ix = gunzip_run(eng, blob, tar, points=None)
        res["record"] = {"s": round(t, 4), "GBps": round(len(tar) / t / 1e9, 3), "kernel_ms": ms, "info": info,
                         "index": ix}
        print("record", json.dumps(res["record"]), flush=True)
        runs = [gunzip_run(eng, blob, tar, points=pts) for _ in range(a.reps + 1)][1:]  # the first is a warm-up
        ts, ms, info, _, ix = min(runs, key=lambda r: r[0])
        assert ix["points_linked"] == len(pts)
        res["indexed"] = {"s": round(ts, 4), "GBps": round(len(tar) / ts / 1e9, 3), "kernel_ms": ms, "info": info,
                          "index": ix}
        print("indexed", json.dumps(res["indexed"]), flush=True)
    tar = blob = None
    if a.layers:
        tars = [layer_tar(a.layer_mib << 20, seed=100 + i) for i in range(a.layers)]
        blobs = [gc.gzip_member(gc.deflate(t, 6), t) for t in tars]
        with tempfile.TemporaryDirectory() as tmp:
            res["layers"] = {"n": a.layers, "tar_bytes": sum(map(len, tars)), "blob_bytes": sum(map(len, blobs)),
                             **layers_legs(blobs, a.reps, tmp)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
