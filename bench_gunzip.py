"""Gunzip of layer blobs on the GPU (mksnap_gunzip_*, update_from_tar with MKHOST_GUNZIP) against zlib on one core.

Workload: a synthetic layer tar (default 1 GiB) of files that are text-like, run-heavy or random (incompressible), in
two blobs:
  - pgzip-shaped, the layout makisu's own layers have (1 MiB blocks, each with the previous 32 KiB as a preset
    dictionary and a sync flush): one segment per block, decoded in parallel;
  - one gzip.compress member of the first --single-mib MiB: no flush points, one segment, decoded by one GPU thread.
Legs, best of --reps after one warm-up, every output checked against zlib before it is timed:
  - gunzip: mksnap_gunzip_open + reads into a host buffer; kernel times from the engine's CUDA events;
  - zlib: zlib.decompress on one core (CPython's zlib; Go's compress/flate is not measured here);
  - ingest: update_from_tar(blob, MKHOST_GUNZIP) against zlib streaming the tar through a pipe into
    update_from_tar(pipe).
Prints the card name and power limit, then one JSON line.

    python bench_gunzip.py [--gib 1] [--single-mib 64] [--reps 3]"""
import argparse
import ctypes as C
import gzip
import io
import json
import os
import random
import subprocess
import tarfile
import tempfile
import threading
import time
import zlib

import numpy as np

from makisu_b200 import abi, host
from tests import gzip_corpus as gc


def layer_tar(total: int, seed: int = 1) -> bytes:
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    text = gc.mixed(rng, 32 << 20)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        i, size = 0, 0
        while size < total:
            n = int(min(total - size, rng.choice([4096, 65536, 1 << 20, 8 << 20])))
            k = i % 3
            if k == 0:
                o = rng.randrange(len(text) - n) if n < len(text) else 0
                data = text[o:o + n]
            elif k == 1:
                data = nrng.integers(0, 256, n, dtype=np.uint8).tobytes()
            else:
                data = (bytes(range(256)) * (n // 256 + 1))[:n]
            ti = tarfile.TarInfo("usr/share/f%06d" % i)
            ti.size, ti.mtime, ti.mode = len(data), 1_500_000_000, 0o644
            tf.addfile(ti, io.BytesIO(data))
            i += 1
            size += len(data) + 512
    return buf.getvalue()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def best(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return min(ts), out


def gunzip_leg(eng, blob, want, reps, chunk=256 << 20):
    lib = eng.lib
    buf = (C.c_uint8 * chunk)()
    out = np.empty(len(want), dtype=np.uint8)

    def run():
        eng.gunzip_open(blob)
        pos, got = 0, C.c_uint64()
        while True:
            eng._ck(lib.mksnap_gunzip_read(eng.h, buf, chunk, C.byref(got)), "gunzip_read")
            out[pos:pos + got.value] = np.frombuffer(buf, dtype=np.uint8, count=got.value)
            pos += got.value
            if got.value < chunk:
                break
        t = eng.gunzip_times()
        info_t = {k: round(getattr(t, k), 2) for k, _ in t._fields_}
        eng.gunzip_close()
        return pos, info_t

    pos, _ = run()
    assert pos == len(want) and out.tobytes() == want, "gunzip output differs from zlib"
    info = eng.gunzip_open(blob)
    eng.gunzip_close()
    s, (_, times) = best(run, reps)
    return s, times, {k: getattr(info, k) for k, _ in info._fields_}


def ingest_legs(blob, want, reps, tmp):
    path = os.path.join(tmp, "layer.gz")
    open(path, "wb").write(blob)

    def engine():
        return abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=64 << 20,
                          max_extents=1 << 14)

    def gpu():
        root = tempfile.mkdtemp(dir=tmp)
        with engine() as e, open(path, "rb") as f:
            return host.MemFS(root).update_from_tar(e, 1_600_000_000, f.fileno(), flags=host.MKHOST_GUNZIP)

    def cpu():
        root = tempfile.mkdtemp(dir=tmp)
        r, w = os.pipe()

        def feed():
            d = zlib.decompressobj(31)
            with open(w, "wb", closefd=True) as wf:
                for i in range(0, len(blob), 4 << 20):
                    wf.write(d.decompress(blob[i:i + (4 << 20)]))
                wf.write(d.flush())
        t = threading.Thread(target=feed)
        t.start()
        with engine() as e:
            res = host.MemFS(root).update_from_tar(e, 1_600_000_000, r)
        t.join()
        os.close(r)
        return res

    a, b = gpu(), cpu()
    assert a == b, "update_from_tar(MKHOST_GUNZIP) differs from zlib + update_from_tar"
    tg, _ = best(gpu, reps)
    tc, _ = best(cpu, reps)
    return tg, tc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--single-mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    tar = layer_tar(int(a.gib * (1 << 30)))
    pg = gc.pgzip(tar, block=1 << 20, level=6)
    single_tar = tar[:a.single_mib << 20]
    single = gzip.compress(single_tar, 6)
    res = {"card": card(), "tar_bytes": len(tar), "pgzip_bytes": len(pg), "single_bytes": len(single),
           "single_tar_bytes": len(single_tar)}
    with abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=1, host_arena_bytes=8 << 20) as eng:
        for name, blob, want in (("pgzip", pg, tar), ("single", single, single_tar)):
            tz, out = best(lambda: zlib.decompress(blob, 31), a.reps)
            assert out == want
            tg, times, info = gunzip_leg(eng, blob, want, a.reps)
            res[name] = {"gpu_s": round(tg, 4), "zlib_s": round(tz, 4), "gpu_GBps": round(len(want) / tg / 1e9, 3),
                         "zlib_GBps": round(len(want) / tz / 1e9, 3), "kernel_ms": times, "info": info}
            print(name, json.dumps(res[name]), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        tg, tc = ingest_legs(pg, tar, a.reps, tmp)
    res["ingest_pgzip"] = {"gpu_gunzip_s": round(tg, 4), "zlib_pipe_s": round(tc, 4)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
