"""Applying a run of layers: one update_from_tar call per layer (each its own engine session, its DiffID chain hashed
alone) against one update_from_tars call (one session, every layer's DiffID deferred to the stream log and the chains
hashed together).

Workload: 1, 4 and 16 synthetic layers whose sizes cycle through 4, 16, 32 and 8 MiB (files of 4 KiB - 8 MiB:
text-like, random and repetitive), as plain tars and as pgzip-shaped gzip blobs (MKHOST_GUNZIP), each without and with
MKHOST_UNTAR (members owned by the running user, so that no privilege is needed).  Per leg: best of --reps after one
warm-up, wall time of the whole call on a 64 MiB-arena engine; the engine's ms_stream of the last submit and ms_flush
of the last stream-log flush (CUDA events) from the timed call.  Results of both ways are checked to be identical before
anything is timed.  Prints the card name and power limit (read in the same process), then one JSON line per leg and one
JSON line with everything.

    python bench_apply_layers.py [--layers 1,4,16] [--reps 3]"""
import argparse
import io
import json
import os
import random
import shutil
import subprocess
import tarfile
import tempfile
import time

import numpy as np

from makisu_b200 import abi, host
from tests import gzip_corpus as gc

SIZES_MIB = (4, 16, 32, 8)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def layer_tar(i: int, total: int) -> bytes:
    rng = random.Random(i)
    nrng = np.random.default_rng(i)
    text = gc.mixed(rng, 4 << 20)
    buf = io.BytesIO()
    with tarfile.open(fileobj=buf, mode="w", format=tarfile.PAX_FORMAT) as tf:
        d = tarfile.TarInfo("layer%02d" % i)  # untar writes members into existing directories only
        d.type, d.mtime, d.mode, d.uid, d.gid = tarfile.DIRTYPE, 1_500_000_000, 0o755, os.getuid(), os.getgid()
        tf.addfile(d)
        k, size = 0, 0
        while size < total:
            n = int(min(total - size, rng.choice([4096, 65536, 1 << 20, 8 << 20])))
            if k % 3 == 0:
                o = rng.randrange(len(text) - n) if n < len(text) else 0
                data = text[o:o + n]
            elif k % 3 == 1:
                data = nrng.integers(0, 256, n, dtype=np.uint8).tobytes()
            else:
                data = (bytes(range(256)) * (n // 256 + 1))[:n]
            ti = tarfile.TarInfo("layer%02d/f%05d" % (i, k))
            ti.size, ti.mtime, ti.mode, ti.uid, ti.gid = len(data), 1_500_000_000, 0o644, os.getuid(), os.getgid()
            tf.addfile(ti, io.BytesIO(data))
            k += 1
            size += len(data) + 512
    return buf.getvalue()


def engine():
    return abi.Engine(device=0, device_arena_bytes=64 << 20, n_host_arenas=2, host_arena_bytes=64 << 20,
                      max_extents=1 << 14)


def leg(eng, paths, gz, flags, run, tmp):
    """One application of the layers on a fresh tree -> (seconds, results, ms_stream, ms_flush)."""
    root = tempfile.mkdtemp(dir=tmp)
    fs = host.MemFS(root)
    g = host.MKHOST_GUNZIP if gz else 0
    fh = [open(p, "rb") for p in paths]
    try:
        t0 = time.perf_counter()
        if run:
            res = fs.update_from_tars(eng, 1_600_000_000, [(f.fileno(), g) for f in fh], flags=flags)
        else:
            res = [fs.update_from_tar(eng, 1_600_000_000, f.fileno(), flags=flags | g) for f in fh]
        t = time.perf_counter() - t0
    finally:
        for f in fh:
            f.close()
    st = eng.stats()
    fs.close()
    shutil.rmtree(root)
    return t, res, st.ms_stream, st.ms_flush


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", default="1,4,16")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    name = card()
    print("card:", name, flush=True)
    counts = [int(x) for x in a.layers.split(",")]
    out = {"card": name, "sizes_mib": SIZES_MIB, "legs": []}
    with tempfile.TemporaryDirectory() as tmp:
        tars = [layer_tar(i, SIZES_MIB[i % len(SIZES_MIB)] << 20) for i in range(max(counts))]
        plain, gzp = [], []
        for i, t in enumerate(tars):
            plain.append(os.path.join(tmp, "l%02d.tar" % i))
            open(plain[-1], "wb").write(t)
            gzp.append(os.path.join(tmp, "l%02d.tar.gz" % i))
            open(gzp[-1], "wb").write(gc.pgzip(t, block=1 << 20, level=1))
        with engine() as eng:
            for n in counts:
                for gz in (False, True):
                    for untar in (False, True):
                        paths = (gzp if gz else plain)[:n]
                        flags = host.MKHOST_UNTAR if untar else 0
                        r_one = leg(eng, paths, gz, flags, False, tmp)[1]
                        r_run = leg(eng, paths, gz, flags, True, tmp)[1]
                        assert [(x["tar_digest"], x["n_entries"], x["tar_bytes"]) for x in r_one] == \
                               [(x["tar_digest"], x["n_entries"], x["tar_bytes"]) for x in r_run], "run differs"
                        rec = {"layers": n, "gzip": gz, "untar": untar,
                               "tar_bytes": sum(x["tar_bytes"] for x in r_run)}
                        for label, run in (("per_layer", False), ("run", True)):
                            best = None
                            for _ in range(a.reps):
                                t, _, ms_stream, ms_flush = leg(eng, paths, gz, flags, run, tmp)
                                if best is None or t < best[0]:
                                    best = (t, ms_stream, ms_flush)
                            rec[label] = {"wall_s": round(best[0], 4), "ms_stream_last_submit": round(best[1], 3),
                                          "ms_flush": round(best[2], 3) if run else None}
                        rec["speedup"] = round(rec["per_layer"]["wall_s"] / rec["run"]["wall_s"], 3)
                        print(json.dumps(rec), flush=True)
                        out["legs"].append(rec)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
