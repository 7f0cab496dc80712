"""Gunzip of multi-member gzip blobs on the GPU (mksnap_gunzip_*) against zlib on one core.

Workload: the synthetic layer tar of bench_gunzip.py (default 1 GiB), compressed two ways at level 6:
  - BGZF-shaped (bgzip): one member per 65 280 input bytes, FEXTRA `BC` subfield, empty EOF member;
  - eStargz-shaped: one member per tar entry, large files split into 4 MiB chunk members, a TOC member and a footer.
Legs, best of --reps after one warm-up, every output checked against zlib before it is timed:
  - gpu: mksnap_gunzip_open + reads into a host buffer, with the kernel times and extra decodes of the engine;
  - zlib: zlib on one core, member after member (CPython's zlib; Go's compress/gzip is not measured here);
  - parent (with --parent-lib, a libmksnap.so built from an earlier commit): the same open + reads through that library
    in a subprocess, on the first --parent-mib MiB of the tar only: an engine that decodes each later member with a
    single-thread launch of its own takes minutes per GiB.  The new engine and zlib are timed on that smaller blob too.
Prints the card name and power limit, then one JSON line.

    python bench_gunzip_members.py [--gib 1] [--reps 2] [--parent-lib PATH] [--parent-mib 32]"""
import argparse
import ctypes as C
import json
import subprocess
import sys
import zlib

from bench_gunzip import best, card, layer_tar
from tests import gzip_corpus as gc
from tests import gzip_members as gm


def zlib_members(blob: bytes) -> bytes:
    """Every member in turn, fed in 1 MiB pieces so that finding where a member ends stays linear in the blob."""
    out, off, mv = [], 0, memoryview(blob)
    while off < len(blob):
        d = zlib.decompressobj(31)
        while not d.eof:
            if off >= len(blob):
                raise zlib.error("truncated member")
            piece = mv[off:off + (1 << 20)]
            out.append(d.decompress(piece))
            off += len(piece) - len(d.unused_data)
    return b"".join(out)


def engine_leg(lib, h, blob, want, reps, chunk=256 << 20):
    gc.bind(lib)
    lib.mksnap_gunzip_get_times.argtypes = [C.c_void_p, C.POINTER(gm.GunzipTimes)]
    buf = (C.c_uint8 * chunk)()
    out = bytearray(len(want))

    def run():
        info = gc.GunzipInfo()
        assert lib.mksnap_gunzip_open(h, blob, len(blob), C.byref(info)) == 0
        pos, got = 0, C.c_uint64()
        while True:
            assert lib.mksnap_gunzip_read(h, buf, chunk, C.byref(got)) == 0
            out[pos:pos + got.value] = memoryview(buf)[:got.value]
            pos += got.value
            if got.value < chunk:
                break
        t = gm.GunzipTimes()
        assert lib.mksnap_gunzip_get_times(h, C.byref(t)) == 0
        assert lib.mksnap_gunzip_close(h) == 0
        return pos, {k: round(getattr(t, k), 2) for k, _ in t._fields_}, \
            {k: getattr(info, k) for k, _ in info._fields_}

    pos, _, _ = run()
    assert pos == len(want) and out == want, "gunzip output differs from zlib"
    s, (_, times, info) = best(run, reps)
    return {"s": round(s, 4), "GBps": round(len(want) / s / 1e9, 3), "kernel_ms": times, "info": info}


def open_engine(lib_path):
    from makisu_b200 import abi
    lib = C.CDLL(lib_path) if lib_path else abi.load()
    lib.mksnap_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
    cfg = abi.Config()
    cfg.device, cfg.n_host_arenas, cfg.host_arena_bytes, cfg.device_arena_bytes = 0, 1, 8 << 20, 64 << 20
    cfg.max_extents = 1 << 20
    h = C.c_void_p()
    assert lib.mksnap_create(C.byref(cfg), C.byref(h)) == 0
    return lib, h


def blobs(tar):
    """{layout: (blob, its decompressed stream)}: the eStargz stream is the tar plus its TOC entry"""
    out = {"bgzf": gm.bgzf(tar), "estargz": gm.estargz(tar)}
    return {k: (b, tar if k == "bgzf" else zlib_members(b)) for k, b in out.items()}


def one_engine(lib_path, mib, reps):
    """{layout: leg} for one library on the first `mib` MiB layer (run in a subprocess of its own)."""
    tar = layer_tar(mib << 20)
    lib, h = open_engine(lib_path)
    res = {k: engine_leg(lib, h, b, want, reps) for k, (b, want) in blobs(tar).items()}
    lib.mksnap_destroy(h)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--parent-mib", type=int, default=32)
    ap.add_argument("--one-engine", nargs=3, metavar=("LIB", "MIB", "REPS"), help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.one_engine:
        lib_path, mib, reps = a.one_engine
        print(json.dumps(one_engine(lib_path if lib_path != "-" else None, int(mib), int(reps))))
        return
    print("card:", card(), flush=True)
    tar = layer_tar(int(a.gib * (1 << 30)))
    res = {"card": card(), "tar_bytes": len(tar)}
    lib, h = open_engine(None)
    for name, (blob, want) in blobs(tar).items():
        tz, out = best(lambda: zlib_members(blob), a.reps)
        assert out == want
        leg = engine_leg(lib, h, blob, want, a.reps)
        res[name] = {"gz_bytes": len(blob), "members": leg["info"]["n_members"], "gpu": leg,
                     "zlib_s": round(tz, 4), "zlib_GBps": round(len(want) / tz / 1e9, 3)}
        print(name, json.dumps(res[name]), flush=True)
    lib.mksnap_destroy(h)
    if a.parent_lib:
        small = layer_tar(a.parent_mib << 20)
        cmp = {"tar_bytes": len(small)}
        for who, path in (("new", "-"), ("parent", a.parent_lib)):
            r = subprocess.run([sys.executable, __file__, "--one-engine", path, str(a.parent_mib), "1"],
                               capture_output=True, text=True, check=True)
            cmp[who] = json.loads(r.stdout.strip().splitlines()[-1])
        for name, (blob, _) in blobs(small).items():
            cmp.setdefault("zlib_s", {})[name] = round(best(lambda: zlib_members(blob), a.reps)[0], 4)
        res["vs_parent"] = cmp
        print("vs_parent", json.dumps(cmp), flush=True)
    else:
        res["vs_parent"] = "not measured (no --parent-lib)"
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
