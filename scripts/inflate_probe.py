"""Measures the device chunk inflater (include/esvo_b200_inflate.h) and the closed loop on a bz2 bag.  Prints one JSON line:
- the card and its power limit, read in the same call;
- device inflate throughput, decompressed GB/s, for batches of 16, 128, 1 024 and 4 096 chunks of 768 KiB, bz2 and LZ4:
  one esvo_inflate_chunks call, host call to its (synchronising) return, median of --reps after one warm-up.  The batches
  repeat a set of distinct seeded event-bag chunks (chunks are independent; compressing gigabytes in Python would take
  too long);
- the all-core host baseline in the same call: Python's bz2.decompress of the same bz2 chunks over a process pool with
  every host core (the workers return only the length, so no output is shipped back);
- bag_system (examples/bag_system.cpp) wall ms per second of stream on the dense hkust scene written as an uncompressed
  and as a bz2 bag, alternating, --runs each; the start-up inflate time of the bz2 bag (printed by bag_system) apart.
Writes bags and binaries into a temporary directory; writes nothing in the tree.
usage: python scripts/inflate_probe.py [--reps 3] [--runs 2] [--distinct 8] [--seconds 2.0]"""
import argparse
import bz2
import ctypes as C
import json
import multiprocessing as mp
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
L, R, LI, RI = "/davis/left/events", "/davis/right/events", "/davis/left/camera_info", "/davis/right/camera_info"
CHUNK = 768 * 1024


def _bz2_len(c):
    return len(bz2.decompress(c))


def event_chunks(tmp, distinct, seed=1):
    """distinct chunks of an event bag (about CHUNK bytes each, uncompressed) and their uncompressed data"""
    import compressed_bags as cb
    import rosbag_writer as rw
    rng = np.random.default_rng(seed)
    n = distinct * CHUNK // 13 + 20_000
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(1_600_000_000 * 10**9 + np.cumsum(rng.integers(0, 2000, n))).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    raw = rw.write_event_bag(os.path.join(tmp, "p.bag"), {L: e}, chunk_threshold=CHUNK, extras=False)
    plain = [d for _, _, _, d in cb.chunks(raw)][:distinct]
    return plain, [bz2.compress(d, 9) for d in plain], [cb.frame(d, bd=5, block_checksum=True, content_checksum=True) for d in plain]


def device(a, plain, comp, codec):
    from esvo_b200 import capi
    lib = capi.load_product()
    inf = capi.Inflater(lib, 0, 1 << 30)
    srcs = [np.frombuffer(c, np.uint8) for c in comp]
    dsts = [np.empty(len(p), np.uint8) for p in plain]
    f = lib.fn("inflate_chunks")
    f.argtypes = [C.c_void_p, C.POINTER(capi.Chunk), C.c_int]
    out = {}
    for n in a.sizes:
        arr = (capi.Chunk * n)()
        for k in range(n):
            j = k % len(srcs)
            arr[k] = capi.Chunk(srcs[j].ctypes.data, srcs[j].size, dsts[j].ctypes.data, dsts[j].size, codec, 0)
        ms = []
        for r in range(a.reps + 1):
            t = time.perf_counter()
            rc = f(inf.h, arr, n)
            ms.append((time.perf_counter() - t) * 1e3)
            if rc != 0:
                raise SystemExit(f"esvo_inflate_chunks: {rc} {inf.last_error()}")
        assert all(d.tobytes() == p for d, p in zip(dsts, plain))
        med = float(np.median(ms[1:]))
        out[n] = {"ms": round(med, 2), "GB_per_s": round(sum(len(plain[k % len(plain)]) for k in range(n)) / med / 1e6, 3)}
    inf.close()
    return out


def host(a, plain, comp):
    out = {}
    cores = os.cpu_count()
    with mp.get_context("fork").Pool(cores) as pool:
        pool.map(_bz2_len, comp)   # warm the workers
        for n in a.sizes:
            batch = [comp[k % len(comp)] for k in range(n)]
            t = time.perf_counter()
            got = pool.map(_bz2_len, batch, chunksize=max(1, n // (4 * cores)))
            ms = (time.perf_counter() - t) * 1e3
            assert sum(got) == sum(len(plain[k % len(plain)]) for k in range(n))
            out[n] = {"ms": round(ms, 2), "GB_per_s": round(sum(got) / ms / 1e6, 3)}
    return out, cores


def loop(a, tmp):
    import compressed_bags as cb
    import indep_system as isy
    import rosbag_writer as rw
    from bag_probe import compile_example
    from esvo_b200 import configs, synth
    exe = compile_example(tmp, "bag_system")
    rr = configs.RIGS["hkust"]
    infos = {t: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for t, sd in ((LI, "left"), (RI, "right"))}
    s = synth.make_stream("hkust", seed=2, t_ts=a.seconds, history_ms=a.seconds * 1e3)
    t0 = s["t_ts_ns"] - int(round(a.seconds * 1e9)) + 10_000_000
    n = int(round(a.seconds * 100))
    plain = os.path.join(tmp, "plain.bag")
    raw = rw.write_event_bag(plain, {L: s["left"], R: s["right"]}, infos=infos, msg_events=1500, chunk_threshold=CHUNK)
    bzb = os.path.join(tmp, "bz2.bag")
    with open(bzb, "wb") as f:
        f.write(cb.recompress(raw, "bz2"))
    res, traj = os.path.join(tmp, "r.bin"), os.path.join(tmp, "t.txt")
    out = {"plain": [], "bz2": [], "bz2_inflate_ms": [], "bag_MB": round(len(raw) / 1e6, 1), "bz2_bag_MB": round(os.path.getsize(bzb) / 1e6, 1)}
    for _ in range(a.runs):
        for k, bag in (("plain", plain), ("bz2", bzb)):
            p = subprocess.run([exe, bag, L, R, LI, RI, res, traj, "--t0-ns", str(t0), "--dt-ns", "10000000", "--ticks", str(n)],
                               capture_output=True, text=True)
            if p.returncode:
                raise SystemExit(p.stdout + p.stderr)
            out[k].append(round(isy.parse_result(res)[4] / a.seconds, 1))
            m = re.search(r"inflated \d+ bytes of compressed chunks in ([0-9.]+) ms", p.stdout)
            if k == "bz2":
                out["bz2_inflate_ms"].append(float(m.group(1)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--distinct", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 128, 1024, 4096])
    a = ap.parse_args()
    from bag_probe import card
    name, power = card()
    with tempfile.TemporaryDirectory() as tmp:
        plain, zb, zl = event_chunks(tmp, a.distinct)
        res = {"card": name, "power_limit": power, "chunk_bytes": len(plain[0]),
               "bz2_ratio": round(sum(map(len, plain)) / sum(map(len, zb)), 2), "lz4_ratio": round(sum(map(len, plain)) / sum(map(len, zl)), 2)}
        res["device_bz2"] = device(a, plain, zb, 1)
        res["device_lz4"] = device(a, plain, zl, 2)
        res["host_bz2_all_cores"], res["host_cores"] = host(a, plain, zb)
        res["bag_system_dense_wall_ms_per_stream_s"] = loop(a, tmp)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
