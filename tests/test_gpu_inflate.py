"""The device chunk inflater (esvo_b200/csrc/inflate.cu through capi.Inflater), the inflating bag reader (examples/bag_dump.cpp
--inflate-device 0) and the closed loop on compressed bags (examples/bag_system.cpp).  References: Python's bz2 and the
uncompressed data for the decoder, the uncompressed bag for the reader and the loop.  Structurally malformed streams are
exercised by the host build of the decoders only (tests/test_inflate_core_host.py); here the defects are checksums, CRCs
and declared sizes."""
import bz2
import os
import subprocess

import numpy as np
import pytest

import compressed_bags as cb
import rosbag_writer as rw
from test_inflate_core_host import BZ2, LZ4, bz2_inputs, lz4_inputs, lz4_sequence_frames, FLAGS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
L, R = "/davis/left/events", "/davis/right/events"
LI, RI = "/davis/left/camera_info", "/davis/right/camera_info"


def _compile(tmp_path_factory, name):
    exe = str(tmp_path_factory.mktemp("bin") / name)
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", name + ".cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    return exe


def _corpus():
    items = []
    for data in bz2_inputs().values():
        for level in range(1, 10):
            items.append((BZ2, bz2.compress(data, level), data))
    for k, fl in enumerate(FLAGS):
        for data in lz4_inputs().values():
            items.append((LZ4, cb.frame(data, bd=4 + k % 4, **fl), data))
    for f, data in lz4_sequence_frames():
        items.append((LZ4, f, data))
    return items


def test_corpus_in_mixed_batches(product_lib):
    from esvo_b200 import capi
    scratch = 24 << 20
    items = _corpus()
    assert max(len(d) for _, _, d in items) == 2_000_000   # the 2 MB bz2 chunks need more than half the scratch
    inf = capi.Inflater(product_lib, 0, scratch)
    order = np.random.default_rng(4).permutation(len(items))
    for a in range(0, len(order), 37):
        batch = [items[i] for i in order[a:a + 37]]
        rc, st, out = inf.inflate([(c, s, len(d)) for c, s, d in batch])
        assert rc == 0 and st == [0] * len(batch)
        for (c, s, d), o in zip(batch, out):
            assert o == d
    inf.close()


def test_capacity(product_lib):
    from esvo_b200 import capi
    inf = capi.Inflater(product_lib, 0, 1 << 20)
    data = bytes(range(256)) * 3072
    rc, st, _ = inf.inflate([(BZ2, bz2.compress(b"ok"), 2), (BZ2, bz2.compress(data), len(data))], ok=(-4,))
    assert rc == -4 and st == [0, -4] and "chunk 1" in inf.last_error() and "needs" in inf.last_error()


def _flip(b, byte, mask=1):
    b = bytearray(b)
    b[byte] ^= mask
    return bytes(b)


def test_checksum_and_size_defects(product_lib):
    """One defect per chunk: stored block CRC, combined CRC, LZ4 content checksum, declared size.  The first failing chunk is
    named, every defective chunk is refused with INVALID_ARG and every other chunk is decoded."""
    from esvo_b200 import capi
    data = lz4_inputs()["text"][:300_000]
    z, f = bz2.compress(data, 9), cb.frame(data, bd=5, content_checksum=True, block_checksum=True)
    defects = {
        "block_crc": (BZ2, _flip(z, 10), len(data)),                # the first block's CRC: bytes 10..13
        "combined_crc": (BZ2, _flip(z, len(z) - 2), len(data)),     # inside the last 32 bits before the padding
        "content_checksum": (LZ4, _flip(f, len(f) - 1), len(data)),
        "bz2_size": (BZ2, z, len(data) - 1),
        "lz4_size": (LZ4, f, len(data) + 1),
    }
    inf = capi.Inflater(product_lib, 0, 64 << 20)
    for k, (name, bad) in enumerate(defects.items()):
        chunks = [(BZ2, z, len(data)), (LZ4, f, len(data))] * 2
        chunks.insert(1 + k % 3, bad)
        rc, st, out = inf.inflate(chunks, ok=(-1,))
        assert rc == -1 and st[1 + k % 3] == -1 and f"chunk {1 + k % 3}:" in inf.last_error(), (name, st, inf.last_error())
        assert sum(s != 0 for s in st) == 1 and all(o == data for o, s in zip(out, st) if s == 0), name
    inf.close()


# ---------------------------------------------------------------- the reader
def _bag_corpus(tmp_path, threshold, conn_in_chunks):
    """test_bag_reader.py's corpus: message sizes 0, 1 and 100 000 and mixed, one message per chunk up to one chunk."""
    from test_bag_reader import _stream
    e, r = _stream(230_000, 1), _stream(30_000, 2)
    n = e["t"].size
    cuts = [(0, 0), (0, 1), (1, 1), (1, 100_001), (100_001, 100_001), (100_001, 100_002)]
    cuts += [(a, min(n, a + 7_777)) for a in range(100_002, n, 7_777)] + [(n, n)]
    info = {LI: (346, 260, "plumb_bob", [0.1, -0.2, 0.001, 0.002], [200, 0, 170, 0, 201, 130, 0, 0, 1], np.eye(3).ravel(),
                 [190, 0, 160, 0, 0, 190, 125, 0, 0, 0, 1, 0])}
    raw = rw.write_event_bag(tmp_path / "plain.bag", {L: e, R: r}, infos=info, msg_stamps={L: cuts}, msg_events=999,
                             chunk_threshold=threshold, conn_in_chunks=conn_in_chunks)
    return raw, e["t"]


def _run(args):
    p = subprocess.run(args, capture_output=True, text=True)
    assert p.returncode == 0, p.stdout + p.stderr
    return p


@pytest.mark.parametrize("threshold,conn_in_chunks", [(1, True), (1, False), (4096, True), (200_000, False), (1 << 30, True)])
def test_reader_equals_uncompressed(product_lib, tmp_path_factory, tmp_path, threshold, conn_in_chunks):
    exe = _compile(tmp_path_factory, "bag_dump")
    raw, t = _bag_corpus(tmp_path, threshold, conn_in_chunks)
    plain = tmp_path / "plain.bag"
    rng = np.random.default_rng(threshold)
    q = np.sort(np.concatenate([t[rng.integers(0, t.size, 50)], t[rng.integers(0, t.size, 50)] + 1, [t[0] - 1, t[-1], t[-1] + 1]]))
    (tmp_path / "q.bin").write_bytes(q.astype(np.int64).tobytes())

    def dumps(bag, pre):
        out = {}
        for mode, topic in (("events", L), ("events", R), ("take", L), ("calib", LI)):
            o = tmp_path / f"{mode}{topic.replace('/', '_')}.bin"
            args = [exe, *pre, mode, str(bag), topic] + ([str(tmp_path / "q.bin")] if mode == "take" else []) + [str(o)]
            _run(args)
            out[(mode, topic)] = o.read_bytes()
        return out

    want = dumps(plain, [])
    for codec in ("bz2", "lz4"):
        bag = tmp_path / f"{codec}.bag"
        bag.write_bytes(cb.recompress(raw, codec, bd=5, content_checksum=True))
        assert {c[1] for c in cb.chunks(bag.read_bytes())} == {codec}
        got = dumps(bag, ["--inflate-device", "0"])
        for k in want:
            assert got[k] == want[k], (codec, k)


# ---------------------------------------------------------------- the loop
@pytest.mark.parametrize("scene", ["dense", "mapping"])
def test_bag_system_on_compressed_bags(product_lib, tmp_path_factory, tmp_path, scene):
    """bag_system on bz2 and LZ4 versions of test_bag_system_equals_system_loop's scene bags gives the uncompressed bag's
    tick records, final map and trajectory file, byte for byte, with and without --hot-pixels 5."""
    import indep_system as isy
    import test_system_loop as tsl
    from esvo_b200 import configs
    exe = _compile(tmp_path_factory, "bag_system")
    s = tsl._stream(scene)
    t0, n = tsl._ticks(s)
    rr = configs.RIGS["hkust"]
    infos = {tp: (rr["width"], rr["height"], rr["model"], rr[sd]["D"], rr[sd]["K"], rr[sd]["R"], rr[sd]["P"]) for tp, sd in ((LI, "left"), (RI, "right"))}
    raw = rw.write_event_bag(tmp_path / "plain.bag", {L: s["left"], R: s["right"]}, infos=infos, msg_events=1500, chunk_threshold=64 * 1024)
    bags = {"none": tmp_path / "plain.bag"}
    for codec in ("bz2", "lz4"):
        bags[codec] = tmp_path / f"{codec}.bag"
        bags[codec].write_bytes(cb.recompress(raw, codec, independent=False, block_checksum=True))
    for hot in ([], ["--hot-pixels", "5"]):
        res = {}
        for codec, bag in bags.items():
            rb, tb = tmp_path / f"{codec}.bin", tmp_path / f"{codec}.txt"
            p = _run([exe, str(bag), L, R, LI, RI, str(rb), str(tb), "--t0-ns", str(t0), "--dt-ns", str(tsl.DT_NS), "--ticks", str(n), *hot])
            assert ("inflated" in p.stdout) == (codec != "none"), p.stdout
            res[codec] = (isy.parse_result(rb), tb.read_bytes())
        (a, ta) = res["none"]
        assert a[0].size == n and a[3] == 0 and len(ta) > 0
        for codec in ("bz2", "lz4"):
            b, tb = res[codec]
            for k in ("t", "status", "has_pose", "T"):
                assert a[0][k].tobytes() == b[0][k].tobytes(), (codec, hot, k)
            assert a[1].tobytes() == b[1].tobytes() and a[2].tobytes() == b[2].tobytes() and b[3] == 0, (codec, hot)
            assert ta == tb, (codec, hot)
