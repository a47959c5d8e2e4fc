"""The chunk decoders (esvo_b200/csrc/inflate_core.h: the stage functions inflate.cu launches) run on the host by
tests/inflate_host_check.cpp, built twice: -O2, and -O1 with AddressSanitizer and UndefinedBehaviorSanitizer.  bz2 is held
byte for byte against Python's bz2 (libbz2), LZ4 against the frame writer of tests/compressed_bags.py.  Corrupted streams
(sanitizer build only) must be refused or decode to exactly what the reference decodes them to.  Also: without a GPU the
inflater and the inflating bag reader refuse cleanly.  CPU only."""
import bz2
import ctypes as C
import os
import re
import struct
import subprocess

import numpy as np
import pytest

import compressed_bags as cb
import rosbag_writer as rw
from conftest import has_gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "esvo_b200", "_build")
BZ2, LZ4 = 1, 2
L = "/davis/left/events"


def _reasons():
    """inflate_core.h's Reason enumerators by name."""
    src = open(os.path.join(ROOT, "esvo_b200", "csrc", "inflate_core.h")).read()
    body = src[src.index("enum Reason"):src.index("R_COUNT")]
    names = [w for w in re.findall(r"\b(R_OK|BZ_\w+|LZ4_\w+|R_\w+)\b", body)]
    out, k = {}, 0
    for n in names:
        if n == "R_FIRST_UNSUPPORTED":
            continue
        out[n] = k
        k += 1
    return out


R = _reasons()


def _build(tmp_path_factory, name, flags):
    exe = str(tmp_path_factory.mktemp("inflate") / name)
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", *flags, os.path.join(ROOT, "tests", "inflate_host_check.cpp"), "-o", exe])
    return exe


def _runner(exe):
    def run(items):
        """items: [(codec, src, dst_size)] -> [(reason, bytes or None)]"""
        fin, fout = exe + ".in", exe + ".out"
        with open(fin, "wb") as f:
            for codec, src, m in items:
                f.write(struct.pack("<IQQ", codec, len(src), m) + bytes(src))
        p = subprocess.run([exe, fin, fout], capture_output=True, text=True)
        assert p.returncode == 0 and not p.stderr, p.stdout + p.stderr
        raw, o, out = open(fout, "rb").read(), 0, []
        for _, _, m in items:
            r = struct.unpack_from("<i", raw, o)[0]; o += 4
            out.append((r, raw[o:o + m] if r == 0 else None))
            o += m if r == 0 else 0
        return out
    return run


@pytest.fixture(scope="module")
def fast(tmp_path_factory):
    return _runner(_build(tmp_path_factory, "ihc", ["-O2"]))


@pytest.fixture(scope="module")
def san(tmp_path_factory):
    return _runner(_build(tmp_path_factory, "ihc_san", ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all"]))


def bz2_inputs():
    """The bz2 corpus: edge sizes, runs around the initial-RLE lengths, RLE-heavy, incompressible, small and full
    alphabets, inputs across the 100 k / 900 k block limits."""
    rng = np.random.default_rng(11)
    out = {"empty": b"", "one": b"\x07"}
    for n in (3, 4, 5, 255, 256, 259):
        out[f"run{n}"] = b"x" * n
    out["runs_mixed"] = b"".join(bytes([k % 7]) * int(k % 300) for k in range(400))
    out["zeros2M"] = bytes(2_000_000)
    out["random"] = rng.integers(0, 256, 150_000, dtype=np.uint8).tobytes()
    out["one_symbol"] = b"\xaa" * 70_000
    out["two_symbols"] = rng.integers(0, 2, 120_000, dtype=np.uint8).tobytes()
    out["all_256"] = rng.permutation(np.repeat(np.arange(256, dtype=np.uint8), 300)).tobytes()
    out["periodic_256"] = bytes(range(256)) * 400
    text = (b"the quick brown fox jumps over the lazy dog %d\n" * 1)
    out["block_99999"] = b"".join(text % k for k in range(2400))[:99_999]
    out["block_100001"] = b"".join(text % k for k in range(2400))[:100_001]
    base = rng.integers(0, 40, 2_000_000, dtype=np.uint8).tobytes()
    out["block_899999"] = base[:899_999]
    out["block_900001"] = base[:900_001]
    return out


def _bag_chunks(tmp_path, codec="bz2"):
    rng = np.random.default_rng(3)
    n = 60_000
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(1_600_000_000 * 10**9 + np.cumsum(rng.integers(0, 3000, n))).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    raw = rw.write_event_bag(tmp_path / "b.bag", {L: e}, chunk_threshold=200_000, compression=codec)
    return [(d, size) for _, comp, size, d in cb.chunks(raw)]


def test_bz2_corpus_all_levels(fast, tmp_path):
    items, refs = [], []
    for name, data in bz2_inputs().items():
        for level in range(1, 10):
            items.append((BZ2, bz2.compress(data, level), len(data)))
            refs.append((name, level, data))
    for (name, level, data), (r, got) in zip(refs, fast(items)):
        assert r == 0 and got == data, (name, level, r)


def test_bz2_event_bag_chunks(fast, san, tmp_path):
    ch = _bag_chunks(tmp_path)
    assert len(ch) > 3
    items = [(BZ2, d, m) for d, m in ch]
    for run in (fast, san):
        for (d, m), (r, got) in zip(ch, run(items)):
            assert r == 0 and got == bz2.decompress(d) and len(got) == m


def _bz2_or_refused(cases, results, size):
    refused = 0
    for c, (r, got) in zip(cases, results):
        try:
            want = bz2.decompress(c)
        except (OSError, ValueError, EOFError):
            want = None
        if r != 0:
            refused += 1
            continue
        assert want is not None and got == want and len(want) == size
    return refused


def test_bz2_corruption_sanitized(san):
    rng = np.random.default_rng(5)
    for data in (bz2_inputs()["runs_mixed"], bz2_inputs()["two_symbols"][:30_000], bytes(range(256)) * 20):
        z = bz2.compress(data, 9)
        cuts = sorted(set(range(min(64, len(z)))) | set(range(max(0, len(z) - 64), len(z))) | set(rng.integers(0, len(z), 40).tolist()))
        cases = [z[:k] for k in cuts]
        for _ in range(300):
            b = bytearray(z)
            k = int(rng.integers(0, len(z) * 8))
            b[k // 8] ^= 0x80 >> (k % 8)
            cases.append(bytes(b))
        cases.append(z + b"\0")
        cases.append(z + z)
        refused = _bz2_or_refused(cases, san([(BZ2, c, len(data)) for c in cases]), len(data))
        assert refused >= len(cases) - 5


def test_bz2_wrong_size_refused(fast):
    z = bz2.compress(b"abc" * 1000)
    r = [r for r, _ in fast([(BZ2, z, 2999), (BZ2, z, 3001), (BZ2, z, 0)])]
    assert r[:2] == [R["BZ_SIZE"], R["BZ_SIZE"]] and 0 < r[2] < R["BZ_RANDOMISED"]   # 0 bytes: the block does not fit the work sizes


# ---------------------------------------------------------------- LZ4
def lz4_inputs():
    rng = np.random.default_rng(8)
    words = [bytes(rng.integers(97, 123, rng.integers(2, 9), dtype=np.uint8)) for _ in range(300)]
    text = b" ".join(words[i] for i in rng.integers(0, 300, 120_000))[:600_000]
    return {"empty": b"", "one": b"z", "short": b"abcdefgh" * 3, "text": text, "random": rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes(),
            "zeros": bytes(300_000), "periodic": bytes(range(13)) * 30_000}


FLAGS = [dict(independent=i, block_checksum=b, content_size=s, content_checksum=c)
         for i in (True, False) for b in (False, True) for s in (False, True) for c in (False, True)]


@pytest.mark.parametrize("bd", [4, 5, 6, 7])
def test_lz4_every_flag_and_block_size(fast, bd):
    items, refs = [], []
    for fl in FLAGS:
        for name, data in lz4_inputs().items():
            if name in ("random", "periodic") and bd > 4 and not fl["block_checksum"]:
                continue
            items.append((LZ4, cb.frame(data, bd=bd, **fl), len(data)))
            refs.append((name, fl, data))
    for (name, fl, data), (r, got) in zip(refs, fast(items)):
        assert r == 0 and got == data, (name, fl, r)


def lz4_sequence_frames():
    """Hand-built blocks: overlapping matches at offsets 1..31 (and 32, 64, 1000), literal and match lengths on the 15 and
    15 + 255 k boundaries, uncompressed blocks between compressed ones, and linked blocks whose matches reach back."""
    rng = np.random.default_rng(9)
    seqs = []
    for off in list(range(1, 32)) + [32, 64, 1000]:
        seqs.append((rng.integers(0, 256, max(off, 1), dtype=np.uint8).tobytes(), off, 4 + int(rng.integers(0, 300))))
    for lit in (0, 1, 14, 15, 16, 269, 270, 271, 524, 525, 526):
        seqs.append((rng.integers(0, 256, lit, dtype=np.uint8).tobytes(), 5, 4))
    for ml in (4, 18, 19, 20, 273, 274, 275, 528, 529, 530, 70_000):
        seqs.append((b"ab", 2, ml))
    seqs.append((rng.integers(0, 256, 7, dtype=np.uint8).tobytes(),))
    blk, out = cb.seq_block(seqs)
    frames = [(cb.frame(out, bd=7, blocks=[(True, blk)]), out)]
    # linked: the second block's first match reaches 10 bytes into the first block; an uncompressed block in between
    b1, o1 = cb.seq_block([(b"0123456789abcdef" * 4,)])
    raw = b"stored block!"
    b2, _ = cb.seq_block([(b"", 20, 40), (b"tail!",)], history=bytes(20))
    hist = bytearray(o1 + raw)
    for _ in range(40):
        hist.append(hist[-20])
    frames.append((cb.frame(b"", bd=4, independent=False, blocks=[(True, b1), (False, raw), (True, b2)]), bytes(hist) + b"tail!"))
    return frames


def test_lz4_hand_built_sequences(fast, san):
    fr = lz4_sequence_frames()
    for run in (fast, san):
        for (f, want), (r, got) in zip(fr, run([(LZ4, f, len(w)) for f, w in fr])):
            assert r == 0 and got == want


def test_lz4_refusals(fast):
    data = lz4_inputs()["text"][:100_000]
    good = cb.frame(data, bd=4, block_checksum=True, content_size=True, content_checksum=True)
    b2, _ = cb.seq_block([(b"", 20, 40), (b"tail!",)], history=bytes(20))
    cases = {
        "legacy": (struct.pack("<I", 0x184C2102) + b"\0" * 8, R["LZ4_LEGACY"]),
        "skippable": (struct.pack("<II", 0x184D2A53, 0), R["LZ4_SKIPPABLE"]),
        "dict": (struct.pack("<I", cb.LZ4_MAGIC) + bytes([0x41, 0x40, 0, 0, 0, 0, 0]), R["LZ4_DICT_ID"]),
        "content_size": (good, R["LZ4_SIZE"]),                                       # declared 100 001
        "content_checksum": (good[:-1] + bytes([good[-1] ^ 1]), R["LZ4_CONTENT_CHECKSUM"]),
        "independent_reach_back": (cb.frame(b"", bd=4, independent=True, blocks=[(True, cb.seq_block([(b"x" * 30,)])[0]), (True, b2)]), R["LZ4_OFFSET"]),
        "linked_reach_before_start": (cb.frame(b"", bd=4, independent=False, blocks=[(True, b2)]), R["LZ4_OFFSET"]),
        "trailing": (good + b"\0", R["LZ4_TRAILING"]),
        "truncated": (good[:-9], R["LZ4_TRUNCATED"]),
    }
    items = [(LZ4, f, 100_001 if k == "content_size" else (len(data) if f in (good, good + b"\0") or k in ("content_checksum", "truncated") else 75)) for k, (f, _) in cases.items()]
    got = fast(items)
    for (k, (_, want)), (r, _) in zip(cases.items(), got):
        assert r == want, (k, r)


def test_lz4_corruption_sanitized(san):
    """With a block or content checksum a corrupted frame is refused or decodes to the original; without one (a flipped
    literal is then undetectable by the format) it must still stay inside its buffers."""
    rng = np.random.default_rng(6)
    data = lz4_inputs()["text"][:150_000]
    for fl in (dict(content_checksum=True), dict(independent=False, content_checksum=True), dict(block_checksum=True, content_size=True),
               dict(), dict(independent=False)):
        f = cb.frame(data, bd=4, **fl)
        cases = [f[:k] for k in sorted(set(range(64)) | set(range(len(f) - 64, len(f))) | set(rng.integers(0, len(f), 30).tolist()))]
        for _ in range(300):
            b = bytearray(f)
            k = int(rng.integers(0, len(f) * 8))
            b[k // 8] ^= 0x80 >> (k % 8)
            cases.append(bytes(b))
        checked = fl.get("content_checksum") or fl.get("block_checksum")
        for r, got in san([(LZ4, c, len(data)) for c in cases]):
            assert r != 0 or not checked or got == data


# ---------------------------------------------------------------- no GPU: clean refusals
def test_inflater_without_gpu(product_lib, tmp_path_factory, tmp_path):
    if has_gpu():
        return
    f = product_lib.fn("inflater_create")
    f.argtypes = [C.c_int, C.c_size_t, C.POINTER(C.c_void_p)]
    h = C.c_void_p()
    assert f(0, 1 << 20, C.byref(h)) == -2 and not h.value
    exe = str(tmp_path_factory.mktemp("bin") / "bag_dump")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I" + os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "bag_dump.cpp"),
                           "-L" + BUILD, "-lesvo_b200", "-Wl,-rpath," + BUILD, "-o", exe])
    rng = np.random.default_rng(1)
    n = 3000
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(10**18 + np.arange(n) * 1000).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    plain = tmp_path / "plain.bag"
    raw = rw.write_event_bag(plain, {L: e}, chunk_threshold=5000)
    for codec in ("bz2", "lz4"):
        cbag = tmp_path / f"{codec}.bag"
        cbag.write_bytes(cb.recompress(raw, codec))
        p = subprocess.run([exe, "--inflate-device", "0", "events", str(cbag), L, str(tmp_path / "x.bin")], capture_output=True, text=True)
        assert p.returncode == 2 and "no CUDA device" in p.stdout, p.stdout + p.stderr
        p = subprocess.run([exe, "events", str(cbag), L, str(tmp_path / "x.bin")], capture_output=True, text=True)
        assert p.returncode == 3 and "rosbag decompress" in p.stdout
    outs = []
    for pre in ([], ["--inflate-device", "0"]):
        out = tmp_path / f"ev{len(pre)}.bin"
        p = subprocess.run([exe, *pre, "events", str(plain), L, str(out)], capture_output=True, text=True)
        assert p.returncode == 0, p.stdout + p.stderr
        outs.append(out.read_bytes())
    assert outs[0] == outs[1] and len(outs[0]) == 8 + 21 * n


def test_recompressed_bag_chunks_decode(fast, tmp_path):
    """The test bags' compressed chunk records hold exactly the uncompressed bag's chunk data."""
    rng = np.random.default_rng(2)
    n = 20_000
    e = dict(x=rng.integers(0, 346, n).astype(np.uint16), y=rng.integers(0, 260, n).astype(np.uint16),
             t=(10**18 + np.cumsum(rng.integers(0, 2000, n))).astype(np.int64), p=rng.integers(0, 2, n).astype(np.uint8))
    raw = rw.write_event_bag(tmp_path / "p.bag", {L: e}, chunk_threshold=50_000)
    want = [d for _, _, _, d in cb.chunks(raw)]
    for codec, code in (("bz2", BZ2), ("lz4", LZ4)):
        ch = cb.chunks(cb.recompress(raw, codec))
        assert [c[1] for c in ch] == [codec] * len(want) and [c[2] for c in ch] == [len(w) for w in want]
        got = fast([(code, d, m) for _, _, m, d in ch])
        assert [g for _, g in got] == want
