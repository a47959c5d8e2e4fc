"""Compressed ROS bags for the inflater's tests, written from the format descriptions, not from the decoder:

- xxh32: xxHash32 (https://github.com/Cyan4973/xxHash/blob/dev/doc/xxhash_spec.md);
- an LZ4 frame writer (LZ4 frame format v1.6 and block format, lz4/doc/lz4_Frame_format.md and lz4_Block_format.md): greedy
  matching over a hash of 4-byte sequences, every FLG / BD option, uncompressed blocks, linked or independent blocks, and
  hand-built sequences (seq_block) for exact literal / match lengths and offsets;
- recompress(bag, codec): a bag written by tests/rosbag_writer.py with its chunk records re-encoded as bz2 or lz4 chunks
  (as rosbag record -j / --lz4 write them), the bag header's index_pos and the chunk infos' chunk_pos moved to match.
No chunk written by roslz4 itself is available here, so the LZ4 chunks come from this writer."""
import bz2
import struct

P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
M32 = 0xFFFFFFFF
LZ4_MAGIC = 0x184D2204


def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def xxh32(data, seed=0):
    data = bytes(data)
    n, i = len(data), 0
    if n >= 16:
        v = [(seed + P1 + P2) & M32, (seed + P2) & M32, seed, (seed - P1) & M32]
        words = struct.unpack_from("<%dI" % (n // 16 * 4), data)
        for k in range(0, len(words), 4):
            for j in range(4):
                v[j] = _rotl((v[j] + words[k + j] * P2) & M32, 13) * P1 & M32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M32
        i = n // 16 * 16
    else:
        h = (seed + P5) & M32
    h = (h + n) & M32
    while i + 4 <= n:
        h = _rotl((h + struct.unpack_from("<I", data, i)[0] * P3) & M32, 17) * P4 & M32
        i += 4
    while i < n:
        h = _rotl((h + data[i] * P5) & M32, 11) * P1 & M32
        i += 1
    h ^= h >> 15; h = h * P2 & M32; h ^= h >> 13; h = h * P3 & M32; h ^= h >> 16
    return h


def _length(n):   # the 255-continued extra length bytes after a nibble of 15
    out = bytearray()
    while n >= 255:
        out.append(255); n -= 255
    out.append(n)
    return out


def sequence(literals, offset=None, match_len=None):
    """One sequence: literals, then (unless offset is None: the last sequence) a match of match_len >= 4 bytes at offset."""
    lit = len(literals)
    ml = None if offset is None else match_len - 4
    tok = (min(lit, 15) << 4) | (0 if ml is None else min(ml, 15))
    out = bytearray([tok])
    if lit >= 15:
        out += _length(lit - 15)
    out += literals
    if ml is not None:
        out += struct.pack("<H", offset)
        if ml >= 15:
            out += _length(ml - 15)
    return bytes(out)


def seq_block(seqs, history=b""):
    """A block from [(literals, offset, match_len), ..., (last_literals,)] and the bytes it decodes to after history."""
    blk, out = bytearray(), bytearray(history)
    for s in seqs:
        blk += sequence(*s)
        out += s[0]
        if len(s) > 1:
            for _ in range(s[2]):
                out.append(out[-s[1]])
    return bytes(blk), bytes(out[len(history):])


def _match_len(buf, a, b, limit):
    m = 0
    while m + 64 <= limit and buf[a + m:a + m + 64] == buf[b + m:b + m + 64]:
        m += 64
    while m < limit and buf[a + m] == buf[b + m]:
        m += 1
    return m


def compress_block(buf, s, e, lo, table):
    """Greedy LZ4 block of buf[s:e]; matches may reach back to lo (the block's start, or earlier for linked blocks)."""
    out = bytearray()
    anchor = i = s
    last_match = e - 12          # the last match starts at least 12 bytes before the end, and ends 5 bytes before it
    miss = 0
    while i < last_match:
        key = bytes(buf[i:i + 4])
        c = table.get(key)
        table[key] = i
        if c is not None and c >= lo and 0 < i - c <= 65535:
            m = 4 + _match_len(buf, c + 4, i + 4, e - 5 - i - 4)
            out += sequence(bytes(buf[anchor:i]), i - c, m)
            i += m
            anchor = i
            miss = 0
        else:
            miss += 1
            i += 1 + (miss >> 6)
    out += sequence(bytes(buf[anchor:e]))
    return bytes(out)


def frame(data, bd=4, independent=True, block_checksum=False, content_size=False, content_checksum=False, store=None,
          blocks=None):
    """One LZ4 frame of data.  bd: block maximum size id 4..7 (64 KiB .. 4 MiB).  store: None = a block is written
    uncompressed when that is not larger, True = every block uncompressed, False = never.  blocks: raw blocks
    [(compressed, payload)] to write instead of compressing data (payload ignored when compressed is False)."""
    data = bytes(data)
    flg = 0x40 | (0x20 if independent else 0) | (0x10 if block_checksum else 0) | (8 if content_size else 0) | (4 if content_checksum else 0)
    desc = bytes([flg, bd << 4]) + (struct.pack("<Q", len(data)) if content_size else b"")
    out = bytearray(struct.pack("<I", LZ4_MAGIC) + desc + bytes([(xxh32(desc) >> 8) & 0xFF]))
    bmax = 1 << (8 + 2 * bd)

    def put(payload, raw):
        out.extend(struct.pack("<I", len(payload) | (0x80000000 if raw else 0)) + payload)
        if block_checksum:
            out.extend(struct.pack("<I", xxh32(payload)))

    if blocks is not None:
        for compressed, payload in blocks:
            put(payload, not compressed)
    else:
        table = {}
        for s in range(0, len(data), bmax):
            e = min(len(data), s + bmax)
            if independent:
                table = {}
            c = None if store else compress_block(data, s, e, s if independent else 0, table)
            if store or (store is None and len(c) >= e - s):
                put(data[s:e], True)
            else:
                put(c, False)
    out += struct.pack("<I", 0)
    if content_checksum:
        out += struct.pack("<I", xxh32(data))
    return bytes(out)


# ---------------------------------------------------------------- bags
def _records(b, o, end):
    while o < end:
        hl = struct.unpack_from("<I", b, o)[0]
        h = b[o + 4:o + 4 + hl]
        dl = struct.unpack_from("<I", b, o + 4 + hl)[0]
        yield o, h, b[o + 8 + hl:o + 8 + hl + dl]
        o += 8 + hl + dl


def _fields(h):
    f, o = {}, 0
    while o < len(h):
        n = struct.unpack_from("<I", h, o)[0]
        k, v = h[o + 4:o + 4 + n].split(b"=", 1)
        f[k.decode()] = v
        o += 4 + n
    return f


def _pack(f):
    out = b""
    for k, v in f.items():
        e = k.encode() + b"=" + v
        out += struct.pack("<I", len(e)) + e
    return out


def chunks(bag):
    """The chunk records of a bag: [(file offset, compression, size field, data)]."""
    out = []
    for o, h, d in _records(bag, 13, len(bag)):
        f = _fields(h)
        if f["op"] == b"\x05":
            out.append((o, f["compression"].decode(), struct.unpack("<I", f["size"])[0], d))
    return out


def recompress(bag, codec, level=9, **lz4):
    """bag (bytes of an uncompressed bag) with every chunk's data re-encoded as codec ("bz2" or "lz4": frame options)."""
    out = bytearray(bag[:13])
    moved, hdr_at, index_pos = {}, None, None
    for o, h, d in _records(bag, 13, len(bag)):
        f = _fields(h)
        op = f["op"]
        if op == b"\x03":
            hdr_at, index_pos = len(out), struct.unpack("<Q", f["index_pos"])[0]
        if op == b"\x05":
            assert f["compression"] == b"none"
            moved[o] = len(out)
            d = bz2.compress(d, level) if codec == "bz2" else frame(d, **lz4)
            f["compression"] = codec.encode()
            h = _pack(f)
        if op == b"\x06":
            f["chunk_pos"] = struct.pack("<Q", moved[struct.unpack("<Q", f["chunk_pos"])[0]])
            h = _pack(f)
        if o == index_pos:
            index_pos = len(out)
        out += struct.pack("<I", len(h)) + h + struct.pack("<I", len(d)) + d
    hl = struct.unpack_from("<I", out, hdr_at)[0]
    f = _fields(bytes(out[hdr_at + 4:hdr_at + 4 + hl]))
    f["index_pos"] = struct.pack("<Q", index_pos)
    h = _pack(f)
    assert len(h) == hl
    out[hdr_at + 4:hdr_at + 4 + hl] = h
    return bytes(out)
