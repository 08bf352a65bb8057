"""An independent numpy reader of the packed format of DESIGN.md ("Packed format", version 2): a packed full blob or
delta decoded to the version-1 bytes it stands for, its directory, and the mode the documented rule picks for a block
(the smallest of the five, the first on a tie).  Version-1 layouts come from tests/checkpoint_delta_format.py.
Test infrastructure only."""
import numpy as np

import checkpoint_delta_format as dfmt
import checkpoint_format as fmt

VERSION = 2
BLOCK = 1024
RAW, CONST, FOR, SPARSE, DICT = range(5)
MODES = ("RAW", "CONST", "FOR", "SPARSE", "DICT")
ENTRY = np.dtype([("off", "<u8"), ("mode", "u1"), ("width", "u1"), ("aux", "<u2"), ("zero", "<u4")])
RAW_BYTES_AT = 14 * 8  # header word 14: the version-1 length
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
NONE = {"since": I64_MIN, "det_start": I64_MIN, "wait": I64_MIN, "deadline": I64_MAX}
SIGNED = {1: "i1", 4: "<i4", 8: "<i8"}


def sections(hd_words):
    """[(name, signed dtype, version-1 byte offset, elements)] a blob with these header words encodes, in order (a
    delta's offsets first, the change bits as u32 words); the end of the version-1 sections"""
    magic, sw = int(hd_words[0]), int(hd_words[1]) >> 32
    delta = magic == dfmt.MAGIC
    m = int(hd_words[10]) if delta else int(hd_words[5])
    secs, end = dfmt.sections(m, sw, dfmt.start_of(m) if delta else fmt.HEADER)
    out = [("offsets", "<i4", fmt.HEADER, m)] if delta else []
    for name, dt, off, nbytes in secs:
        if dt == "bit":
            out.append((name, "<i4", off, (m + 31) // 32))
        else:
            out.append((name, SIGNED[np.dtype(dt).itemsize], off, m))
    return out, end


def block_bytes(mode, w, aux, cnt, esize):
    words = lambda bits: (bits + 63) // 64 * 8
    if mode == RAW:
        return (cnt * esize + 7) // 8 * 8
    if mode == CONST:
        return 8
    if mode == FOR:
        return 8 + words(cnt * w)
    if mode == SPARSE:
        return words(cnt) + 8 + words(aux * w)
    return (aux * esize + 7) // 8 * 8 + words(cnt * w)


def code_bits(k):
    return 0 if k <= 1 else int(k - 1).bit_length()


def best_mode(v, none):
    """(mode, width, aux, bytes) the documented rule picks for the signed elements v"""
    esize, cnt = v.dtype.itemsize, len(v)
    x = [int(a) for a in (v.min(), v.max())]
    cands = [(RAW, 8 * esize, 0)]
    if x[0] == x[1]:
        cands.append((CONST, 0, 0))
    cands.append((FOR, (x[1] - x[0]).bit_length(), 0))
    p = v[v != none]
    cands.append((SPARSE, (int(p.max()) - int(p.min())).bit_length() if len(p) else 0, len(p)))
    k = len(np.unique(v))
    if k <= 256:
        cands.append((DICT, code_bits(k), k))
    best = None
    for mode, w, aux in cands:
        b = block_bytes(mode, w, aux, cnt, esize)
        if best is None or b < best[3]:
            best = (mode, w, aux, b)
    return best


def _fields(words, count, w):
    """fields 0..count-1 of width w packed from bit 0 of the u64 words"""
    if w == 0 or count == 0:
        return np.zeros(count, np.uint64)
    pos = np.arange(count, dtype=np.uint64) * np.uint64(w)
    q, sh = (pos >> np.uint64(6)).astype(np.int64), pos & np.uint64(63)
    lo = words[q] >> sh
    spill = sh + np.uint64(w) > np.uint64(64)
    nxt = words[np.minimum(q + 1, len(words) - 1)]
    hi = np.where(spill, nxt << ((np.uint64(64) - sh) & np.uint64(63)), np.uint64(0))
    mask = np.uint64((1 << w) - 1) if w < 64 else np.uint64(0xFFFFFFFFFFFFFFFF)
    return (lo | hi) & mask


def directory(blob):
    """the blob's blocks: [(section, first element, elements, entry as a dict)], and the payload's start"""
    raw = np.frombuffer(blob, np.uint8)
    words = raw[:fmt.HEADER].view("<u8")
    assert int(words[1]) & 0xFFFFFFFF == VERSION
    secs, _ = sections(words)
    out = []
    for name, dt, off, cnt in secs:
        for j0 in range(0, cnt, BLOCK):
            out.append((name, dt, j0, min(BLOCK, cnt - j0)))
    dire = raw[fmt.HEADER:fmt.HEADER + 16 * len(out)].view(ENTRY)
    return [(n, dt, j0, c, {k: int(dire[b][k]) for k in ENTRY.names}) for b, (n, dt, j0, c) in enumerate(out)], \
        fmt.HEADER + 16 * len(out)


def decode(blob):
    """the version-1 bytes a packed blob decodes to (asserting the directory's rules: canonical offsets, widths and
    sizes that fit each block, codes inside their dictionaries, as many present elements as SPARSE says)"""
    raw = np.frombuffer(blob, np.uint8)
    words = raw[:fmt.HEADER].view("<u8").copy()
    assert int(words[1]) & 0xFFFFFFFF == VERSION and int(words[2]) == len(blob) and len(blob) % 8 == 0
    raw_len = int(words[14])
    secs, end = sections(words)
    blocks, pay = directory(blob)
    out = bytearray(raw_len)
    hd = words.copy()
    hd[1] = (int(words[1]) & ~0xFFFFFFFF) | 1
    hd[2], hd[14] = raw_len, 0
    out[:fmt.HEADER] = hd.tobytes()
    at = 0
    offs = {name: off for name, dt, off, cnt in secs}
    for name, dt, j0, cnt, e in blocks:
        esize = np.dtype(dt).itemsize
        mode, w, aux = e["mode"], e["width"], e["aux"]
        assert e["zero"] == 0 and e["off"] == at, (name, j0, e, at)
        size = block_bytes(mode, w, aux, cnt, esize)
        at += size
        p = raw[pay + e["off"]:pay + e["off"] + size]
        assert len(p) == size
        pw = p.view("<u8")
        if mode == RAW:
            assert w == 8 * esize and aux == 0
            v = p[:cnt * esize].view(dt).astype(np.int64)
        elif mode == CONST:
            assert w == 0 and aux == 0
            v = np.full(cnt, pw[0].view(np.int64))
        elif mode == FOR:
            assert w <= 8 * esize and aux == 0
            v = (_fields(pw[1:], cnt, w) + pw[0]).view(np.int64)
        elif mode == SPARSE:
            assert w <= 8 * esize and aux <= cnt
            nbm = (cnt + 63) // 64
            bits = ((pw[:nbm][np.arange(cnt) // 64] >> (np.arange(cnt, dtype=np.uint64) % np.uint64(64))) & np.uint64(1)).astype(bool)
            assert bits.sum() == aux
            v = np.full(cnt, NONE.get(name, 0), np.int64)
            v[bits] = (_fields(pw[nbm + 1:], aux, w) + pw[nbm]).view(np.int64)
        else:
            assert mode == DICT and 1 <= aux <= min(256, cnt) and w == code_bits(aux)
            d = p[:aux * esize].view(dt).astype(np.int64)
            assert np.all(d[1:] > d[:-1]), (name, j0, e)
            c = _fields(pw[(aux * esize + 7) // 8:], cnt, w)
            assert np.all(c < aux)
            v = d[c.astype(np.int64)]
        o = offs[name] + j0 * esize
        out[o:o + cnt * esize] = v.astype(dt).tobytes()
    zones_at = pay + at
    out[end:] = raw[zones_at:].tobytes()
    assert end + (len(blob) - zones_at) == raw_len
    return bytes(out)


def bound(v1_len, blob):
    """the documented bound of a packed blob's length: the version-1 length plus the directory"""
    return v1_len + 16 * len(directory(blob)[0])
