"""An independent numpy reader of the delta format of DESIGN.md ("Delta format"): the header, the offset section, the
sections over the changed slots, the zone table and the checksum, recomputed from the documented rule; and a delta
applied to the arrays of a full blob.  Full blobs are read with tests/checkpoint_format.py, here extended by the
waiting-second section of AM_CKPT_ADMISSION.  Test infrastructure only."""
import numpy as np

import checkpoint_format as fmt

MAGIC = int.from_bytes(b"AMSWCKDL", "little")
HEADER = fmt.HEADER
ADMISSION = 0x20
HEADER_FIELDS = np.dtype([("magic", "<u8"), ("version", "<u4"), ("switches", "<u4"), ("bytes", "<u8"),
                          ("checksum", "<u8"), ("first_global", "<u8"), ("n", "<u8"), ("swept_end", "<u8"),
                          ("prev_tick", "<i8"), ("seed", "<u8"), ("n_zones", "<u4"), ("reserved32", "<u4"),
                          ("n_changed", "<u8"), ("seq", "<u8"), ("parent_prev_tick", "<i8"),
                          ("parent_checksum", "<u8"), ("reserved", "<u8", (2,))])
assert HEADER_FIELDS.itemsize == HEADER
FIELDS = ("switches", "bytes", "checksum", "first_global", "n", "swept_end", "prev_tick", "seed", "n_zones")


def sections(n, switches, start=HEADER):
    """checkpoint_format.sections with the waiting second, from byte `start` on"""
    secs, end = fmt.sections(n, switches)
    secs = [(name, dt, off - HEADER + start, nbytes) for name, dt, off, nbytes in secs]
    end += start - HEADER
    if switches & ADMISSION:
        secs.append(("wait", "<i8", end, n * 8))
        end += n * 8
    return secs, end


def start_of(m):
    """the first section of a delta of m slots: after the header and the offset section"""
    return HEADER + (m * 4 + 7) // 8 * 8


def _elements(raw, secs, n):
    out, s = {}, 0
    for name, dt, off, nbytes in secs:
        if dt == "bit":
            w = raw[off:off + (n + 31) // 32 * 4].view("<u4")
            bits = (w[np.arange(n) // 32] >> (np.arange(n, dtype=np.uint32) % 32)) & 1
            s += fmt._sum(fmt.mix(np.uint64(off * 8) + np.arange(n, dtype=np.uint64), bits.astype(np.uint64)))
            out[name] = bits.astype(bool)
        else:
            size = np.dtype(dt).itemsize
            v = raw[off:off + n * size].view(dt)
            u = v.view({1: "<u1", 4: "<u4", 8: "<u8"}[size]).astype(np.uint64)
            s += fmt._sum(fmt.mix((np.uint64(off) + np.arange(n, dtype=np.uint64) * np.uint64(size)) * np.uint64(8), u))
            out[name] = v.copy()
    return out, s


def _header_and_zones(raw, end, hd, n_zones):
    words = raw[:HEADER].view("<u8").copy()
    words[fmt.CHECKSUM_AT // 8] = 0
    s = fmt._sum(fmt.mix(np.arange(0, HEADER, 8, dtype=np.uint64) * np.uint64(8), words))
    zones, at = {}, end
    for _ in range(n_zones):
        zid, nl = (int(x) for x in raw[at:at + 8].view("<u4"))
        zones[zid] = bytes(raw[at + 8:at + 8 + nl]).decode()
        at += 8 + (nl + 7) // 8 * 8
    zw = raw[end:at].view("<u8")
    s += fmt._sum(fmt.mix((np.uint64(end) + np.arange(len(zw), dtype=np.uint64) * np.uint64(8)) * np.uint64(8), zw))
    return zones, at, s


def read_full(blob):
    """a full blob as checkpoint_format.read returns it, for every switch (the waiting second included)"""
    raw = np.frombuffer(blob, dtype=np.uint8)
    hd = raw[:HEADER].view(fmt.HEADER_FIELDS)[0]
    assert int(hd["magic"]) == fmt.MAGIC and int(hd["version"]) == 1
    n, sw = int(hd["n"]), int(hd["switches"])
    secs, end = sections(n, sw)
    out = {f: int(hd[f]) for f in FIELDS}
    arrays, s = _elements(raw, secs, n)
    out.update(arrays)
    out["zones"], at, sz = _header_and_zones(raw, end, hd, out["n_zones"])
    assert at == out["bytes"] == len(blob), (at, out["bytes"], len(blob))
    out["checksum_ok"] = (s + sz) % (1 << 64) == out["checksum"]
    return out


def read(blob):
    """a delta as a dict: its header fields, `offsets` (slots relative to the range's first), every section over the
    changed slots by name (`changed` as bools), zones {id: name}, and whether its checksum holds"""
    raw = np.frombuffer(blob, dtype=np.uint8)
    hd = raw[:HEADER].view(HEADER_FIELDS)[0]
    assert int(hd["magic"]) == MAGIC and int(hd["version"]) == 1
    m, sw = int(hd["n_changed"]), int(hd["switches"])
    out = {f: int(hd[f]) for f in FIELDS + ("n_changed", "seq", "parent_prev_tick", "parent_checksum")}
    offs = raw[HEADER:HEADER + 4 * m].view("<u4").copy()
    s = fmt._sum(fmt.mix((np.uint64(HEADER) + np.arange(m, dtype=np.uint64) * np.uint64(4)) * np.uint64(8),
                         offs.astype(np.uint64)))
    secs, end = sections(m, sw, start_of(m))
    arrays, se = _elements(raw, secs, m)
    out.update(arrays)
    out["offsets"] = offs
    out["zones"], at, sz = _header_and_zones(raw, end, hd, out["n_zones"])
    assert at == out["bytes"] == len(blob), (at, out["bytes"], len(blob))
    out["checksum_ok"] = (s + se + sz) % (1 << 64) == out["checksum"]
    return out


def apply(full, delta):
    """the arrays and header fields of `full` (read_full of the previous link's state) with `delta` applied: its slots
    replaced, swept_end, P and the seed the delta's, the zone table that of the zones the records now use"""
    out = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in full.items()}
    for name, *_ in sections(0, full["switches"])[0]:
        out[name][delta["offsets"]] = delta[name]
    for k in ("swept_end", "prev_tick", "seed"):
        out[k] = delta[k]
    names = {**full["zones"], **delta["zones"]}
    f = out["flags"]
    used = np.unique((f >> np.uint32(24))[((f & np.uint32(7)) == 3) & ((f >> np.uint32(24)) != 0)])
    out["zones"] = {int(z): names[int(z)] for z in used}
    return out


def diff(a, b):
    """the slots (relative to the range's first) where any section element of two full reads differs"""
    d = np.zeros(a["n"], bool)
    for name, *_ in sections(0, a["switches"])[0]:
        d |= a[name] != b[name]
    return np.flatnonzero(d).astype(np.uint32)
