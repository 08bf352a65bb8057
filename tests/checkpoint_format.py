"""An independent numpy reader of the checkpoint format of DESIGN.md ("Checkpoint format"): the header, the sections,
the zone table and the checksum, recomputed from the documented rule.  Test infrastructure only."""
import numpy as np

MAGIC = int.from_bytes(b"AMSWCKPT", "little")
HEADER = 128
HOLD, REMEDY, TRACK, DETAILS, TIMEOUTS = 0x1, 0x2, 0x4, 0x8, 0x10
COLUMNS = [("minute", "<u8"), ("hour", "<u8"), ("dom", "<u8"), ("month", "<u8"), ("dow", "<u8"), ("ras", "<i4"),
           ("flags", "<u4"), ("finished_at", "<i8"), ("runs_limit", "<i4"), ("reset_interval", "<i4"),
           ("success", "<i4"), ("failed", "<i4"), ("remedy_success", "<i4"), ("remedy_failed", "<i4"),
           ("remedy_total", "<i4"), ("remedy_finished_at", "<i8")]
HEADER_FIELDS = np.dtype([("magic", "<u8"), ("version", "<u4"), ("switches", "<u4"), ("bytes", "<u8"),
                          ("checksum", "<u8"), ("first_global", "<u8"), ("n", "<u8"), ("swept_end", "<u8"),
                          ("prev_tick", "<i8"), ("seed", "<u8"), ("n_zones", "<u4"), ("reserved32", "<u4"),
                          ("reserved", "<u8", (6,))])
assert HEADER_FIELDS.itemsize == HEADER
CHECKSUM_AT = HEADER_FIELDS.fields["checksum"][1]

G, M = np.uint64(0x9E3779B97F4A7C15), np.uint64(0xBF58476D1CE4E5B9)


def mix(key, v):
    """the checksum term of one item: x = (v ^ key * G) * M (mod 2^64), x ^ (x >> 31)"""
    with np.errstate(over="ignore"):
        x = (np.asarray(v, np.uint64) ^ (np.asarray(key, np.uint64) * G)) * M
    return x ^ (x >> np.uint64(31))


def _sum(terms):
    return int(np.sum(terms, dtype=np.uint64)) if np.size(terms) else 0


def sections(n, switches):
    """[(name, dtype or "bit", byte offset, bytes)] in blob order; the end of the last one"""
    out, at = [], HEADER
    def put(name, dt, nbytes):
        nonlocal at
        out.append((name, dt, at, nbytes))
        at += (nbytes + 7) // 8 * 8
    for name, dt in COLUMNS:
        put(name, dt, n * np.dtype(dt).itemsize)
    if switches & TIMEOUTS:
        put("wf_timeout", "<i4", n * 4)
        put("deadline", "<i8", n * 8)
    if switches & HOLD:
        put("since", "<i8", n * 8)
    if switches & TRACK:
        put("changed", "bit", (n + 31) // 32 * 4)
    if switches & DETAILS:
        put("det_applied", "<u1", n)
        put("det_start", "<i8", n * 8)
    return out, at


def checksum(blob, hd, secs, end):
    """the documented checksum of a blob: header words (its checksum word as 0), every element of every section (key =
    the element's bit offset, value = its bits zero-extended; one bit per slot in the bit section) and the zone table's
    words"""
    raw = np.frombuffer(blob, dtype=np.uint8)
    n = int(hd["n"])
    words = raw[:HEADER].view("<u8").copy()
    words[CHECKSUM_AT // 8] = 0
    s = _sum(mix(np.arange(0, HEADER, 8, dtype=np.uint64) * np.uint64(8), words))
    for name, dt, off, nbytes in secs:
        if dt == "bit":
            w = raw[off:off + (n + 31) // 32 * 4].view("<u4")
            bits = (w[np.arange(n) // 32] >> (np.arange(n, dtype=np.uint32) % 32)) & 1
            s += _sum(mix(np.uint64(off * 8) + np.arange(n, dtype=np.uint64), bits.astype(np.uint64)))
        else:
            size = np.dtype(dt).itemsize
            v = raw[off:off + n * size].view(dt)
            u = v.view({1: "<u1", 4: "<u4", 8: "<u8"}[size]).astype(np.uint64)
            s += _sum(mix((np.uint64(off) + np.arange(n, dtype=np.uint64) * np.uint64(size)) * np.uint64(8), u))
    zw = raw[end:int(hd["bytes"])].view("<u8")
    s += _sum(mix((np.uint64(end) + np.arange(len(zw), dtype=np.uint64) * np.uint64(8)) * np.uint64(8), zw))
    return s % (1 << 64)


def read(blob):
    """the blob as a dict: header fields, every section by name (numpy arrays; `changed` as bools), zones {id: name},
    and whether its checksum holds"""
    raw = np.frombuffer(blob, dtype=np.uint8)
    hd = raw[:HEADER].view(HEADER_FIELDS)[0]
    assert int(hd["magic"]) == MAGIC and int(hd["version"]) == 1
    n, sw = int(hd["n"]), int(hd["switches"])
    secs, end = sections(n, sw)
    out = {f: int(hd[f]) for f in ("switches", "bytes", "checksum", "first_global", "n", "swept_end", "prev_tick",
                                   "seed", "n_zones")}
    for name, dt, off, nbytes in secs:
        if dt == "bit":
            w = raw[off:off + nbytes].view("<u4")
            out[name] = ((w[np.arange(n) // 32] >> (np.arange(n, dtype=np.uint32) % 32)) & 1).astype(bool)
        else:
            out[name] = raw[off:off + n * np.dtype(dt).itemsize].view(dt).copy()
    zones, at = {}, end
    for _ in range(out["n_zones"]):
        zid, nl = (int(x) for x in raw[at:at + 8].view("<u4"))
        zones[zid] = bytes(raw[at + 8:at + 8 + nl]).decode()
        at += 8 + (nl + 7) // 8 * 8
    assert at == out["bytes"] == len(blob), (at, out["bytes"], len(blob))
    out["zones"] = zones
    out["checksum_ok"] = checksum(blob, hd, secs, end) == out["checksum"]
    return out


def reseal(blob):
    """a copy of `blob` (bytes-like) with its checksum recomputed: for tests that edit a blob on purpose"""
    b = bytearray(blob)
    raw = np.frombuffer(bytes(b), dtype=np.uint8)
    hd = raw[:HEADER].view(HEADER_FIELDS)[0]
    secs, end = sections(int(hd["n"]), int(hd["switches"]))
    b[CHECKSUM_AT:CHECKSUM_AT + 8] = checksum(bytes(b), hd, secs, end).to_bytes(8, "little")
    return bytes(b)
