"""rb_build_agg's result restated: the reference adds each non-NULL value's low 32 bits to a CRoaring (v0.2.66) bitmap per group
(agg_fn_call.cpp:642-651, ExprValue::get_numberic<uint32_t>) and returns runOptimize() + the portable serialization
(ExprValue::get_string, expr_value.h:751-760).

- add(): values are grouped by their high 16 bits into containers, keys ascending.  A container is an ARRAY while it holds at most
  4096 values; the 4097th turns it into a BITSET.
- runOptimize(): with n maximal runs of consecutive low halves, an ARRAY becomes a RUN when 2 + 4n < 2 + 2 card (a tie stays ARRAY),
  a BITSET when 2 + 4n < 8192.
- portable write (little-endian): without a RUN container, cookie 12346, the container count, (key, card - 1) pairs, one uint32 offset
  per container (the first 8 + 8 size), the payloads.  With one: 12347 | (size - 1) << 16, a bitset of the RUN containers
  (ceil(size / 8) bytes), the pairs, the offsets only when size >= 4 (the first 4 + 8 size + ceil(size / 8)), the payloads.
  ARRAY: card uint16; BITSET: 1024 uint64 (value v is bit v % 64 of word v / 64); RUN: uint16 n, then n x (start, length - 1).

`parse` reads the bytes back and asserts the format's invariants, including that each container has the type the rules give."""
import struct

import numpy as np

COOKIE_NO_RUN, COOKIE = 12346, 12347
NO_OFFSET_THRESHOLD = 4
ARRAY, BITSET, RUN = "array", "bitset", "run"
EMPTY = struct.pack("<II", COOKIE_NO_RUN, 0)


def low32(values) -> np.ndarray:
    """get_numberic<uint32_t>: the low 32 bits of the integer (two's complement); BOOL is 0 / 1"""
    v = np.asarray(values)
    if v.dtype == np.uint64:
        return (v & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return (v.astype(np.int64) & 0xFFFFFFFF).astype(np.uint32)


def container_type(card: int, runs: int) -> str:
    if card <= 4096:
        return RUN if 2 + 4 * runs < 2 + 2 * card else ARRAY
    return RUN if 2 + 4 * runs < 8192 else BITSET


def _runs(lo: np.ndarray):
    """maximal runs of sorted distinct low halves: (starts, lengths)"""
    brk = np.flatnonzero(np.diff(lo.astype(np.int64)) != 1) + 1
    s = np.concatenate([[0], brk])
    e = np.concatenate([brk, [len(lo)]])
    return lo[s].astype(np.int64), (e - s).astype(np.int64)


def serialize(values) -> bytes:
    """the bytes of a bitmap built by add() of every value (uint32), after runOptimize()"""
    u = np.unique(np.asarray(values, dtype=np.uint64)).astype(np.uint64)
    if len(u) and int(u[-1]) > 0xFFFFFFFF:
        raise ValueError("values must be uint32")
    if len(u) == 0:
        return EMPTY
    hi, lo = (u >> np.uint64(16)).astype(np.int64), (u & np.uint64(0xFFFF)).astype(np.uint16)
    keys, starts = np.unique(hi, return_index=True)
    ends = np.concatenate([starts[1:], [len(u)]])
    conts = []
    for k, s, e in zip(keys.tolist(), starts.tolist(), ends.tolist()):
        l = lo[s:e]
        rs, rl = _runs(l)
        t = container_type(len(l), len(rs))
        if t == ARRAY:
            payload = l.astype("<u2").tobytes()
        elif t == RUN:
            payload = struct.pack("<H", len(rs)) + np.stack([rs, rl - 1], axis=1).astype("<u2").tobytes()
        else:
            words = np.zeros(1024, dtype="<u8")
            np.bitwise_or.at(words, (l >> 6).astype(np.int64), np.left_shift(np.uint64(1), (l & 63).astype(np.uint64)))
            payload = words.tobytes()
        conts.append((k, len(l), t, payload))
    size = len(conts)
    has_run = any(c[2] == RUN for c in conts)
    out = bytearray()
    if has_run:
        out += struct.pack("<I", COOKIE | ((size - 1) << 16))
        bits = bytearray((size + 7) // 8)
        for i, c in enumerate(conts):
            if c[2] == RUN:
                bits[i // 8] |= 1 << (i % 8)
        out += bits
        start = 4 + 8 * size + len(bits)
    else:
        out += struct.pack("<II", COOKIE_NO_RUN, size)
        start = 8 + 8 * size
    for k, card, _, _ in conts:
        out += struct.pack("<HH", k, card - 1)
    if not has_run or size >= NO_OFFSET_THRESHOLD:
        for c in conts:
            out += struct.pack("<I", start)
            start += len(c[3])
    for c in conts:
        out += c[3]
    return bytes(out)


def parse(b: bytes) -> np.ndarray:
    """the sorted uint32 values of a serialized bitmap; asserts keys ascending, cards and offsets consistent, runs disjoint and maximal,
    every byte accounted for, and each container's type the one add() + runOptimize() give its values"""
    (cookie,) = struct.unpack_from("<I", b, 0)
    if cookie & 0xFFFF == COOKIE:
        size = (cookie >> 16) + 1
        nb = (size + 7) // 8
        run_bits = b[4:4 + nb]
        pos = 4 + nb
        is_run = [bool((run_bits[i // 8] >> (i % 8)) & 1) for i in range(size)]
        assert not any((run_bits[-1] >> j) & 1 for j in range(size - 8 * (nb - 1), 8)), "run bitset bits past the last container"
        assert any(is_run), "cookie 12347 without a RUN container"
        has_off = size >= NO_OFFSET_THRESHOLD
    else:
        assert cookie == COOKIE_NO_RUN, hex(cookie)
        (size,) = struct.unpack_from("<I", b, 4)
        pos = 8
        is_run = [False] * size
        has_off = True
    pairs = [struct.unpack_from("<HH", b, pos + 4 * i) for i in range(size)]
    pos += 4 * size
    keys = [k for k, _ in pairs]
    assert keys == sorted(set(keys)), "container keys not strictly ascending"
    offs = None
    if has_off:
        offs = list(struct.unpack_from(f"<{size}I", b, pos))
        pos += 4 * size
    out = []
    for i, (k, c1) in enumerate(pairs):
        card = c1 + 1
        if offs is not None:
            assert offs[i] == pos, ("offset", i, offs[i], pos)
        if is_run[i]:
            (n,) = struct.unpack_from("<H", b, pos)
            rr = np.frombuffer(b, dtype="<u2", count=2 * n, offset=pos + 2).reshape(n, 2).astype(np.int64)
            pos += 2 + 4 * n
            starts, lens = rr[:, 0], rr[:, 1] + 1
            assert n >= 1 and (starts + lens <= 65536).all()
            assert (starts[1:] > starts[:-1] + lens[:-1]).all(), "runs overlap, touch or are unsorted"
            lo = np.concatenate([np.arange(s, s + l) for s, l in zip(starts, lens)])
            t = RUN
        else:
            stored_type = BITSET if card > 4096 else ARRAY
            if stored_type == ARRAY:
                lo = np.frombuffer(b, dtype="<u2", count=card, offset=pos).astype(np.int64)
                pos += 2 * card
                assert (np.diff(lo) > 0).all(), "array values not strictly ascending"
            else:
                words = np.frombuffer(b, dtype="<u8", count=1024, offset=pos)
                pos += 8192
                lo = np.flatnonzero(np.unpackbits(words.view(np.uint8), bitorder="little")).astype(np.int64)
            t = stored_type
        assert len(lo) == card, ("card", i, len(lo), card)
        assert t == container_type(card, len(_runs(lo)[0])), ("container type", i, t, card, len(_runs(lo)[0]))
        out.append((np.int64(k) << 16) | lo)
    assert pos == len(b), ("trailing or missing bytes", pos, len(b))
    return np.concatenate(out).astype(np.uint32) if out else np.zeros(0, np.uint32)


def bitmaps(values, keys=None, n_groups: int = 1, valid=None) -> list:
    """per group 0 .. n_groups - 1: rb_build_agg over the group's non-NULL values (a group without one: the empty bitmap)"""
    v = low32(values).astype(np.uint64)
    g = np.zeros(len(v), np.int64) if keys is None else np.asarray(keys, np.int64)
    if valid is not None:
        keep = np.asarray(valid, bool)
        v, g = v[keep], g[keep]
    pk = np.unique((g.astype(np.uint64) << np.uint64(32)) | v)
    gs = (pk >> np.uint64(32)).astype(np.int64)
    cut = np.searchsorted(gs, np.arange(n_groups + 1))
    lo = pk & np.uint64(0xFFFFFFFF)
    return [serialize(lo[cut[i]:cut[i + 1]]) for i in range(n_groups)]
