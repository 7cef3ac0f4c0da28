"""TEST INFRASTRUCTURE - CPU restatement of baseline JPEG decoding as PIL drives libjpeg-turbo.

The reference loads every frame with `np.asarray(PIL.Image.open(f).convert("RGB"))` (gtsfm/utils/io.py:39-72).  PIL decodes
through libjpeg-turbo with its defaults: the islow integer IDCT, fancy (triangle-filter) upsampling and the 16-bit fixed-point
YCbCr -> RGB tables.  This file restates that arithmetic in numpy for the subset of JPEG the device decoder accepts (baseline,
8-bit, Huffman, one interleaved scan, luma h1v1 / h2v1 / h1v2 / h2v2 with chroma 1x1, or grayscale, optional restart intervals)
and `tests/test_jpeg_cpu.py` pins it bit for bit against the installed PIL.

It also models the device's self-synchronising entropy decode (`sync_decode`): the unstuffed scan is cut into fixed-length
subsequences, each decoded from a guessed state until it crosses its end, then re-decoded from its predecessor's exit state
until no exit state changes.  That model must give the sequential decode's coefficients for any subsequence length."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np


class JpegUnsupported(ValueError):
    pass


# zig-zag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63], np.int64)


@dataclass
class Huffman:
    bits: List[int]  # counts of codes of length 1..16
    vals: List[int]
    lut: Dict[Tuple[int, int], int] = field(default_factory=dict)  # (length, code) -> symbol

    def __post_init__(self):
        code, k = 0, 0
        for length in range(1, 17):
            for _ in range(self.bits[length - 1]):
                self.lut[(length, code)] = self.vals[k]
                code += 1
                k += 1
            code <<= 1


@dataclass
class Component:
    cid: int
    h: int
    v: int
    tq: int
    td: int = 0
    ta: int = 0


@dataclass
class Header:
    height: int
    width: int
    comps: List[Component]
    qt: Dict[int, np.ndarray]  # natural order
    dc: Dict[int, Huffman]
    ac: Dict[int, Huffman]
    restart: int
    scan_offset: int  # first byte of the entropy-coded segment


def parse(data: bytes) -> Header:
    """Marker walk up to SOS with the device parser's acceptance rules."""
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise JpegUnsupported("not a JPEG file (no SOI marker)")
    p = 2
    qt, dc, ac = {}, {}, {}
    restart, frame, jfif, adobe = 0, None, False, None
    while True:
        while p < n and data[p] == 0xFF and p + 1 < n and data[p + 1] == 0xFF:
            p += 1
        if p + 4 > n or data[p] != 0xFF:
            raise JpegUnsupported("truncated or corrupt header")
        m = data[p + 1]
        seglen = (data[p + 2] << 8) | data[p + 3]
        if seglen < 2 or p + 2 + seglen > n:
            raise JpegUnsupported("truncated or corrupt header")
        seg = data[p + 4:p + 2 + seglen]
        p += 2 + seglen
        if m in (0xC0, 0xC1):
            if frame is not None or len(seg) < 6:
                raise JpegUnsupported("corrupt frame header")
            prec, hgt, wid, nc = seg[0], (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            if prec != 8:
                raise JpegUnsupported(f"{prec}-bit samples")
            if hgt == 0:
                raise JpegUnsupported("DNL (height defined after the first scan)")
            if wid == 0 or len(seg) < 6 + 3 * nc:
                raise JpegUnsupported("corrupt frame header")
            if nc not in (1, 3):
                raise JpegUnsupported(f"{nc} components (CMYK / YCCK)")
            comps = [Component(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nc)]
            frame = (hgt, wid, comps)
        elif m in (0xC2, 0xC6, 0xCA, 0xCE):
            raise JpegUnsupported("progressive JPEG")
        elif m in (0xC3, 0xC7, 0xCB, 0xCF):
            raise JpegUnsupported("lossless JPEG")
        elif m in (0xC5, 0xC9, 0xCD):
            raise JpegUnsupported("arithmetic coding" if m != 0xC5 else "hierarchical JPEG")
        elif m == 0xCC:
            raise JpegUnsupported("arithmetic coding")
        elif m == 0xC4:
            q = 0
            while q < len(seg):
                if q + 17 > len(seg):
                    raise JpegUnsupported("corrupt Huffman table")
                tc, th = seg[q] >> 4, seg[q] & 15
                bits = list(seg[q + 1:q + 17])
                cnt = sum(bits)
                if tc > 1 or th > 3 or cnt > 256 or q + 17 + cnt > len(seg):
                    raise JpegUnsupported("corrupt Huffman table")
                vals = list(seg[q + 17:q + 17 + cnt])
                _check_huffman(bits, vals, tc == 0)
                (dc if tc == 0 else ac)[th] = Huffman(bits, vals)
                q += 17 + cnt
        elif m == 0xDB:
            q = 0
            while q < len(seg):
                pq, tq = seg[q] >> 4, seg[q] & 15
                size = 64 * (pq + 1)
                if pq > 1 or tq > 3 or q + 1 + size > len(seg):
                    raise JpegUnsupported("corrupt quantisation table")
                raw = seg[q + 1:q + 1 + size]
                zz = np.frombuffer(raw, np.uint8).astype(np.int64) if pq == 0 else np.frombuffer(raw, ">u2").astype(np.int64)
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = zz
                qt[tq] = t
                q += 1 + size
        elif m == 0xDD:
            if len(seg) < 2:
                raise JpegUnsupported("corrupt restart interval")
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            jfif = jfif or (len(seg) >= 14 and seg[:5] == b"JFIF\0")  # libjpeg's examine_app0 needs 14 bytes
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif m == 0xDA:
            if frame is None:
                raise JpegUnsupported("scan before frame header")
            hgt, wid, comps = frame
            ns = seg[0] if seg else 0
            if len(seg) < 4 + 2 * ns:
                raise JpegUnsupported("corrupt scan header")
            if ns != len(comps):
                raise JpegUnsupported("multi-scan JPEG (a scan without every component)")
            for i in range(ns):
                if seg[1 + 2 * i] != comps[i].cid:
                    raise JpegUnsupported("scan component order differs from the frame")
                comps[i].td, comps[i].ta = seg[2 + 2 * i] >> 4, seg[2 + 2 * i] & 15
            ss, se, ahal = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or ahal != 0:
                raise JpegUnsupported("corrupt scan header (spectral selection in a sequential scan)")
            _check_colour(comps, jfif, adobe)
            _check_sampling(comps)
            for c in comps:
                if c.tq not in qt or c.td not in dc or c.ta not in ac:
                    raise JpegUnsupported("missing quantisation or Huffman table")
            if not _has_eoi(data, p):
                raise JpegUnsupported("truncated file (no EOI marker after the scan)")
            return Header(hgt, wid, comps, qt, dc, ac, restart, p)
        elif m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegUnsupported("corrupt header (unexpected marker)")
        # APPn, COM, DNL before the scan, anything else with a length: skipped


def _has_eoi(data: bytes, start: int) -> bool:
    return data.rfind(b"\xff\xd9", start) >= 0


def _check_huffman(bits, vals, is_dc):
    code = 0
    k = 0
    for length in range(1, 17):
        code += bits[length - 1]
        if code > (1 << length):
            raise JpegUnsupported("corrupt Huffman table")
        # an all-ones code would make the scan's end padding ambiguous; encoders never emit one (ITU T.81 Annex C)
        if code == (1 << length) and bits[length - 1]:
            raise JpegUnsupported("Huffman table with an all-ones code")
        code <<= 1
        k += bits[length - 1]
    if is_dc and any(v > 15 for v in vals):
        raise JpegUnsupported("corrupt Huffman table")


def _check_colour(comps, jfif, adobe):
    if len(comps) != 3:
        return
    if jfif:
        return
    if adobe is not None:
        if adobe == 0:
            raise JpegUnsupported("RGB colour space (Adobe transform 0)")
        return
    if [c.cid for c in comps] == [82, 71, 66]:
        raise JpegUnsupported("RGB colour space (component ids R, G, B)")


def _check_sampling(comps):
    if len(comps) == 1:
        if not (1 <= comps[0].h <= 4 and 1 <= comps[0].v <= 4):
            raise JpegUnsupported("corrupt sampling factors")
        return
    y = comps[0]
    if (y.h, y.v) not in ((1, 1), (2, 1), (1, 2), (2, 2)) or any((c.h, c.v) != (1, 1) for c in comps[1:]):
        raise JpegUnsupported("sampling factors " + ",".join(f"{c.h}x{c.v}" for c in comps))


def info(data: bytes) -> Tuple[int, int, int]:
    h = parse(data)
    return h.height, h.width, len(h.comps)


# ---- geometry ------------------------------------------------------------------------------------------------------------
@dataclass
class Geometry:
    mcux: int
    mcuy: int
    blocks: List[Tuple[int, int]]  # per component: (h, v) blocks per MCU
    bpm: int  # blocks per MCU
    comp_w: List[int]  # downsampled widths
    comp_h: List[int]


def geometry(hd: Header) -> Geometry:
    if len(hd.comps) == 1:
        return Geometry(-(-hd.width // 8), -(-hd.height // 8), [(1, 1)], 1, [hd.width], [hd.height])
    hm, vm = hd.comps[0].h, hd.comps[0].v
    blocks = [(c.h, c.v) for c in hd.comps]
    cw = [-(-hd.width * c.h // hm) for c in hd.comps]
    ch = [-(-hd.height * c.v // vm) for c in hd.comps]
    return Geometry(-(-hd.width // (8 * hm)), -(-hd.height // (8 * vm)), blocks, sum(h * v for h, v in blocks), cw, ch)


def unstuff(data: bytes, start: int) -> Tuple[bytes, List[int]]:
    """Entropy-coded segment -> (data bytes without stuffing or markers, start byte of every restart interval after the first)."""
    out = bytearray()
    rst = []
    p, n = start, len(data)
    while p < n:
        b = data[p]
        if b != 0xFF:
            out.append(b)
            p += 1
            continue
        nxt = data[p + 1] if p + 1 < n else None
        if nxt == 0x00:
            out.append(0xFF)
            p += 2
        elif nxt == 0xFF:
            p += 1
        elif nxt is not None and 0xD0 <= nxt <= 0xD7:
            if nxt != 0xD0 + (len(rst) & 7):
                raise JpegUnsupported("corrupt scan (restart marker out of sequence)")
            rst.append(len(out))
            p += 2
        else:
            break
    return bytes(out), rst


# ---- sequential entropy decode (libjpeg's decode_mcu, restated) ----------------------------------------------------------
class _Bits:
    def __init__(self, buf: bytes):
        self.bits = np.unpackbits(np.frombuffer(buf, np.uint8)).astype(np.int64) if buf else np.zeros(0, np.int64)
        n = len(self.bits)
        pad = np.concatenate([self.bits, np.zeros(32, np.int64)])
        peek = np.zeros(n + 1, np.int64)
        for k in range(16):
            peek = (peek << 1) | pad[k:k + n + 1]
        self.peek = peek.tolist()  # 16 bits starting at every bit position (zeros past the end)
        self.n = n


def _decode_huff(bits: _Bits, pos: int, tab: Huffman, end: int):
    """One Huffman symbol at `pos` -> (symbol, new pos) or None (invalid code or past `end`)."""
    w = bits.peek[pos] if pos <= bits.n else 0
    for length in range(1, 17):
        s = tab.lut.get((length, w >> (16 - length)))
        if s is not None:
            return (s, pos + length) if pos + length <= end else None
    return None


def _receive(bits: _Bits, pos: int, s: int, end: int):
    if s == 0:
        return 0, pos
    if pos + s > end:
        return None
    w = bits.peek[pos] >> (16 - s)
    v = w if w >= (1 << (s - 1)) else w - (1 << s) + 1  # HUFF_EXTEND
    return v, pos + s


def decode_coefficients(data: bytes, hd: Optional[Header] = None) -> Tuple[Header, List[np.ndarray]]:
    """Sequential decode -> per component int16 [blocks_y][blocks_x][64] quantised coefficients in natural order."""
    hd = hd or parse(data)
    g = geometry(hd)
    stream, rst = unstuff(data, hd.scan_offset)
    bits = _Bits(stream)
    n_mcu = g.mcux * g.mcuy
    ri = hd.restart or n_mcu
    n_seg = -(-n_mcu // ri)
    if len(rst) != n_seg - 1:
        raise JpegUnsupported("corrupt scan (restart marker count)")
    seg_start = [0] + [8 * r for r in rst] + [8 * len(stream)]
    coefs = [np.zeros((g.mcuy * v, g.mcux * h, 64), np.int64) for h, v in g.blocks]
    for s in range(n_seg):
        pos, end = seg_start[s], seg_start[s + 1]
        pred = [0] * len(hd.comps)
        for m in range(s * ri, min((s + 1) * ri, n_mcu)):
            my, mx = divmod(m, g.mcux)
            for ci, (h, v) in enumerate(g.blocks):
                c = hd.comps[ci]
                for by in range(v):
                    for bx in range(h):
                        blk = np.zeros(64, np.int64)
                        r = _decode_huff(bits, pos, hd.dc[c.td], end)
                        if r is None:
                            raise JpegUnsupported("corrupt scan (invalid Huffman code)")
                        t, pos = r
                        r = _receive(bits, pos, t, end)
                        if r is None:
                            raise JpegUnsupported("corrupt scan (truncated)")
                        d, pos = r
                        pred[ci] += d
                        blk[0] = pred[ci]
                        k = 1
                        while k < 64:
                            r = _decode_huff(bits, pos, hd.ac[c.ta], end)
                            if r is None:
                                raise JpegUnsupported("corrupt scan (invalid Huffman code)")
                            rs, pos = r
                            run, sz = rs >> 4, rs & 15
                            if sz:
                                k += run
                                if k > 63:
                                    raise JpegUnsupported("corrupt scan (coefficient index past 63)")
                                r = _receive(bits, pos, sz, end)
                                if r is None:
                                    raise JpegUnsupported("corrupt scan (truncated)")
                                val, pos = r
                                blk[ZIGZAG[k]] = val
                                k += 1
                            elif run == 15:
                                k += 16
                            else:
                                break
                        if k > 64:
                            raise JpegUnsupported("corrupt scan (coefficient index past 63)")
                        coefs[ci][my * v + by, mx * h + bx] = blk
        # what is left of the interval must be the byte-alignment padding: fewer than 8 one bits
        if end - pos >= 8 or any(bits.bits[pos:end] != 1):
            raise JpegUnsupported("corrupt scan (data after the last MCU of an interval)")
    return hd, [c.astype(np.int16) for c in coefs]


# ---- self-synchronising decode model ---------------------------------------------------------------------------------------
ERR = (-1, -1, -1)


def _f(bits: _Bits, hd: Header, g: Geometry, seg_start: List[int], state, sub_end: int, write=None):
    """Decode from `state` = (bit position, block within the MCU, zig-zag index: 0 = DC next) until the first symbol boundary
    at or past `sub_end`.  At the end of a restart interval (an MCU boundary followed by fewer than 8 one bits up to the
    interval's end) decoding continues from the next interval's start; a decode error restarts the guess there, or at the
    next bit in the last interval (only a confirmed decode, `write` given, reports it).  Returns (exit state, number of DC symbols decoded)."""
    comp_of_block = [ci for ci, (h, v) in enumerate(g.blocks) for _ in range(h * v)]
    pos, b, z = state
    if pos < 0:
        return ERR, 0
    count = 0
    pos = min(pos, seg_start[-1])
    seg = min(int(np.searchsorted(seg_start, pos, side="right")) - 1, len(seg_start) - 2)
    while True:
        end = seg_start[seg + 1]
        if b == 0 and z == 0 and end - pos < 8 and all(bits.bits[pos:end] == 1):
            if write is not None:
                write("done", seg)
            if seg + 2 >= len(seg_start):
                return (end, 0, 0), count
            seg += 1
            pos = seg_start[seg]
            if pos >= sub_end:
                return (pos, 0, 0), count
            continue
        if pos >= sub_end:
            return (pos, b, z), count
        c = hd.comps[comp_of_block[b]]
        ok = True
        if z == 0:
            r = _decode_huff(bits, pos, hd.dc[c.td], end)
            r = r and _receive(bits, r[1], r[0], end)
            if r:
                if write is not None:
                    write("dc", r[0])
                count += 1
                pos, z = r[1], 1
            else:
                ok = False
        else:
            r = _decode_huff(bits, pos, hd.ac[c.ta], end)
            if r:
                rs, pos2 = r
                run, sz = rs >> 4, rs & 15
                if sz:
                    k = z + run
                    r2 = _receive(bits, pos2, sz, end) if k <= 63 else None
                    if r2:
                        if write is not None:
                            write("ac", (k, r2[0]))
                        pos, z = r2[1], k + 1
                    else:
                        ok = False
                elif run == 15:
                    if z + 16 > 64:
                        ok = False
                    else:
                        pos, z = pos2, z + 16
                else:
                    pos, z = pos2, 64
            else:
                ok = False
        if not ok:
            if write is not None:
                write("error", None)
                return ERR, count
            # a wrong guess: guess again from the next interval, or from the next bit in the last one
            b, z = 0, 0
            if seg + 2 < len(seg_start):
                seg += 1
                pos = seg_start[seg]
            else:
                pos += 1
            if pos >= sub_end:
                return (pos, 0, 0), count
            continue
        if z == 64:
            z = 0
            b = (b + 1) % g.bpm


SYNC_SUB_BITS, SYNC_CHUNK, SYNC_ROUNDS = 1024, 256, 8  # csrc/jpeg.cu JPEG_SUB, JPEG_CHUNK, JPEG_ROUNDS


def sync_decode(data: bytes, sub_bits: int = SYNC_SUB_BITS, chunk: int = SYNC_CHUNK, max_rounds: int = SYNC_ROUNDS,
                stats: Optional[dict] = None) -> Tuple[List[np.ndarray], int]:
    """The device's parallel decode (csrc/jpeg.cu k_jpeg_sync_chunk, k_jpeg_sync_round, k_jpeg_sync_serial) run serially:
    returns (coefficients as decode_coefficients gives them, rounds: the first round that changed nothing, or max_rounds + 1
    when the serial chain finished the image).  Rounds read the exits the previous round left (the slowest interleaving the
    device allows).  `stats`, when given, receives the number of subsequence decodes of each phase."""
    hd = parse(data)
    g = geometry(hd)
    stream, rst = unstuff(data, hd.scan_offset)
    bits = _Bits(stream)
    n_mcu = g.mcux * g.mcuy
    ri = hd.restart or n_mcu
    n_seg = -(-n_mcu // ri)
    if len(rst) != n_seg - 1:
        raise JpegUnsupported("corrupt scan (restart marker count)")
    seg_start = [0] + [8 * r for r in rst] + [8 * len(stream)]
    total = 8 * len(stream)
    n_sub = max(1, -(-total // sub_bits))
    ends = [min((j + 1) * sub_bits, total) for j in range(n_sub)]
    stats = {} if stats is None else stats
    stats.update(chunk=0, rounds=0, serial=0)

    def walk(state, k, phase):
        stats[phase] += 1
        return _f(bits, hd, g, seg_start, state, ends[k])

    # chunk pass: threads in lock step, each stops once its path merges with the one started a subsequence later
    ex = [None] * n_sub
    for c0 in range(0, n_sub, chunk):
        c1 = min(c0 + chunk, n_sub)
        st = {t: ((c0 + t) * sub_bits, c0 + t) for t in range(c1 - c0)}  # thread -> (entry position or state, slot)
        active = {t: ((st[t][0], 0, 0), c0 + t, True) for t in st}
        while active:
            res = {t: (walk(state, k, "chunk"), ex[k]) for t, (state, k, _) in active.items()}
            nxt = {}
            for t in sorted(active, reverse=True):  # writes of one iteration go to distinct slots
                state, k, first = active[t]
                v, old = res[t]
                ex[k] = v
                merged = not first and old is not None and v[0] == old[0]
                if not merged and k + 1 < c1:
                    nxt[t] = (v[0], k + 1, False)
            active = nxt
    # rounds over chunks
    rounds = 0
    converged = False
    while rounds < max_rounds:
        rounds += 1
        prev = list(ex)
        changed = False
        for c0 in range(chunk, n_sub, chunk):
            e = prev[c0 - 1][0]
            for k in range(c0, min(c0 + chunk, n_sub)):
                v = walk(e, k, "rounds")
                old = ex[k]
                if v == old:
                    break
                ex[k], changed = v, True
                if v[0] == old[0]:
                    break
                e = v[0]
        if not changed:
            converged = True
            break
    if not converged:
        rounds = max_rounds + 1
        for k in range(1, n_sub):
            ex[k] = walk(ex[k - 1][0], k, "serial")
    # block bases: exclusive scan of DC counts
    base = np.concatenate([[0], np.cumsum([c for _, c in ex])])
    total_blocks = n_mcu * g.bpm
    flat = np.zeros((total_blocks, 64), np.int64)
    status = {"err": False}
    for j in range(n_sub):
        entry = (0, 0, 0) if j == 0 else ex[j - 1][0]
        # a block in progress at the entry was started by an earlier subsequence
        cur = {"blk": int(base[j]) - 1}  # the block being written: a block in progress at the entry is the previous one

        def write(kind, val, cur=cur):
            if kind == "dc":
                cur["blk"] += 1
                if cur["blk"] >= total_blocks:
                    status["err"] = True
                else:
                    flat[cur["blk"], 0] = val
            elif kind == "ac":
                k, v = val
                if 0 <= cur["blk"] < total_blocks:
                    flat[cur["blk"], ZIGZAG[k]] = v
            elif kind == "done":
                if cur["blk"] + 1 != min((val + 1) * ri, n_mcu) * g.bpm:
                    status["err"] = True
            elif kind == "error":
                status["err"] = True

        _f(bits, hd, g, seg_start, entry, ends[j], write)
    if status["err"] or base[-1] != total_blocks:
        raise JpegUnsupported("corrupt scan")
    # DC: per-component prefix sums that restart with every interval
    coefs = [np.zeros((g.mcuy * v, g.mcux * h, 64), np.int64) for h, v in g.blocks]
    pred = [0] * len(g.blocks)
    i = 0
    for m in range(n_mcu):
        if m % ri == 0:
            pred = [0] * len(g.blocks)
        my, mx = divmod(m, g.mcux)
        for ci, (h, v) in enumerate(g.blocks):
            for by in range(v):
                for bx in range(h):
                    pred[ci] += int(flat[i, 0])
                    blk = flat[i].copy()
                    blk[0] = pred[ci]
                    coefs[ci][my * v + by, mx * h + bx] = blk
                    i += 1
    return [c.astype(np.int16) for c in coefs], rounds


# ---- reconstruction -----------------------------------------------------------------------------------------------------
CONST_BITS, PASS1_BITS = 13, 2
F_0_298, F_0_390, F_0_541, F_0_765 = 2446, 3196, 4433, 6270
F_0_899, F_1_175, F_1_501, F_1_847 = 7373, 9633, 12299, 15137
F_1_961, F_2_053, F_2_562, F_3_072 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(s0, s1, s2, s3, s4, s5, s6, s7):
    """The LL&M islow butterfly on int64 arrays; returns the even/odd partial sums (tmp10..13, tmp0..3)."""
    z1 = (s2 + s6) * F_0_541
    tmp2 = z1 + s6 * (-F_1_847)
    tmp3 = z1 + s2 * F_0_765
    tmp0 = (s0 + s4) << CONST_BITS
    tmp1 = (s0 - s4) << CONST_BITS
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    o0, o1, o2, o3 = s7, s5, s3, s1
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F_1_175
    o0, o1, o2, o3 = o0 * F_0_298, o1 * F_2_053, o2 * F_3_072, o3 * F_1_501
    z1, z2, z3, z4 = z1 * (-F_0_899), z2 * (-F_2_562), z3 * (-F_1_961) + z5, z4 * (-F_0_390) + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    return (t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3)


def range_limit_idct(v: np.ndarray) -> np.ndarray:
    """libjpeg's post-IDCT range-limit table indexed with (v & 1023): v in [-128, 127] -> v + 128, above -> 255 up to 511,
    then 0 (the table wraps: 512..895 reads as negative)."""
    x = v & 1023
    out = np.where(x < 128, x + 128, np.where(x < 512, 255, np.where(x < 896, 0, x - 896)))
    return out.astype(np.uint8)


def idct_islow(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """[..., 64] quantised coefficients (natural order) x quant table -> [..., 8, 8] uint8 samples."""
    d = coef.astype(np.int64) * q.astype(np.int64)
    d = d.reshape(d.shape[:-1] + (8, 8))
    cols = _idct_1d(*[d[..., r, :] for r in range(8)])  # pass 1 on columns: each is [..., 8 (column)]
    ws = np.stack([_descale(c, CONST_BITS - PASS1_BITS) for c in cols], -2)  # [..., row, col]
    rows = _idct_1d(*[ws[..., :, c] for c in range(8)])  # pass 2 on rows
    out = np.stack([_descale(r, CONST_BITS + PASS1_BITS + 3) for r in rows], -1)
    return range_limit_idct(out)


def planes(hd: Header, coefs: List[np.ndarray]) -> List[np.ndarray]:
    """Component sample planes, cropped to each component's downsampled size."""
    g = geometry(hd)
    out = []
    for ci, c in enumerate(coefs):
        s = idct_islow(c, hd.qt[hd.comps[ci].tq])  # [by, bx, 8, 8]
        by, bx = s.shape[:2]
        p = s.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)
        out.append(p[:g.comp_h[ci], :g.comp_w[ci]])
    return out


def upsample(p: np.ndarray, fh: int, fv: int, width: int, height: int) -> np.ndarray:
    """libjpeg-turbo's fancy upsampling of one chroma plane by (fh, fv), edges replicated at the plane's size.  h2v1 and h2v2
    fall back to pixel replication when the plane is at most 2 samples wide."""
    x = p.astype(np.int64)
    if fh == 1 and fv == 1:
        return p
    h, w = x.shape
    if fv == 2:
        up, dn = x[np.maximum(np.arange(h) - 1, 0)], x[np.minimum(np.arange(h) + 1, h - 1)]
        if fh == 2 and w <= 2:
            r = np.repeat(np.repeat(x, 2, 0), 2, 1)
            return r[:height, :width].astype(np.uint8)
        s0, s1 = 3 * x + up, 3 * x + dn  # column sums of output rows 2y and 2y + 1
        if fh == 1:
            rows = np.stack([(s0 + 1) >> 2, (s1 + 2) >> 2], 1).reshape(2 * h, w)
            return rows[:height, :width].astype(np.uint8)
        out = []
        for s in (s0, s1):
            left, right = s[:, np.maximum(np.arange(w) - 1, 0)], s[:, np.minimum(np.arange(w) + 1, w - 1)]
            out.append(np.stack([(3 * s + left + 8) >> 4, (3 * s + right + 7) >> 4], 2).reshape(h, 2 * w))
        rows = np.stack(out, 1).reshape(2 * h, 2 * w)
        return rows[:height, :width].astype(np.uint8)
    # h2v1
    if w <= 2:
        return np.repeat(x, 2, 1)[:height, :width].astype(np.uint8)
    left, right = x[:, np.maximum(np.arange(w) - 1, 0)], x[:, np.minimum(np.arange(w) + 1, w - 1)]
    r = np.stack([(3 * x + left + 1) >> 2, (3 * x + right + 2) >> 2], 2).reshape(h, 2 * w)
    return r[:height, :width].astype(np.uint8)


SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)


def _fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def ycc_tables():
    """jdcolor.c build_ycc_rgb_table: (Cr->R, Cb->B, Cr->G, Cb->G) for input bytes 0..255."""
    x = np.arange(256, dtype=np.int64) - 128
    cr_r = (_fix(1.40200) * x + ONE_HALF) >> SCALEBITS
    cb_b = (_fix(1.77200) * x + ONE_HALF) >> SCALEBITS
    cr_g = -_fix(0.71414) * x
    cb_g = -_fix(0.34414) * x + ONE_HALF
    return cr_r, cb_b, cr_g, cb_g


def ycc_to_rgb(y: np.ndarray, cb: np.ndarray, cr: np.ndarray) -> np.ndarray:
    cr_r, cb_b, cr_g, cb_g = ycc_tables()
    yy = y.astype(np.int64)
    r = yy + cr_r[cr]
    g = yy + ((cb_g[cb] + cr_g[cr]) >> SCALEBITS)
    b = yy + cb_b[cb]
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def reconstruct(hd: Header, coefs: List[np.ndarray]) -> np.ndarray:
    pl = planes(hd, coefs)
    if len(pl) == 1:
        return np.repeat(pl[0][:, :, None], 3, 2)
    fh, fv = hd.comps[0].h, hd.comps[0].v
    cb = upsample(pl[1], fh, fv, hd.width, hd.height)
    cr = upsample(pl[2], fh, fv, hd.width, hd.height)
    return ycc_to_rgb(pl[0], cb, cr)


def decode(data: bytes) -> np.ndarray:
    """H x W x 3 uint8, equal to np.asarray(PIL.Image.open(f).convert("RGB")) for every file `parse` accepts."""
    hd, coefs = decode_coefficients(data)
    return reconstruct(hd, coefs)


# ---- test corpus -----------------------------------------------------------------------------------------------------------
CORPUS_SMALL_SIZES = [(1, 1), (8, 8), (15, 17), (16, 16), (37, 53)]  # (height, width)
MODES = {"444": 0, "422": 1, "420": 2}  # PIL's subsampling= values: h1v1, h2v1, h2v2 luma


def content(kind: str, height: int, width: int, seed: int = 0) -> np.ndarray:
    """Seeded RGB content: noise (long codes, many stuffed bytes), flat (EOB only), a gradient, or a synthetic.py frame."""
    rng = np.random.default_rng(seed + 7919 * height + width)
    if kind == "noise":
        return rng.integers(0, 256, (height, width, 3), dtype=np.uint8)
    if kind == "flat":
        return np.broadcast_to(np.array([200, 30, 90], np.uint8), (height, width, 3)).copy()
    if kind == "grad":
        y, x = np.meshgrid(np.linspace(0, 255, height), np.linspace(0, 255, width), indexing="ij")
        return np.stack([x, y, 255 - (x + y) / 2], -1).astype(np.uint8)
    if kind == "synthetic":
        from gtsfm_b200 import synthetic

        return np.ascontiguousarray(synthetic.synthetic_frame(seed, height, width))
    raise ValueError(kind)


def encode(rgb: np.ndarray, mode: str = "420", **kw) -> bytes:
    """PIL's encoder: mode '444' / '422' / '420' (YCbCr) or 'L' (gray from the red channel)."""
    import io

    from PIL import Image as PILImage

    buf = io.BytesIO()
    if mode == "L":
        PILImage.fromarray(np.ascontiguousarray(rgb[..., 0])).save(buf, "JPEG", **kw)
    else:
        PILImage.fromarray(rgb).save(buf, "JPEG", subsampling=MODES[mode], **kw)
    return buf.getvalue()


def corpus(large: bool = True):
    """(name, bytes) of the generated corpus: small sizes x contents x sampling x quality, the encoder options (optimised
    tables, restart intervals) at quality 75, and 517 x 389 / 1296 x 1936 frames."""
    out = []
    for h, w in CORPUS_SMALL_SIZES:
        for kind in ("noise", "flat", "grad"):
            rgb = content(kind, h, w)
            for mode in ("444", "422", "420", "L"):
                for q in (1, 50, 75, 95, 100):
                    out.append((f"{h}x{w}-{kind}-{mode}-q{q}", encode(rgb, mode, quality=q)))
                for opt in ({"optimize": True}, {"restart_marker_blocks": 1}, {"restart_marker_blocks": 3},
                            {"restart_marker_rows": 1}):
                    tag = "-".join(f"{k}{v}" for k, v in opt.items())
                    out.append((f"{h}x{w}-{kind}-{mode}-{tag}", encode(rgb, mode, quality=75, **opt)))
    for kind in ("noise", "synthetic"):
        rgb = content(kind, 517, 389)
        for mode in ("444", "422", "420", "L"):
            out.append((f"517x389-{kind}-{mode}-q90", encode(rgb, mode, quality=90)))
        out.append((f"517x389-{kind}-420-rmb3", encode(rgb, "420", quality=75, restart_marker_blocks=3)))
        out.append((f"517x389-{kind}-422-rmr1-opt", encode(rgb, "422", quality=95, restart_marker_rows=1, optimize=True)))
    if large:
        rgb = content("synthetic", 1936, 1296, seed=3)
        out.append(("1936x1296-synthetic-420-q90", encode(rgb, "420", quality=90)))
        out.append(("1936x1296-synthetic-444-q100-rmb1", encode(rgb, "444", quality=100, restart_marker_blocks=1)))
    return out


def unsupported_cases():
    """(name, bytes) that every parser of this project must refuse."""
    rgb = content("grad", 37, 53)
    out = [("progressive", encode(rgb, "420", quality=75, progressive=True))]
    import io

    from PIL import Image as PILImage

    buf = io.BytesIO()
    PILImage.fromarray(rgb).convert("CMYK").save(buf, "JPEG", quality=75)
    out.append(("cmyk", buf.getvalue()))
    good = encode(content("noise", 64, 48), "420", quality=90)
    for frac in (0.0, 0.01, 0.1, 0.5, 0.9):
        out.append((f"truncated-{frac}", good[:max(1, int(len(good) * frac))]))
    out.append(("truncated-eoi", good[:-2]))
    rng = np.random.default_rng(5)
    out.append(("random", rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()))
    out.append(("random-soi", b"\xff\xd8" + rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()))
    out.append(("empty", b""))
    return out
