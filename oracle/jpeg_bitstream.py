"""A small baseline JPEG parser  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Reads what the codec wrote (ITU T.81): the DQT, SOF0, DHT and SOS segments, then Huffman-decodes the scan into the
quantised coefficients of every block.  It pins the two halves of the round trip separately: the encoder's quantisation
tables and coefficients, and (through oracle/jpeg_oracle.decode) the decoder's pixels from those coefficients.
Sequential (SOF0) frames with 8-bit tables and no restart intervals only: what the JPEG test command's cv2.imencode
writes.  Only oracle/ and tests/ import this file.
"""
import numpy as np

from jpeg_oracle import ZIGZAG


class _Bits:
    """MSB-first bit reader over entropy-coded data, with the 0xFF00 byte stuffing removed."""

    def __init__(self, data):
        out = bytearray()
        i = 0
        while i < len(data):
            b = data[i]
            if b == 0xFF:
                nxt = data[i + 1]
                if nxt == 0x00:
                    out.append(0xFF)
                    i += 2
                    continue
                break  # a marker ends the scan
            out.append(b)
            i += 1
        self.bits = np.unpackbits(np.frombuffer(bytes(out), np.uint8)).tolist()
        self.pos = 0

    def bit(self):
        b = self.bits[self.pos]
        self.pos += 1
        return b

    def receive(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | self.bit()
        return v


def _extend(v, n):
    return v - (1 << n) + 1 if n and v < (1 << (n - 1)) else v


def _huffman(counts, symbols):
    """{(length, code): symbol} of a DHT table (ITU T.81 Annex C)."""
    table, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(counts[length - 1]):
            table[(length, code)] = symbols[k]
            code += 1
            k += 1
        code <<= 1
    return table


def _decode_symbol(bits, table):
    code = 0
    for length in range(1, 17):
        code = (code << 1) | bits.bit()
        if (length, code) in table:
            return table[(length, code)]
    raise ValueError("bad Huffman code")


def parse(data):
    """data: the bytes of a baseline JPEG.  Returns a dict:
    H, W: the frame size; components: [(id, h_samp, v_samp, table index)]; qt: {index: (64,) int64 natural order};
    coefs: [(rows, cols, 8, 8) int64 quantised coefficients per component, natural order], the coded blocks only (the
    MCU's dummy blocks at the right and bottom edges are dropped)."""
    data = bytes(data)
    assert data[:2] == b"\xff\xd8", "not a JPEG"
    i, qt, dc, ac, frame = 2, {}, {}, {}, None
    while True:
        while data[i] != 0xFF:
            i += 1
        marker = data[i + 1]
        i += 2
        if marker == 0xD9:
            break
        n = (data[i] << 8) | data[i + 1]
        seg = data[i + 2:i + n]
        if marker == 0xDB:  # DQT
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                assert pq == 0, "16-bit quantisation tables are not baseline"
                t = np.zeros(64, np.int64)
                t[ZIGZAG] = np.frombuffer(seg[j + 1:j + 65], np.uint8)
                qt[tq] = t
                j += 65
        elif marker == 0xC0:  # SOF0
            assert seg[0] == 8
            H, W, nc = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            comps = [(seg[6 + 3 * k], seg[7 + 3 * k] >> 4, seg[7 + 3 * k] & 15, seg[8 + 3 * k]) for k in range(nc)]
            frame = (H, W, comps)
        elif marker in (0xC1, 0xC2, 0xC3) or 0xC5 <= marker <= 0xCF and marker not in (0xC8, 0xCC):
            raise ValueError(f"frame type 0x{marker:02X} is not baseline")
        elif marker == 0xC4:  # DHT
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                counts = list(seg[j + 1:j + 17])
                syms = list(seg[j + 17:j + 17 + sum(counts)])
                (ac if tc else dc)[th] = _huffman(counts, syms)
                j += 17 + sum(counts)
        elif marker == 0xDD:
            raise ValueError("restart intervals are not supported")
        elif marker == 0xDA:  # SOS: the one scan of a baseline frame
            ns = seg[0]
            sel = [(seg[1 + 2 * k], seg[2 + 2 * k] >> 4, seg[2 + 2 * k] & 15) for k in range(ns)]
            coefs = _scan(data[i + n:], frame, sel, dc, ac)
            H, W, comps = frame
            return {"H": H, "W": W, "components": comps, "qt": qt, "coefs": coefs}
        i += n
    raise ValueError("no scan")


def _scan(data, frame, sel, dc, ac):
    H, W, comps = frame
    hmax, vmax = max(c[1] for c in comps), max(c[2] for c in comps)
    bits = _Bits(data)
    # coded blocks of each component (T.81 A.1.1) and the padded grid the interleaved MCUs cover
    dims = []
    for _, h, v, _ in comps:
        cw, ch = -(-W * h // hmax), -(-H * v // vmax)
        dims.append((-(-ch // 8), -(-cw // 8)))
    order = {c[0]: k for k, c in enumerate(comps)}
    scomps = [(order[cid], dc[td], ac[ta]) for cid, td, ta in sel]
    if len(scomps) == 1:  # non-interleaved: one block per MCU, coded blocks only
        k = scomps[0][0]
        grids = {k: np.zeros(dims[k] + (8, 8), np.int64)}
        mcus = [[(k, r, c)] for r in range(dims[k][0]) for c in range(dims[k][1])]
    else:
        mrows, mcols = -(-H // (8 * vmax)), -(-W // (8 * hmax))
        grids = {k: np.zeros((mrows * comps[k][2], mcols * comps[k][1], 8, 8), np.int64) for k, _, _ in scomps}
        mcus = [[(k, my * comps[k][2] + by, mx * comps[k][1] + bx) for k, _, _ in scomps
                 for by in range(comps[k][2]) for bx in range(comps[k][1])]
                for my in range(mrows) for mx in range(mcols)]
    tabs = {k: (d, a) for k, d, a in scomps}
    pred = {k: 0 for k in tabs}
    for mcu in mcus:
        for k, r, c in mcu:
            dtab, atab = tabs[k]
            zz = np.zeros(64, np.int64)
            s = _decode_symbol(bits, dtab)
            pred[k] += _extend(bits.receive(s), s)
            zz[0] = pred[k]
            j = 1
            while j < 64:
                rs = _decode_symbol(bits, atab)
                run, size = rs >> 4, rs & 15
                if size == 0:
                    if run == 15:
                        j += 16
                        continue
                    break  # EOB
                j += run
                zz[j] = _extend(bits.receive(size), size)
                j += 1
            blk = np.zeros(64, np.int64)
            blk[ZIGZAG] = zz
            grids[k][r, c] = blk.reshape(8, 8)
    return [grids[k][:dims[k][0], :dims[k][1]] for k in range(len(comps))]
