"""A small deterministic baseline JPEG writer for test fixtures: coefficient planes in, file bytes out.

It writes what an encoder is allowed to write but photos and common libraries never do -- 16-bit quantisers, Huffman
codes up to 16 bits long, magnitude categories up to 15 (12 and above only to make files a decoder must refuse) -- so
that the coder can be held to the reference at its numeric limits.  Supported: 1 or 3 components, any sampling factors
(4:4:4, 4:2:2, 4:2:0), one sequential scan (interleaved when there are several components), DRI restart intervals, 8- or
16-bit DQT tables.

Coefficients are given per component as an int array of shape (blocks down, blocks across, 64) in zig-zag order,
covering the whole MCU grid; DC values are absolute (the writer codes the differences).
"""
import struct

# zig-zag index -> raster index inside the 8x8 block
ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
          28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54,
          47, 55, 62, 63]

DC_SYMBOLS = list(range(16))                                                        # magnitude categories 0..15
AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]  # EOB, ZRL, run/size


class BitWriter:
    """MSB-first entropy-coded segment writer with 0xFF byte stuffing."""

    def __init__(self):
        self.out = bytearray()
        self.acc = 0
        self.n = 0

    def put(self, v, n):
        if n == 0:
            return
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.n += n
        while self.n >= 8:
            b = (self.acc >> (self.n - 8)) & 255
            self.out.append(b)
            if b == 255:
                self.out.append(0)
            self.n -= 8
        self.acc &= (1 << self.n) - 1

    def pad(self, bit=1):
        """Fill the last byte with `bit` (1 is what libjpeg and the reference expect before a marker)."""
        while self.n & 7:
            self.put(bit, 1)


def canonical_codes(bits, vals):
    """DHT counts per code length (bits[0] = number of 1-bit codes) + symbols -> {symbol: (code, length)}."""
    enc, code, k = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            enc[vals[k]] = (code, ln)
            k += 1
            code += 1
        code <<= 1
    return enc


def fit_lengths(desired):
    """[(symbol, wanted code length)] -> [(symbol, length)] that form a valid table: lengths are only ever raised, as
    little as the Kraft budget of the symbols that follow needs, and the all-ones code stays unused."""
    out = []
    budget = (1 << 16) - 1                              # in units of 2^-16; one unit left for the all-ones code
    for i, (sym, ln) in enumerate(desired):
        ln = max(1, min(16, ln))
        left = len(desired) - i - 1
        while (1 << (16 - ln)) > budget - left:
            ln += 1
        assert ln <= 16, "too many symbols for a 16-bit code space"
        budget -= 1 << (16 - ln)
        out.append((sym, ln))
    return out


class HuffTable:
    """A DHT table built from code lengths: `lengths` is [(symbol, length)], lengths 1..16 (canonical codes assigned in
    order of length, then in the order given)."""

    def __init__(self, lengths):
        lengths = sorted(lengths, key=lambda sl: sl[1])
        self.bits = [0] * 16
        for _, ln in lengths:
            assert 1 <= ln <= 16
            self.bits[ln - 1] += 1
        self.vals = [s for s, _ in lengths]
        assert sum((1 << (16 - ln)) for _, ln in lengths) < (1 << 16), "code lengths exceed the code space"
        self.enc = canonical_codes(self.bits, self.vals)

    def segment_body(self, tc, th):
        return bytes([(tc << 4) | th] + self.bits + self.vals)


def uniform_table(symbols, length):
    return HuffTable(fit_lengths([(s, length) for s in symbols]))


def put_block(bw, z, pred, dc, ac):
    """Huffman-codes one block (64 values in zig-zag order, absolute DC) after DC predictor `pred` with the code maps `dc`
    and `ac` ({symbol: (code, length)}); -> the new predictor."""
    z = [int(v) for v in z]
    d = z[0] - pred
    s = abs(d).bit_length()
    bw.put(*dc[s])
    bw.put(d if d > 0 else d - 1 + (1 << s), s)
    end = 63
    while end > 0 and z[end] == 0:
        end -= 1
    run = 0
    for k in range(1, end + 1):
        if z[k] == 0:
            run += 1
            continue
        while run >= 16:
            bw.put(*ac[0xF0])
            run -= 16
        s = abs(z[k]).bit_length()
        bw.put(*ac[(run << 4) | s])
        bw.put(z[k] if z[k] > 0 else z[k] - 1 + (1 << s), s)
        run = 0
    if end != 63:
        bw.put(*ac[0x00])
    return z[0]


def dqt_segment(qtables, qbits):
    body = bytearray()
    for t, q in enumerate(qtables):
        assert len(q) == 64 and all(1 <= v < (1 << qbits) for v in q)
        body.append(((1 if qbits == 16 else 0) << 4) | t)
        body += b"".join(struct.pack(">H" if qbits == 16 else ">B", int(v)) for v in q)
    return b"\xff\xdb" + struct.pack(">H", 2 + len(body)) + bytes(body)


def geometry(width, height, sampling):
    """-> (mcuh, mcuv, [(blocks across, blocks down) of the MCU grid per component], [(coded blocks across, down)])"""
    hmax = max(h for h, _ in sampling)
    vmax = max(v for _, v in sampling)
    mcuh = -(-width // (8 * hmax))
    mcuv = -(-height // (8 * vmax))
    grid = [(mcuh * h, mcuv * v) for h, v in sampling]
    coded = [(-(-(-(-width * h // hmax)) // 8), -(-(-(-height * v // vmax)) // 8)) for h, v in sampling]
    return mcuh, mcuv, grid, coded


def write_baseline(planes, width, height, sampling, qtables, qbits=8, dc_tables=None, ac_tables=None, restart=0,
                   extra_markers=b"", padbit=1):
    """planes[c]: int array (mcuv * V, mcuh * H, 64), zig-zag order.  qtables: one 64-entry table (zig-zag order) per
    component or one for all; dc_tables / ac_tables: HuffTable for luma and for chroma (one table serves all components when
    only one is given).  restart: DRI interval in MCUs (0 = none).  padbit: the bit that fills the last byte of every
    restart interval, or a list of them, one per interval.  Returns the file bytes."""
    ncmp = len(planes)
    assert ncmp in (1, 3) and len(sampling) == ncmp
    dc_tables = dc_tables or [uniform_table(DC_SYMBOLS[:12], 5)]
    ac_tables = ac_tables or [uniform_table(AC_SYMBOLS, 8)]
    mcuh, mcuv, grid, coded = geometry(width, height, sampling)
    for c in range(ncmp):
        assert planes[c].shape == (grid[c][1], grid[c][0], 64), (c, planes[c].shape, grid[c])
    qidx = [min(c, len(qtables) - 1) for c in range(ncmp)]
    tidx = [min(1 if c else 0, len(dc_tables) - 1) for c in range(ncmp)]
    aidx = [min(1 if c else 0, len(ac_tables) - 1) for c in range(ncmp)]
    o = bytearray(b"\xff\xd8")
    o += b"\xff\xe0" + struct.pack(">H", 16) + b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    o += dqt_segment(qtables, qbits)
    o += b"\xff\xc0" + struct.pack(">HBHHB", 8 + 3 * ncmp, 8, height, width, ncmp)
    for c in range(ncmp):
        o += bytes([c + 1, (sampling[c][0] << 4) | sampling[c][1], qidx[c]])
    for tc, tabs in ((0, dc_tables), (1, ac_tables)):
        for th, t in enumerate(tabs):
            body = t.segment_body(tc, th)
            o += b"\xff\xc4" + struct.pack(">H", 2 + len(body)) + body
    if restart:
        o += b"\xff\xdd" + struct.pack(">HH", 4, restart)
    o += extra_markers
    o += b"\xff\xda" + struct.pack(">HB", 6 + 2 * ncmp, ncmp)
    for c in range(ncmp):
        o += bytes([c + 1, (tidx[c] << 4) | aidx[c]])
    o += bytes([0, 63, 0])
    if ncmp == 1:                      # a one-component scan is not interleaved: only the coded blocks, one per MCU
        units = [[(0, by, bx)] for by in range(coded[0][1]) for bx in range(coded[0][0])]
    else:
        units = [[(c, my * sampling[c][1] + v, mx * sampling[c][0] + h)
                  for c in range(ncmp) for v in range(sampling[c][1]) for h in range(sampling[c][0])]
                 for my in range(mcuv) for mx in range(mcuh)]
    bw = BitWriter()
    pred = [0] * ncmp
    pads = [padbit] * (len(units) + 1) if isinstance(padbit, int) else list(padbit)
    for i, unit in enumerate(units):
        if restart and i and i % restart == 0:
            bw.pad(pads[i // restart - 1])
            bw.out += bytes([0xFF, 0xD0 + ((i // restart - 1) & 7)])
            pred = [0] * ncmp
        for c, by, bx in unit:
            pred[c] = put_block(bw, planes[c][by, bx], pred[c], dc_tables[tidx[c]].enc, ac_tables[aidx[c]].enc)
    bw.pad(pads[(len(units) - 1) // restart if restart else 0])
    o += bw.out + b"\xff\xd9"
    return bytes(o)

