"""JPEG files written by oracle.jpeg_ref with every writer knob, shared by test_oracle_jpeg.py (PIL equals the numpy back end)
and test_gpu_jpeg_bitstreams.py (the GPU decoder equals both).  Each case is (name, jpeg_ref.Written)."""
import io

import numpy as np

from oracle import jpeg_ref as J

Q75 = [J.quality_table(J.STD_Q_LUMA, 75), J.quality_table(J.STD_Q_CHROMA, 75)]


def photo(h, w, seed):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    f = rng.uniform(0.02, 0.2, 3)
    base = np.stack([127.5 + 110 * np.sin(f[c] * (xx + rng.uniform(0, 1) * yy) + rng.uniform(0, 6)) for c in range(3)], -1)
    return np.clip(base + rng.normal(0, 20, base.shape), 0, 255).astype(np.uint8)


def content(layout, h=37, w=53, seed=0, qt=Q75):
    """Conforming coefficients of a photo-like image: (coefs, sampling)."""
    return J.pixels_to_coefs(photo(h, w, seed), layout, qt)


def write(layout, h=37, w=53, seed=0, qt=Q75, **kw):
    coefs, samp = content(layout, h, w, seed, qt)
    kw.setdefault("sampling", samp)
    return J.write_jpeg(coefs, {0: qt[0]} if layout == "gray" else {0: qt[0], 1: qt[1]}, height=h, width=w, **kw)


def small_jpeg():
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(photo(16, 16, 9)).save(b, "JPEG", quality=80)
    return b.getvalue()


def writer_cases():
    """Every writer knob in each layout where it applies, on conforming content."""
    cases = []
    lays = list(J.LAYOUTS)
    colour = [l for l in lays if l != "gray"]
    for lay in lays:
        cases.append((f"std-{lay}", write(lay, seed=1)))
        cases.append((f"optimal-{lay}", write(lay, seed=2, huffman="optimal")))
        n = 1 if lay == "gray" else 3
        # SOF1, quantisation and Huffman table ids 2 and 3, 16-bit DQT
        coefs, samp = content(lay, seed=3)
        qt = {2: Q75[0], 3: Q75[1]} if n == 3 else {2: Q75[0]}
        cases.append((f"sof1-ids23-{lay}", J.write_jpeg(coefs, qt, height=37, width=53, sampling=samp, sof=0xC1,
                                                        tq=[2] + [3] * (n - 1), hsel=[(2, 3)] + [(3, 2)] * (n - 1),
                                                        huffman="optimal")))
        big = [np.clip(Q75[0] * 37, 1, 65535), np.clip(Q75[1] * 101, 1, 65535)]
        cases.append((f"dqt16-{lay}", write(lay, seed=4, qt=big, qprec={0: 1, 1: 1})))
        cases.append((f"dqt16-small-{lay}", write(lay, seed=5, qprec={0: 1, 1: 1} if n == 3 else {0: 1})))
        # restart intervals: every MCU, one that does not divide an MCU row, one larger than the image; an extra RSTn
        for r in (1, 3, 1000):
            cases.append((f"dri{r}-{lay}", write(lay, seed=6 + r, restart=r, extra_rst=r == 3)))
        # pad bits and fill bytes
        cases.append((f"pad-zeros-{lay}", write(lay, seed=7, restart=2, pad="zeros")))
        cases.append((f"pad-random-fill-{lay}", write(lay, seed=8, restart=2, pad="random", fill=3)))
        cases.append((f"tail-byte-{lay}", write(lay, seed=9, restart=5, tail_bytes=1)))
        # table placement
        cases.append((f"after-sof-{lay}", write(lay, seed=10, tables="after_sof", huffman="optimal")))
        cases.append((f"redefined-{lay}", write(lay, seed=11, tables="redefined")))
        # extra segments: an APP1 holding a whole JPEG, COM and APP13 payloads containing SOI / EOI
        segs = [(0xE1, b"Exif\x00\x00" + small_jpeg()), (0xFE, b"\xff\xd8 comment \xff\xd9"), (0xED, b"\xff\xd9\xff\xd8" * 7)]
        cases.append((f"segments-{lay}", write(lay, seed=12, segments=segs)))
    for lay in colour:
        # component ids in any order, Huffman ids 0-3 in any assignment (a scan listing the components out of frame order
        # is refused by libjpeg-turbo, see test_oracle_jpeg / test_jpeg_bitstreams)
        cases.append((f"ids-{lay}", write(lay, seed=13, ids=[200, 7, 42])))
        cases.append((f"ids-desc-{lay}", write(lay, seed=14, ids=[3, 2, 1], hsel=[(3, 1), (0, 2), (3, 1)], huffman="optimal")))
        cases.append((f"shared-table-{lay}", write(lay, seed=15, tq=[0, 0, 0], hsel=[(0, 0)] * 3)))
    # grey frame declaring non-1 sampling factors
    for samp in ((2, 2), (1, 3), (4, 1)):
        cases.append((f"gray-declared-{samp[0]}x{samp[1]}", write("gray", seed=16, sampling=[samp])))
    cases += huffman_cases()
    return cases


def _long16(freq):
    """The most common symbols get 16-bit codes, the rest short ones."""
    syms = sorted(freq, key=lambda s: -freq[s])
    top, rest = syms[:8], syms[8:]
    lengths = {s: 16 for s in top}
    if rest:
        lengths.update({s: int(np.ceil(np.log2(len(rest) + 1))) + 1 for s in rest})
    return J.table_from_lengths(lengths)


def huffman_cases():
    """Hand-made Huffman code-length distributions."""
    cases = []
    for lay in ("420", "gray", "422"):
        coefs, samp = content(lay, seed=20)
        n = len(coefs)
        qt = {0: Q75[0], 1: Q75[1]} if n == 3 else {0: Q75[0]}
        w = J.write_jpeg(coefs, qt, height=37, width=53, sampling=samp, huffman="optimal")
        # frequencies through the optimal tables' symbol sets: rebuild long-code tables over the same symbols
        hs = {}
        for key in [("dc", 0), ("ac", 0)] + ([("dc", 1), ("ac", 1)] if n == 3 else []):
            bits, vals = _table_of(w.data, key)
            order = {v: len(vals) - i for i, v in enumerate(vals)}   # shorter optimal code = more common
            hs[key] = _long16(order)
        cases.append((f"long16-{lay}", J.write_jpeg(coefs, qt, height=37, width=53, sampling=samp, huffman=hs)))
        # single-symbol DC table (every DC difference 0) and an AC table with only EOB (DC-only blocks)
        flat = [c.copy() for c in coefs]
        for c in flat:
            c[..., 0, 0] = 0
        one = {("dc", 0): ([1] + [0] * 15, [0]), ("ac", 0): "optimal", ("dc", 1): ([1] + [0] * 15, [0]), ("ac", 1): "optimal"}
        cases.append((f"dc-one-symbol-{lay}", J.write_jpeg(flat, qt, height=37, width=53, sampling=samp,
                                                           huffman={k: v for k, v in one.items() if n == 3 or k[1] == 0})))
        dconly = [c.copy() for c in coefs]
        for c in dconly:
            dc = c[..., 0, 0].copy()
            c[:] = 0
            c[..., 0, 0] = dc
        eob = {("dc", 0): "optimal", ("ac", 0): ([1] + [0] * 15, [0]), ("dc", 1): "optimal", ("ac", 1): ([1] + [0] * 15, [0])}
        cases.append((f"ac-eob-only-{lay}", J.write_jpeg(dconly, qt, height=37, width=53, sampling=samp,
                                                         huffman={k: v for k, v in eob.items() if n == 3 or k[1] == 0})))
    # AC magnitude categories 11-15 (and DC categories up to 15) with 16-bit tables of 1s: raw coefficients
    rng = np.random.default_rng(21)
    blocks = np.zeros((64, 8, 8), np.int64)
    for i, b in enumerate(blocks):
        s = 11 + i % 5
        k = rng.choice(63, 6, replace=False) + 1
        b.reshape(64)[k] = rng.integers(1 << (s - 1), 1 << s, 6) * rng.choice([-1, 1], 6)
        b[0, 0] = (i * 4093) % 32767 - 16000
    J.fix_dc_chain(blocks)
    cases.append(("ac-cat11-15", J.grey_file(blocks, np.ones(64, np.int64), 8, huffman="optimal")))
    return cases


def _table_of(data, key):
    """(bits, values) of DHT table `key` in a file (the last definition)."""
    out, i = None, 2
    while i < len(data):
        m, ln = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        if m == 0xDA:
            break
        if m == 0xC4:
            s, k = data[i + 4:i + 2 + ln], 0
            while k < len(s):
                cls, tid = ("ac" if s[k] >> 4 else "dc"), s[k] & 15
                bits = list(s[k + 1:k + 17])
                vals = list(s[k + 17:k + 17 + sum(bits)])
                if (cls, tid) == key:
                    out = (bits, vals)
                k += 17 + sum(bits)
        i += 2 + ln
    return out


def size_cases():
    """1xN, Nx1, sizes off the MCU grid, and a width of at least 8192."""
    cases = []
    for (h, w), lay in [((1, 37), "420"), ((29, 1), "422"), ((1, 1), "411"), ((1, 9000), "gray"), ((9, 1), "440"),
                        ((17, 33), "411"), ((23, 19), "420"), ((8, 8193), "420"), ((3, 8200), "444")]:
        cases.append((f"size-{h}x{w}-{lay}", write(lay, h=h, w=w, seed=h * 31 + w)))
    return cases


def extreme_cases():
    """Out-of-range coefficients in complete files: DC-only and full blocks with 8- and 16-bit tables, DC differences that
    walk the decoder's running DC past +-32767, 16-bit tables above 32767, in grey and colour."""
    rng = np.random.default_rng(30)
    cases = []
    for kind in ("dc", "full"):
        for wide in (False, True):
            q = rng.integers(1, 65536 if wide else 256, 64)
            cases.append((f"extreme-{kind}-{'q16' if wide else 'q8'}", J.grey_file(J.extreme_blocks(rng, 600, kind), q, 40,
                                                                                 huffman="optimal")))
    q = rng.integers(32768, 65536, 64)
    cases.append(("extreme-q-above-32767", J.grey_file(J.extreme_blocks(rng, 300, "full"), q, 20, huffman="optimal")))
    walk = np.zeros((200, 8, 8), np.int64)
    walk[:, 0, 0] = ((np.arange(200) * 20000 + 32768) & 0xFFFF) - 32768   # every difference +20000
    walk[1::3, 0, 3] = 5
    cases.append(("extreme-dc-walk", J.grey_file(walk, rng.integers(1, 256, 64), 25, huffman="optimal")))
    # colour: every component extreme, 4:2:0 and 4:4:4
    for lay in ("420", "444"):
        samp = [J.LAYOUTS[lay], (1, 1), (1, 1)]
        grid = J.block_grid(45, 70, samp)
        coefs = []
        for gh, gw in grid:
            b = J.extreme_blocks(rng, gh * gw, "full" if lay == "444" else "dc")
            b[:, 0, 0] //= 2   # DC within +-16384: no difference in MCU order is -32768
            coefs.append(b.reshape(gh, gw, 8, 8))
        qt = {0: rng.integers(1, 65536, 64), 1: rng.integers(1, 256, 64)}
        cases.append((f"extreme-colour-{lay}", J.write_jpeg(coefs, qt, height=45, width=70, sampling=samp, huffman="optimal")))
    return cases


# ---------------------------------------------------------------------------------------------------------------------
# Synchronisation boundaries of the Huffman kernel: 512-bit subsequences, windows of 256 of them
# ---------------------------------------------------------------------------------------------------------------------
SUBSEQ, WINDOW = 512, 256 * 512
# DC: difference 0 in 4 bits (the only one used); AC: EOB, ZRL and (0, 1..15) of 8 bits, so a coefficient of
# category s costs 8 + s bits (9-23), and (1, 15) of 16 bits: a 31-bit codeword with its magnitude.
SYNC_HUFF = {("dc", 0): J.table_from_lengths({0: 4, **{s: 5 for s in range(1, 16)}}),
             ("ac", 0): J.table_from_lengths({**{s: 8 for s in [0x00, 0xF0] + list(range(1, 16))}, 0x1F: 16})}


def _block(sizes):
    """Coefficients of a block whose AC codewords (with magnitudes) have the given bit sizes; 31 = run 1, category 15."""
    b = np.zeros(64, np.int64)
    k = 1
    for e in sizes:
        if e == 31:
            k += 1
            b[J.ZIGZAG[k]] = 1 << 14
        else:
            assert 9 <= e <= 23
            b[J.ZIGZAG[k]] = 1 << (e - 9)
        k += 1
    assert k <= 63
    return b.reshape(8, 8)


def segment_blocks(bits, nblocks):
    """`nblocks` blocks whose codewords take exactly `bits` bits with SYNC_HUFF (12 bits per block plus AC codewords)."""
    x = bits - 12 * nblocks
    m = -(-x // 23)
    assert x >= 9 * m and m <= 60 * nblocks, (bits, nblocks)
    sizes = [x // m + (i < x % m) for i in range(m)]
    return [_block(sizes[i::nblocks]) for i in range(nblocks)]


class Stream:
    """Blocks built codeword by codeword, tracking the bit position (DC 4 bits at a block's start, EOB 8 at its end)."""

    def __init__(self):
        self.blocks, self.cur, self.slots, self.pos = [], [], 0, 4

    def _next_block(self):
        self.blocks.append(_block(self.cur))
        self.cur, self.slots, self.pos = [], 0, self.pos + 12

    def add(self, e):
        if self.slots + (2 if e == 31 else 1) > 60:
            self._next_block()
        self.cur.append(e)
        self.slots += 2 if e == 31 else 1
        self.pos += e

    def fill_to(self, target):
        assert target - self.pos >= 40
        while target - self.pos > 32:
            if self.slots > 57:
                self._next_block()
            else:
                self.add(23)
        need = target - self.pos
        if need <= 23:
            self.add(need)
        else:
            self.add(need - 9)
            self.add(9)
        assert self.pos == target

    def finish(self):
        self.blocks.append(_block(self.cur))
        return np.stack(self.blocks)


def sync_cases():
    """Restart segments whose byte-padded length is 512k bits or a byte either side with the last codeword ending 1-8 bits
    before the segment's end; segments of one window and a byte either side; 1-byte segments; 31-bit codewords straddling
    subsequence and window boundaries."""
    cases = []
    padded = [p + d for p in (SUBSEQ, 2 * SUBSEQ, 3 * SUBSEQ) for d in (-8, 0, 8)]
    for tail in (0, 1):
        ends = [8] if tail else range(1, 8)
        targets = [p - e for p in padded for e in ends]
        blocks = np.concatenate([segment_blocks(t, 4) for t in targets])
        w = J.grey_file(blocks, np.ones(64, np.int64), len(blocks), huffman=SYNC_HUFF, restart=4, tail_bytes=tail)
        assert w.seg_bits == targets
        cases.append((f"sync-512k{'-tail-byte' if tail else ''}", w))
    targets = [WINDOW - 8 - 3, WINDOW - 1, WINDOW + 8 - 5, 2 * WINDOW - 2]
    blocks = np.concatenate([segment_blocks(t, 200) for t in targets])
    w = J.grey_file(blocks, np.ones(64, np.int64), 200, huffman=SYNC_HUFF, restart=200)
    assert w.seg_bits == targets
    cases.append(("sync-window", w))
    # 1-byte segments: a zero block costs 2 bits (DC 0 and EOB of 1 bit each); every third block is larger
    tiny = {("dc", 0): J.table_from_lengths({0: 1, **{s: 5 for s in range(1, 16)}}),
            ("ac", 0): J.table_from_lengths({0x00: 1, **{s: 6 for s in [0xF0] + list(range(1, 16))}, 0x1F: 16})}
    blocks = np.zeros((60, 8, 8), np.int64)
    blocks[2::3, 0, 1] = np.arange(20) + 1
    blocks[5::9, 2, 0] = 1 << 14   # zig-zag 3 after zig-zag 1: run 1, category 15
    w = J.grey_file(blocks, np.ones(64, np.int64), 12, huffman=tiny, restart=1)
    assert w.seg_bits[0] == 2
    cases.append(("sync-one-byte-segments", w))
    # 31-bit codewords starting 1-30 bits before a subsequence or window boundary
    s = Stream()
    for b, o in [(SUBSEQ, 1), (2 * SUBSEQ, 8), (3 * SUBSEQ, 15), (4 * SUBSEQ, 30), (7 * SUBSEQ, 16), (WINDOW, 1),
                 (WINDOW + SUBSEQ, 30), (2 * WINDOW, 17)]:
        s.fill_to(b - o)
        s.add(31)
    s.fill_to(s.pos + 100)
    blocks = s.finish()
    w = J.grey_file(blocks, np.ones(64, np.int64), 64, huffman=SYNC_HUFF)
    cases.append(("sync-straddle", w))
    return cases
