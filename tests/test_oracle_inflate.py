"""oracle/inflate_ref.py against PIL (``read_image``) and zlib: the filtered bytes, or the refusal, for every stream of
tests/png_streams.py, and facts about Pillow 12.2 / zlib 1.3 that the GPU inflate restates: after the image's last byte zlib
checks only the rest of the read (at most 64 KiB, never across an IDAT) that completed it, and an invalid code in a stream's
last bits is an error, not a truncation.  Also the chunk search's verdicts the README cites."""
import zlib

import numpy as np
import pytest

from oracle import deflate_ref as D
from oracle import inflate_ref as I
import png_streams as S
from png_cases import filter_rows, pil_read, png_file, random_rows


def _same(f):
    exp, got = pil_read(f), I.pixels_as_pil(f)
    assert isinstance(exp, Exception) == isinstance(got, Exception), (exp, got)
    if not isinstance(exp, Exception):
        np.testing.assert_array_equal(got, exp)
    return not isinstance(exp, Exception)


def _stored_fill(extra):
    """One IDAT: two stored blocks whose last byte is the IDAT's byte 65535 + extra, then a bad Adler-32."""
    n = 65536 + extra - 12
    w_, h_ = n // 4 - 1, 4
    raw = bytearray(np.random.default_rng(0).integers(0, 256, n, dtype=np.uint8).tobytes())
    raw[::w_ + 1] = bytes(h_)
    w = D.BitWriter()
    D.stored(w, bytes(raw[:40000]), False)
    D.stored(w, bytes(raw[40000:]), True)
    z = D.zlib_wrap(w.getvalue(), bytes(raw))
    return png_file(w_, h_, 0, 8, z[:-1] + bytes([z[-1] ^ 1]))


def test_pil_checks_only_the_read_that_completed_the_image():
    # stored blocks that fill exactly the first 64 KiB read: the bad Adler-32 is in the next read
    assert _same(_stored_fill(0)) and not _same(_stored_fill(-4)) and not _same(_stored_fill(4))
    rng = np.random.default_rng(5)
    w, h = 40, 30
    raw = filter_rows(random_rows(rng, w, h, 2, 8, "photo"), 3, (0, 1, 2, 3, 4))
    co = zlib.compressobj(6, zlib.DEFLATED, -15)
    s = b"\x78\x9c" + co.compress(raw) + co.flush(zlib.Z_SYNC_FLUSH)
    bad = s + b"\x07\xff\xff\xff"           # an invalid block after the image
    assert _same(png_file(w, h, 2, 8, bad, split=[len(s)]))
    assert not _same(png_file(w, h, 2, 8, bad, split=[len(s) + 1])) and not _same(png_file(w, h, 2, 8, bad))
    z = zlib.compress(raw)
    z = z[:-1] + bytes([z[-1] ^ 1])
    assert _same(png_file(w, h, 2, 8, z, split=[len(z) - 4])) and _same(png_file(w, h, 2, 8, z, split=[len(z) - 2]))
    assert not _same(png_file(w, h, 2, 8, z))


def test_an_invalid_code_in_the_last_bits_is_an_error():
    rng = np.random.default_rng(5)
    raw = S._raw(rng)
    cases = S.last_bits_cases(raw)
    assert len(cases) == 28
    for name, f in cases:
        assert not _same(f), name
    # with the Adler-32 behind it PIL refuses too
    w = D.BitWriter()
    D.fixed(w, list(raw), False)
    lit = [0] * 257
    lit[256] = 1
    D.dynamic_header(w, True, 257, 1, S._cl(s0=1, s1=1), lit + [0])
    w.bits(1, 1)
    assert not _same(png_file(S.W, S.H, 0, 8, D.zlib_wrap(w.getvalue(), raw)))


def test_every_error_rule_in_three_places():
    cases = S.error_rule_cases()
    seen = set()
    for rule, place, f in cases:
        ok = _same(f)
        seen.add(rule)
        if place == "before":
            assert not ok, rule
        if place == "next IDAT":
            assert ok, rule
        if place == "same read" and rule not in ("distance before the stream", "length code behind an empty distance tree"):
            assert not ok, rule
    assert len(seen) == 21 + 28      # 21 rules, and the invalid code in each of the last 1..14 bits, two ways


@pytest.mark.parametrize("group", ["image_end", "multi_chunk"])
def test_oracle_is_pil(group):
    cases = S.image_end_cases() if group == "image_end" else S.multi_chunk_cases()
    verdicts = {name: _same(f) for name, f in cases}
    if group == "image_end":
        # the read ends after stream byte 65536k - 1: a bad block behind an image completed there is never read
        assert verdicts["literal, last bit at 65536*1-1"] and not verdicts["literal, last bit at 65536*1+0"]
        assert all(v for n, v in verdicts.items() if n.startswith("match past the end"))


def test_oracle_is_zlib_on_valid_streams():
    for name, f in S.multi_chunk_cases() + [(n, f) for n, f in S.image_end_cases() if "IDAT" in n and "bad" not in n and "past" not in n]:
        (w, h, c, d, _), _, idat = I.png_parts(f)
        total = h * (1 + I.row_bytes(w, c, d))
        got = I.inflate_as_pil(f)
        assert got == zlib.decompress(b"".join(idat))[:total], name


def _status(f):
    (w, h, c, d, _), _, idat = I.png_parts(f)
    z = b"".join(idat)
    return z, I.candidates(z), I.chunk_status(z, h * (1 + I.row_bytes(w, c, d)))


def test_chunk_chain_cases():
    cases = dict(S.multi_chunk_cases())
    z, cands, st = _status(cases["distance 32768 back over short chunks"])
    assert st[0] == 3 and st[1] == 2             # every chunk confirmed: the chain resolves references over two chunks
    z, cands, st = _status(cases["a chunk over its symbol capacity"])
    assert cands[1] >= 0 and st[1] == 0          # chunk 1 has a start, but its output overflows CHUNK_SYMBOLS
    z, cands, st = _status(cases["false candidate before the true block boundaries"])
    assert 65536 * 8 <= cands[1] and st[1] == 0  # chunk 1's start lies in a stored block's data: never confirmed
    z, cands, st = _status(cases["photo, fixed Huffman only"])
    assert st[1] == 0 and st[2] == len(zlib.decompress(z))


def test_stored_headers_parse_one_bit_early():
    """Why streams of stored blocks confirm no chunk but the final block's: a non-final stored header also parses strictly one
    bit before itself (its padding absorbs the shift), and the search takes the first bit that parses."""
    z, cands, st = _status(dict(S.multi_chunk_cases())["zlib level 0"])
    starts, br = [], I._Bits(z, 16)
    while True:
        starts.append(br.pos)
        last = br.take(1)
        assert br.take(2) == 0
        br.pos = (br.pos + 7) & ~7
        n = int.from_bytes(z[br.pos // 8:br.pos // 8 + 2], "little")
        br.pos += 32 + 8 * n
        if last:
            break
    for c in cands[1:]:
        if c < 0:
            continue
        t = min(s for s in starts if s >= c)
        assert c == t - 1 or (t == starts[-1] and c == t)
    assert st[1] == 1
