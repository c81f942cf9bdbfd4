"""oracle/deflate_ref.py writes streams zlib never emits; zlib itself must inflate each to the intended bytes."""
import zlib

import numpy as np

from oracle import deflate_ref as D


def _check(blocks, data):
    w = D.BitWriter()
    for k, (kind, tokens, kw) in enumerate(blocks):
        final = k == len(blocks) - 1
        if kind == "stored":
            D.stored(w, bytes(tokens), final)
        elif kind == "fixed":
            D.fixed(w, tokens, final)
        else:
            D.dynamic(w, tokens, final, **kw)
    raw = w.getvalue()
    assert zlib.decompress(raw, -15) == data
    assert zlib.decompress(D.zlib_wrap(raw, data)) == data


def test_stored_blocks_of_0_and_65535_bytes():
    data = np.random.default_rng(0).integers(0, 256, 70000, dtype=np.uint8).tobytes()
    _check([("stored", b"", {}), ("stored", data[:65535], {}), ("stored", data[65535:], {})], data)


def test_fixed_and_dynamic_tokens():
    toks = [1, 2, 3, (10, 3), 9, (258, 1), (258, 4, D.VIA_284), (3, 270)]
    data = D.expand(toks)
    assert len(data) == 3 + 10 + 1 + 258 + 258 + 3
    _check([("fixed", toks, {})], data)
    _check([("dynamic", toks, {})], data)
    _check([("dynamic", toks[:3], {}), ("fixed", toks[3:5], {}), ("dynamic", toks[5:], {})], data)


def test_distance_32768():
    head = np.random.default_rng(1).integers(0, 256, 32768, dtype=np.uint8).tobytes()
    toks = list(head) + [(258, 32768), (258, 32768)]
    _check([("dynamic", toks, {})], D.expand(toks))


def test_one_code_and_empty_distance_trees_and_15_bit_codes():
    toks = [5, (200, 1)]
    _check([("dynamic", toks, {"dist_lens": [1]})], D.expand(toks))
    lits = list(range(15)) * 3
    _check([("dynamic", lits, {"dist_lens": [0]})], bytes(lits))
    lit = [0] * 286
    for s, l in zip(list(range(15)) + [256], list(range(1, 15)) + [15, 15]):
        lit[s] = l
    _check([("dynamic", lits, {"lit_lens": lit, "dist_lens": [0]})], bytes(lits))
