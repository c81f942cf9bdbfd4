"""csrc/png.cu's chunking constants, read from the source, against the GPU PNG cases: the streams tests/test_gpu_png.py decodes
must span several speculative chunks, and the status test must see chunks confirmed.  No GPU needed."""
import os
import re
import zlib

import numpy as np

from png_cases import make_png

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "k210_yolo_framework_b200", "csrc", "png.cu")


def constant(name):
    m = re.search(rf"constexpr (?:int|long long) {name} = ([^;]+);", open(SRC).read())
    assert m, name
    expr = m.group(1).replace("LL", "")
    for other in re.findall(r"[A-Z_]{4,}", expr):
        expr = expr.replace(other, str(constant(other)))
    return int(eval(expr))


def test_gpu_cases_cross_the_chunk_constants():
    chunk, max_chunks = constant("CHUNK_BYTES"), constant("MAX_CHUNKS")
    assert chunk == 65536 and max_chunks == 4096
    rng = np.random.default_rng(7)
    full_hd = make_png(rng, 1920, 1080, 2, 8, content="noise", level=1)          # test_full_hd
    assert len(full_hd) > 50 * chunk and len(full_hd) < chunk * max_chunks
    from jpeg_cases import photo
    from png_cases import pil_png
    status_case = pil_png(photo(720, 1280, 5))                                 # test_status_counts_chunks_and_serial_bytes
    assert len(status_case) > 3 * chunk
    # a speculative chunk holds CHUNK_SYMBOLS symbols: the status case's chunks inflate to far less
    assert constant("CHUNK_SYMBOLS") > 2 * chunk * 720 * 3841 // len(status_case)
    # test_deflate_ref_streams' stored case: 65535-byte stored blocks straddle chunk boundaries
    assert 300 * 256 > chunk
    assert constant("MAX_RAW_BYTES") == 2 ** 31 - 1
