"""Records tests/golden/conv_tc_bitexact.npz: SHA-256 digests of the tensor-core conv outputs and of the cfg-2 bench
detections that tests/test_gpu_conv_tc_bitexact.py checks, computed by the library that is built in the tree.  Run it on an
H100 with the build whose outputs are the reference; the committed digests come from the build of commit 4e4b738.

    python tests/golden/make_conv_tc_bitexact.py [OUT]
"""
import importlib.util
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def main():
    spec = importlib.util.spec_from_file_location("_bitexact", os.path.join(os.path.dirname(HERE), "test_gpu_conv_tc_bitexact.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = sys.argv[1] if len(sys.argv) > 1 else mod.GOLDEN
    with tempfile.TemporaryDirectory() as tmp:
        d = mod.all_digests(tmp)
    np.savez(out, **d)
    print(f"{out}: {len(d)} digests")


if __name__ == "__main__":
    main()
