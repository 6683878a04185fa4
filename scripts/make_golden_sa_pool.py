"""Write tests/golden/sa_pool.npz: the SA max-pool outputs of the signed-zero chains in tests/test_gpu_mlp_pool.py
(ZERO_CASES x folded x linear), as int32 bit patterns of `out` (b, C, npoint).

    python scripts/make_golden_sa_pool.py [OUT]

The committed file was written by the staged shared-memory pool that the register pool replaced, so the test holds the
new pool to the old one's bits, the sign of zero included.  Needs a GPU.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_mlp_pool as T  # noqa: E402


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else T.GOLDEN
    dev = torch.device("cuda", 0)
    gold = {}
    for case in T.ZERO_CASES:
        for folded in (True, False):
            for linear in (False, True):
                o = T.sa_signed_zero_run(dev, case, folded, linear)()[0].view(torch.int32).cpu().numpy().copy()
                k = T.golden_key(case, folded, linear)
                gold[k] = o
                print("%-40s +0: %5d  -0: %5d  words: %d" % (k, (o == 0).sum(), (o == -2 ** 31).sum(), o.size))
    np.savez_compressed(out_path, **gold)


if __name__ == "__main__":
    main()
