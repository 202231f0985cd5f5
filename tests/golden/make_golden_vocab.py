"""Generate the wide-vocabulary golden fixtures (vocab_cases.py) by running the UNMODIFIED reference on CPU, like make_golden.py.

Run in the build container only:  ``python tests/golden/make_golden_vocab.py [case ...]``"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

from make_golden import run_case  # noqa: E402
from vocab_cases import VOCAB_CASES  # noqa: E402


def main():
    only = sys.argv[1:]
    for name, case in VOCAB_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(name, case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        extra = ""
        if "min_margin" in out:
            extra = " min_margin=%.2e unk_top1_steps=%d" % (out["min_margin"], out["unk_top1_steps"])
        print("%-28s %6.1fs %8.1f KB%s" % (name, time.time() - t0, os.path.getsize(path) / 1024, extra), flush=True)


if __name__ == "__main__":
    main()
