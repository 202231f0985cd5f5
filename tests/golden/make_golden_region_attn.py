"""Generate the region_attn_mode golden fixtures (region_attn_cases.py) by running the UNMODIFIED reference on CPU, like make_golden.py.

The 'dual_region' cases use the one documented shim of make_golden_input_mode.py (importing it installs it): the reference's dual_region
step still calls the temporal attention on the dummy frame features and fails; its output is not used in that mode, so the shim returns
zeros of the right shape and nothing the mode computes changes.  No other case needs a shim.

Run in the build container only:  ``python tests/golden/make_golden_region_attn.py [case ...]``"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import gvd_b200.synth as synth  # noqa: E402
import make_golden_input_mode  # noqa: E402,F401  (installs the dual_region shim on ref_harness.build_reference_model)
import ref_harness as rh  # noqa: E402
from make_golden import run_case  # noqa: E402
from region_attn_cases import DP_KEYS_FIXTURES, REGION_ATTN_CASES  # noqa: E402


def state_dict_keys(overrides):
    opt = synth.make_opt(t_attn_size=10, **overrides)
    sd = rh.build_reference_model(opt, synth.make_detectron(opt)).state_dict()
    return dict(keys=np.array(list(sd.keys())), shapes=np.array([",".join(str(n) for n in v.shape) for v in sd.values()]))


def main():
    only = sys.argv[1:]
    for name, case in REGION_ATTN_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(name, case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-30s %6.1fs %8.1f KB" % (name, time.time() - t0, os.path.getsize(path) / 1024), flush=True)
    for name, overrides in DP_KEYS_FIXTURES.items():
        if not only or name in only:
            np.savez_compressed(os.path.join(HERE, name + ".npz"), **state_dict_keys(overrides))


if __name__ == "__main__":
    main()
