"""Generate the att_input_mode golden fixtures (input_mode_cases.py) by running the UNMODIFIED reference on CPU, like make_golden.py.

One shim for 'dual_region' (no reference file is edited): as shipped, TopDownCore.forward still calls the temporal attention on the dummy
1 x 1 frame features (AttModel.py:140-141, model.py:406-408) and fails reshaping them.  Its output `att` is not used in that mode
(AttModel.py:153-156), so the shim makes core.attention return zeros of the right shape; nothing the mode computes changes.

Run in the build container only:  ``python tests/golden/make_golden_input_mode.py [case ...]``"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import gvd_b200.synth as synth  # noqa: E402
import ref_harness as rh  # noqa: E402
from input_mode_cases import DUAL_KEYS_FIXTURE, INPUT_MODE_CASES  # noqa: E402
from make_golden import run_case  # noqa: E402


_build = rh.build_reference_model


def _build_with_dual_shim(opt, detectron):
    model = _build(opt, detectron)
    if opt.att_input_mode == "dual_region":
        model.core.attention.forward = lambda h, *feats: h.new_zeros(h.shape[0], opt.rnn_size)
    return model


rh.build_reference_model = _build_with_dual_shim


def dual_keys():
    opt = synth.make_opt(t_attn_size=10, att_input_mode="dual_region")
    sd = rh.build_reference_model(opt, synth.make_detectron(opt)).state_dict()
    return dict(keys=np.array(list(sd.keys())), shapes=np.array([",".join(str(n) for n in v.shape) for v in sd.values()]))


def main():
    only = sys.argv[1:]
    for name, case in INPUT_MODE_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(name, case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %6.1fs %8.1f KB" % (name, time.time() - t0, os.path.getsize(path) / 1024), flush=True)
    if not only or DUAL_KEYS_FIXTURE in only:
        np.savez_compressed(os.path.join(HERE, DUAL_KEYS_FIXTURE + ".npz"), **dual_keys())


if __name__ == "__main__":
    main()
