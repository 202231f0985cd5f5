"""Generate the transfer_mode 'none' and enable_BUTD golden fixtures (region_feat_cases.py) by running the UNMODIFIED reference on CPU, like make_golden.py.
No shim beyond ref_harness.py's.  It also checks that the reference fails for transfer_mode 'glove' and 'both' at the places the library
names when it refuses them (capi._TRANSFER_REFUSED).

Run in the build container only:  ``python tests/golden/make_golden_region_feat.py [case ...]``"""
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)

import gvd_b200.synth as synth  # noqa: E402
import ref_harness as rh  # noqa: E402
from cases import SMALL, build_case  # noqa: E402
from make_golden import run_case  # noqa: E402
from region_feat_cases import BUTD_KEYS_FIXTURE, NONE_KEYS_FIXTURE, REGION_FEAT_CASES  # noqa: E402
import make_golden_tfm_train as tfm_train  # noqa: E402


def state_dict_keys(**kw):
    opt = synth.make_opt(t_attn_size=10, **kw)
    sd = rh.build_reference_model(opt, synth.make_detectron(opt)).state_dict()
    return dict(keys=np.array(list(sd.keys())), shapes=np.array([",".join(str(n) for n in v.shape) for v in sd.values()]))


def check_refused_modes():
    """'glove' fails while the module is built (fc7 weights into a [300, 2048] layer); 'both' builds, then fails at pool_embed."""
    import torch
    opt = synth.make_opt(**dict(SMALL, transfer_mode="glove"))
    try:
        rh.build_reference_model(opt, synth.make_detectron(opt))
        raise AssertionError("transfer_mode='glove' built")
    except RuntimeError as e:
        print("glove: %s" % str(e).splitlines()[0])
    case = dict(kind="mle", B=2, opt=dict(SMALL, transfer_mode="both"), weight_seed=3, input_seed=5)
    opt = synth.make_opt(**case["opt"])
    model = rh.build_reference_model(opt, synth.make_detectron(opt))
    assert tuple(model.ctx2pool_grd[0].weight.shape) == (2348, 2048) and model.pool_embed[0].weight.shape[1] == 2048 + 300 + opt.detect_size + 1
    opt_c, _, inp = build_case(dict(case, opt=dict(SMALL)))       # inputs do not depend on transfer_mode
    try:
        with torch.no_grad():
            rh.ref_mle(model, inp)
        raise AssertionError("transfer_mode='both' ran")
    except RuntimeError as e:
        print("both: %s" % str(e).splitlines()[0])


def main():
    only = sys.argv[1:]
    for name, case in REGION_FEAT_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = tfm_train.run_case(case) if case["kind"] == "tfm_train" else run_case(name, case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %6.1fs %8.1f KB" % (name, time.time() - t0, os.path.getsize(path) / 1024), flush=True)
    if not only or NONE_KEYS_FIXTURE in only:
        np.savez_compressed(os.path.join(HERE, NONE_KEYS_FIXTURE + ".npz"), **state_dict_keys(transfer_mode="none"))
    if not only or BUTD_KEYS_FIXTURE in only:
        np.savez_compressed(os.path.join(HERE, BUTD_KEYS_FIXTURE + ".npz"),
                            **state_dict_keys(att_model="transformer", att_input_mode="region", enable_BUTD=True))
    if not only:
        check_refused_modes()


if __name__ == "__main__":
    main()
