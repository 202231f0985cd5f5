"""Generate the multinomial-sampling fixtures (sample_max = 0) by running the UNMODIFIED reference (read-only checkout, see ref_harness).

Run in the build container only:  ``python tests/golden/make_golden_sample.py``
The reference draws each token with ``torch.multinomial(prob_prev, 1)`` (misc/model.py:596-601).  For the run that call is replaced by
``argmax(log(prob_prev) + noise(t))`` with the counter-based Gumbel noise of tests/sample_ref.py: the Gumbel-max trick, the same
distribution with a reproducible draw.  Everything else is the reference's own code, including its temperature == 1.0 branch.
The case list lives here (not in cases.py::CASES) so the existing fixture parametrizations stay as they are.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(HERE)), "oracle"))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from cases import SMALL, build_case  # noqa: E402

SAMPLE_CASES = {
    # full model dims (H=1024, V=4905, R=10x100); temperature 1.0 takes the reference's exp(logprobs) branch (model.py:596-597)
    "multinomial_T10_B3":       dict(kind="multinomial", B=3, opt=dict(t_attn_size=10), temperature=1.0, noise_seed=2024),
    # reduced dims, a sharpened and a flattened distribution (model.py:599-600)
    "multinomial_small_B5_t07": dict(kind="multinomial", B=5, opt=SMALL, weight_seed=3, input_seed=5, temperature=0.7, noise_seed=7),
    "multinomial_small_B5_t15": dict(kind="multinomial", B=5, opt=SMALL, weight_seed=3, input_seed=5, temperature=1.5, noise_seed=15),
}


def run_case(case):
    import gvd_b200.synth as synth
    import ref_harness as rh
    from sample_ref import noise_fn
    opt, sd, inp = build_case(case)
    model = rh.build_reference_model(opt, synth.make_detectron(opt))
    model.load_state_dict(sd, strict=True)
    model.eval()
    B = inp["ppls"].shape[0]
    noise = noise_fn(case["noise_seed"], np.arange(B), opt.vocab_size)
    calls, gaps = [], []

    def multinomial(prob_prev, n):
        assert n == 1
        key = torch.log(prob_prev.double()) + noise(len(calls))
        calls.append(1)
        top2 = torch.topk(key, 2, dim=1).values
        gaps.append(float((top2[:, 0] - top2[:, 1]).min()))
        return key.argmax(dim=1, keepdim=True)

    orig = torch.multinomial
    torch.multinomial = multinomial
    try:
        with torch.no_grad():
            seq, logp, att2, _ = model._sample(inp["segs_feat"], inp["ppls"], inp["num"], inp["ppls_feat"], inp["sample_idx"], inp["pnt_mask"],
                                               {"sample_max": 0, "beam_size": 1, "temperature": case["temperature"]})
    finally:
        torch.multinomial = orig
    assert len(calls) == opt.seq_length
    return dict(seq=seq.numpy(), logp=logp.numpy(), att2=att2.numpy(), min_gap=np.float64(min(gaps)))


def main():
    only = sys.argv[1:]
    for name, case in SAMPLE_CASES.items():
        if only and name not in only:
            continue
        t0 = time.time()
        out = run_case(case)
        path = os.path.join(HERE, name + ".npz")
        np.savez_compressed(path, **out)
        print("%-28s %6.1fs %8.1f KB min_gap=%.2e uniq=%d" % (name, time.time() - t0, os.path.getsize(path) / 1024, out["min_gap"],
                                                              len(np.unique(out["seq"]))))


if __name__ == "__main__":
    main()
