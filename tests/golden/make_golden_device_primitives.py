"""Generate tests/golden/golden_device_primitives.json: the answers of the UNMODIFIED reference's rl_agents/utils.py on
the generated inputs of tests/device_primitive_cases.py, recorded as a sha256 per family (tests/device_primitive_cases.py
::digest) so that the file stays small:

  kl           bernoulli_kullback_leibler(p, q)
  kl_bound     kl_upper_bound(sum, count, threshold, lower=lower) with a Python-float sum; `float_type` lists the cases
               whose answer changes with an np.float64 sum (a Python float makes 1/x raise ZeroDivisionError, which
               takes newton_iteration's finite difference; an np.float64 gives inf instead), as [index, Python-float
               answer, np.float64 answer]; `named` spells out the named edge cases in full
  expectation  max_expectation_under_constraint(f, counts / counts.sum(), c)

Build-container only (the reference tree does not travel to the GPU box); the output is committed and the same bytes
on every run.  Usage:  python tests/golden/make_golden_device_primitives.py [--out PATH]
"""
import argparse
import json
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import ref_loader  # noqa: E402
from tests import device_primitive_cases as cases  # noqa: E402

ref_loader.load_reference()
from rl_agents.utils import (bernoulli_kullback_leibler, kl_upper_bound,  # noqa: E402
                             max_expectation_under_constraint)

H = float.hex


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or H(a) == H(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(HERE, "golden_device_primitives.json"))
    path = ap.parse_args().out
    warnings.simplefilter("ignore")          # the reference sets np.seterr(all="warn") and divides by zero on purpose
    kl = [float(bernoulli_kullback_leibler(p, q)) for _, p, q in cases.kl_inputs()]
    bounds, float_type, named = [], [], []
    for i, (tag, s, count, thr, lower) in enumerate(cases.kl_bound_inputs()):
        py = float(kl_upper_bound(float(s), count, thr, lower=lower))
        npf = float(kl_upper_bound(np.float64(s), count, thr, lower=lower))
        bounds.append(py)
        if not _same(py, npf):
            float_type.append([i, H(py), H(npf)])
        if tag != "random":
            named.append([tag, H(s), count, H(thr), lower, H(py)])
    expectation = []
    for _, f, counts, c in cases.expectation_inputs():
        expectation.append([float(v) for v in max_expectation_under_constraint(np.asarray(f),
                                                                               np.asarray(cases.q_of(counts)), c)])
    out = {"kl": {"n": len(kl), "sha256": cases.digest(kl)},
           "kl_bound": {"n": len(bounds), "sha256": cases.digest(bounds), "float_type": float_type, "named": named},
           "expectation": {"n": len(expectation), "sha256": cases.digest(expectation)}}
    with open(path, "w") as f:
        json.dump(out, f)
    print("device primitives: %d kl, %d kl_bound, %d expectation" % (len(kl), len(bounds), len(expectation)))


if __name__ == "__main__":
    main()
