"""Generate tests/golden/soft_{alarm,asia,grades,sprinkler}.json by running the real reference on soft evidence.

    python tools/gen_soft_golden.py     # needs the reference sources, as oracle/gen_golden.py does

The reference takes hard evidence only, so each case asks it Pearl's virtual-evidence question: a copy of the
example network with one binary child `__soft__<node>` per soft node, P(child = 1 | node = x) = lik(x) / max lik,
built through the reference's own BayesNet API and queried with the hard evidence and every child at 1.  A case
keeps the likelihoods (in the node's sorted domain order), the posterior and, with at least two observed columns,
log P(hard, lik) = log predict_proba(hard, children at 1) + sum log max.  Only the JSON is committed; it pins the
host entry points on the CPU (tests/test_soft_host.py) and on the GPU (tests/test_gpu_soft.py).  The reference
eliminates in set order, so two runs may differ in the last bit of a posterior.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gen_golden  # noqa: E402


def soft_cases(ref, examples, spec, n_cases, seed):
    import pandas as pd

    rng = np.random.default_rng(seed)
    nodes = list(spec)
    cases = []
    while len(cases) < n_cases:
        perm = [nodes[i] for i in rng.permutation(len(nodes))]
        n_soft = int(rng.integers(1, min(3, len(nodes) - 1) + 1))
        soft = sorted(perm[:n_soft])
        query = perm[n_soft] if rng.random() < 0.7 else soft[0]  # a soft node may be queried
        hard_nodes = [n for n in perm[n_soft + 1:n_soft + 1 + int(rng.integers(0, 3))] if n != query]
        hard = {n: gen_golden.jsonable(spec[n][1][int(rng.integers(len(spec[n][1])))]) for n in hard_nodes}
        virtual = dict(spec)
        lik, log_max = {}, 0.0
        for s in soft:
            states = sorted(spec[s][1])
            lam = rng.random(len(states)) * 10.0 ** rng.integers(-3, 3)
            lam[rng.random(len(states)) < 0.2] = 0.0
            if lam.max() == 0:
                lam[0] = 1.0
            lik[s] = [float(x) for x in lam]
            k = float(lam.max())
            log_max += float(np.log(k))
            virtual[f"__soft__{s}"] = ((s,), (0, 1), {(x,): (1.0 - l / k, l / k) for x, l in zip(states, lam)})
        bn = examples.build(virtual, cls=ref.BayesNet)
        event = {**hard, **{f"__soft__{s}": 1 for s in soft}}
        case = gen_golden.run_case(bn, (query,), event)
        if not case["values"] or not np.isfinite(case["values"]).all():
            continue  # hard evidence of probability zero: the reference's answer is empty
        case["event"] = [[k, v] for k, v in hard.items()]
        case["likelihoods"] = [[s, lik[s]] for s in soft]
        if len(event) >= 2:  # predict_proba of a single column returns the whole marginal
            p = float(bn.predict_proba(pd.DataFrame([event])).iloc[0])
            case["log_evidence"] = float(np.log(p)) + log_max if p > 0 else None
        cases.append(case)
    return cases


def main():
    ref = gen_golden.import_reference()
    from sorobn_b200 import examples

    for name, spec in examples.NETWORKS.items():
        cases = soft_cases(ref, examples, spec, 30, seed=21)
        with open(os.path.join(gen_golden.OUT, f"soft_{name}.json"), "w") as f:
            json.dump({"network": name, "kind": "soft_evidence", "cases": cases}, f)
        print(f"soft evidence {name}: {len(cases)} cases")


if __name__ == "__main__":
    main()
