"""Generate tests/golden/soft_impute_{alarm,asia,grades,sprinkler}.json by running the real reference's `impute` on
soft evidence.

    python tools/gen_soft_impute_golden.py     # needs the reference sources, as oracle/gen_golden.py does

The reference takes hard evidence only, so each case asks it Pearl's virtual-evidence question, as
tools/gen_soft_golden.py does: a copy of the example network with one binary child `__soft__<node>` per soft node,
P(child = 1 | node = x) = lik(x) / max lik, built through the reference's own BayesNet API.  `impute` then fills
2 or 3 missing cells of a sample that observes a few hard cells and every child at 1: the joint mode of the missing
cells given the hard cells and the likelihoods, every other node summed out -- the marginal MAP state that
`BayesNet.map_many(..., likelihoods=)` computes.  (With a single missing cell the reference's `impute` fails: its
posterior then has a flat index, bayes_net.py:905.)  A case keeps the sample's hard and missing cells, the
likelihoods (in the node's sorted domain order) and the imputed values.  Only the JSON is committed.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gen_golden  # noqa: E402


def impute_cases(ref, examples, spec, n_cases, seed):
    rng = np.random.default_rng(seed)
    nodes = list(spec)
    cases = []
    while len(cases) < n_cases:
        perm = [nodes[i] for i in rng.permutation(len(nodes))]
        n_missing = int(rng.integers(2, min(3, len(nodes) - 2) + 1))
        missing = perm[:n_missing]
        rest = perm[n_missing:]
        n_soft = int(rng.integers(1, min(2, len(rest)) + 1))
        soft = sorted(rest[:n_soft])
        hard_nodes = rest[n_soft:n_soft + int(rng.integers(0, 3))]
        hard = {n: gen_golden.jsonable(spec[n][1][int(rng.integers(len(spec[n][1])))]) for n in hard_nodes}
        virtual = dict(spec)
        lik = {}
        for s in soft:
            states = sorted(spec[s][1])
            lam = rng.random(len(states)) * 10.0 ** rng.integers(-3, 3)
            k = float(lam.max())
            lik[s] = [float(x) for x in lam]
            virtual[f"__soft__{s}"] = ((s,), (0, 1), {(x,): (1.0 - l / k, l / k) for x, l in zip(states, lam)})
        bn = examples.build(virtual, cls=ref.BayesNet)
        sample = {**hard, **{m: None for m in missing}, **{f"__soft__{s}": 1 for s in soft}}
        try:
            out = bn.impute(sample)
        except Exception:  # hard cells of probability zero: the reference has no posterior to take the mode of
            continue
        cases.append(dict(hard=[[k, v] for k, v in hard.items()], missing=sorted(missing),
                          likelihoods=[[s, lik[s]] for s in soft],
                          imputed=[[m, gen_golden.jsonable(out[m])] for m in sorted(missing)]))
    return cases


def main():
    ref = gen_golden.import_reference()
    from sorobn_b200 import examples

    for name, spec in examples.NETWORKS.items():
        cases = impute_cases(ref, examples, spec, 20, seed=31)
        with open(os.path.join(gen_golden.OUT, f"soft_impute_{name}.json"), "w") as f:
            json.dump({"network": name, "kind": "soft_impute", "cases": cases}, f)
        print(f"soft impute {name}: {len(cases)} cases")


if __name__ == "__main__":
    main()
