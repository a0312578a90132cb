"""Generate tests/golden/joint_{alarm,asia,grades,sprinkler}.json by running the real reference's `query` on the
unobserved members of CPT families and of pairs of nodes.

    python tools/gen_joint_golden.py     # needs the reference sources, as oracle/gen_golden.py does

Each case is one partial row of the example network: a few hard cells at random states.  For every group -- each
node's family, [*parents, node], and two random pairs of nodes -- the reference answers `query(*unobserved members,
event=hard cells)`, the joint posterior that `BayesNet.joint_marginals_many` places at the row's observed codes; a
group the row observes completely has nothing to ask and is left out.  For hard cells of probability zero the
reference's answers are empty, and `joint_marginals_many` gives NaN.  Only the JSON is committed.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import gen_golden  # noqa: E402


def joint_cases(ref, examples, spec, n_cases, seed):
    rng = np.random.default_rng(seed)
    bn = examples.build(spec, cls=ref.BayesNet)
    nodes = sorted(spec)
    cases = []
    while len(cases) < n_cases:
        perm = [nodes[i] for i in rng.permutation(len(nodes))]
        hard_nodes = perm[:int(rng.integers(0, len(nodes) - 1))]
        hard = {n: gen_golden.jsonable(spec[n][1][int(rng.integers(len(spec[n][1])))]) for n in hard_nodes}
        groups = [[*spec[n][0], n] for n in nodes]
        for _ in range(2):
            a, b = rng.choice(len(nodes), 2, replace=False)
            groups.append([nodes[a], nodes[b]])
        answers = []
        try:
            for g in groups:
                M = [m for m in g if m not in hard]
                if M:
                    answers.append(dict(group=g, **gen_golden.run_case(bn, M, hard)))
        except Exception:  # a row the reference cannot answer at all is left out
            continue
        cases.append(dict(hard=[[k, v] for k, v in hard.items()], answers=answers))
    return cases


def main():
    ref = gen_golden.import_reference()
    from sorobn_b200 import examples

    for name, spec in examples.NETWORKS.items():
        cases = joint_cases(ref, examples, spec, 12, seed=17)
        with open(os.path.join(gen_golden.OUT, f"joint_{name}.json"), "w") as f:
            json.dump({"network": name, "kind": "joint", "cases": cases}, f)
        print(f"joint {name}: {len(cases)} cases, {sum(len(c['answers']) for c in cases)} answers")


if __name__ == "__main__":
    main()
