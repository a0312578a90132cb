"""Seeded search for small networks that reach the step-kernel variants (needs an H100).

Generates candidate cases in the format of tests/kernel_corpus.py (grids and random DAGs over
many cardinality patterns, some with single-state variables or structural zeros), runs each one
under the kernel census (tests/kernel_census.py) with the default dispatch, the plain batched
kernel (`set_tiled(False)`) and no paired steps (`set_tiled(10)`), and writes what each reached
to OUT/variant_search.json.
A greedy cover of the required items (`cover`) is written to OUT/corpus_cases.py: that list is
tests/kernel_corpus.py's CASES.

    python tools/variant_search.py --out DIR [--n 1500]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import kernel_census  # noqa: E402
import kernel_corpus  # noqa: E402

CARDS = [2, 3, 4, 5, 6, 7, 8, 9, 13, [4, 5], [5, 4], [4, 4, 5], [5, 5, 4], [2, 5, 3], [8, 2, 4, 3], [3, 8], [8, 4],
         [5, 8], [2, 8], [1, 4, 5], [4, 1, 4, 4]]


GRID_CARDS = [2, 3, 4, 5, 8, [4, 5], [5, 4], [4, 4, 5], [5, 5, 4], [4, 5, 5, 4]]


def candidates(n, seed=0):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        cards = CARDS[int(rng.integers(len(CARDS)))]
        u = rng.random()
        if u < 0.3:
            # lattices swept from one corner: frontier chains (pairs, triples, expanding products)
            r, c = [(5, 5), (6, 6), (7, 7), (8, 8), (6, 10), (10, 10)][int(rng.integers(6))]
            case = {"gen": "grid", "args": [r, c, GRID_CARDS[int(rng.integers(len(GRID_CARDS)))]], "seed": int(rng.integers(100))}
            n_nodes = r * c
            case["query"] = [n_nodes - 1] if rng.random() < 0.7 else [n_nodes - 2, n_nodes - 1]
            ne = int(rng.integers(0, 5))
            case["evidence"] = sorted(int(k) for k in rng.choice(n_nodes // 2, size=ne, replace=False))
        elif u < 0.4:
            # many parents: steps with up to eight inputs
            n_nodes = int(rng.integers(10, 20))
            case = {"gen": "random_dag", "args": [n_nodes, int(rng.integers(5, 8)), [2, 3][int(rng.integers(2))]],
                    "seed": int(rng.integers(100)), "kwargs": {"window": 8}}
            perm = [int(k) for k in rng.permutation(n_nodes)]
            case["query"] = perm[:1]
            case["evidence"] = perm[1:1 + int(rng.integers(0, 5))]
        if u < 0.4:
            spec = kernel_corpus.make_spec(case)
            if int(np.prod([spec.n_states[spec.nodes[k]] for k in case["evidence"]])) > 625:
                continue
            case["name"] = f"c{len(out):04d}"
            out.append(case)
            continue
        if rng.random() < 0.45:
            r, c = [(3, 3), (3, 4), (4, 4), (4, 5), (5, 5), (3, 6)][int(rng.integers(6))]
            case = {"gen": "grid", "args": [r, c, cards], "seed": int(rng.integers(100))}
            n_nodes = r * c
        else:
            n_nodes = int(rng.integers(6, 17))
            case = {"gen": "random_dag", "args": [n_nodes, int(rng.integers(2, 5)), cards], "seed": int(rng.integers(100)),
                    "kwargs": {"window": int(rng.integers(3, 7))}}
        perm = [int(k) for k in rng.permutation(n_nodes)]
        nq = 1 + int(rng.random() < 0.3)
        ne = int(rng.integers(0, 5))
        case["query"] = perm[:nq]
        case["evidence"] = perm[nq:nq + ne]
        if rng.random() < 0.15:
            case["single"] = [int(k) for k in rng.choice(n_nodes, size=2, replace=False)]
        if rng.random() < 0.2:
            case["zeros"] = 0.3
        try:
            spec = kernel_corpus.make_spec(case)
        except Exception:
            continue
        if int(np.prod([spec.n_states[spec.nodes[k]] for k in case["evidence"]])) > 256:
            continue
        if int(np.prod([spec.n_states[spec.nodes[k]] for k in case["query"]])) > 2000:
            continue
        case["name"] = f"c{len(out):04d}"
        out.append(case)
    # hand-made shapes: big cardinalities, a 37-state pair of query variables
    extra = [
        {"gen": "random_dag", "args": [8, 2, [37, 3, 2]], "seed": 3, "kwargs": {"window": 3}, "query": [0, 3], "evidence": [1, 2]},
        {"gen": "random_dag", "args": [7, 2, [13, 9, 4]], "seed": 5, "kwargs": {"window": 3}, "query": [6], "evidence": [1, 2]},
        {"gen": "random_dag", "args": [6, 2, [37, 2]], "seed": 1, "kwargs": {"window": 3}, "query": [2], "evidence": [1, 3]},
    ]
    extra += [
        # a 5-state lattice with the benchmark grid's 30 observed nodes; and the same shape in 2, 3 and 4 states
        {"gen": "grid", "args": [10, 10, 5], "seed": 0, "query": [99], "evidence": BENCH_EVIDENCE},
        {"gen": "grid", "args": [10, 10, 4], "seed": 0, "query": [99], "evidence": BENCH_EVIDENCE},
        {"gen": "grid", "args": [10, 10, 3], "seed": 0, "query": [99], "evidence": BENCH_EVIDENCE},
        {"gen": "grid", "args": [10, 10, 2], "seed": 0, "query": [99], "evidence": BENCH_EVIDENCE},
        # a root with 4..7 observed 17-state children: the final product has 5..8 inputs that are too big to fold
        {"gen": "random_dag", "args": [300, 1, 17], "seed": 2, "query": [0], "evidence": [11, 129, 135, 183, 227]},
        {"gen": "random_dag", "args": [300, 1, 17], "seed": 5, "query": [0], "evidence": [1, 6, 42, 66, 152, 279]},
        {"gen": "random_dag", "args": [300, 1, 17], "seed": 16, "query": [0], "evidence": [1, 2, 3, 9, 13, 65, 196]},
        {"gen": "random_dag", "args": [300, 1, 17], "seed": 34, "query": [0], "evidence": [3, 6, 9, 29, 36, 181, 211, 262]},
        # a single-state query variable; single-state evidence and hidden variables; structural zeros
        {"gen": "random_dag", "args": [9, 2, [4, 1, 4, 4]], "seed": 54, "kwargs": {"window": 6}, "query": [1, 8], "evidence": [3, 0]},
        {"gen": "random_dag", "args": [16, 4, [5, 8]], "seed": 63, "kwargs": {"window": 4}, "query": [14], "evidence": [15, 8, 13],
         "single": [8, 0]},
        {"gen": "random_dag", "args": [14, 4, [5, 8]], "seed": 1, "kwargs": {"window": 6}, "query": [10, 13], "evidence": [0],
         "zeros": 0.3},
        # 8 states, 4 parents: 128 KB tables, staged in slices
        {"gen": "random_dag", "args": [16, 4, 8], "seed": 0, "kwargs": {"window": 8}, "query": [15], "evidence": [3, 9]},
    ]
    for k, case in enumerate(extra):
        case["name"] = f"x{k:02d}"
        out.append(case)
    # lattices with many observed nodes (expanding products, triples, slab), pure 5-state lattices (GB / GC pairs)
    rng = np.random.default_rng(seed + 1)
    for k in range(n // 2):
        r, c = [(5, 5), (6, 6), (7, 7), (8, 8), (10, 10)][int(rng.integers(5))]
        cards = [2, 3, 4, 5, 5, 5, [4, 5], [5, 4]][int(rng.integers(8))]
        n_nodes = r * c
        ne = int(rng.integers(0, min(41, n_nodes // 2)))
        case = {"gen": "grid", "args": [r, c, cards], "seed": int(rng.integers(100)), "query": [n_nodes - 1],
                "evidence": sorted(int(v) for v in rng.choice(n_nodes - 1, size=ne, replace=False)), "name": f"d{k:04d}"}
        out.append(case)
    return out


# the observed nodes of the benchmark grid (sorobn_b200.workloads.grid10x10)
BENCH_EVIDENCE = [2, 7, 10, 12, 19, 21, 22, 24, 30, 31, 33, 34, 36, 43, 47, 50, 54, 55, 62, 68, 69, 73, 76, 77, 79, 84,
                  88, 90, 91, 96]


def cover(results, required):
    """The hand-made cases (x..) always, then greedily the case that reaches most items still missing
    (ties: fewer evidence columns, then the earlier candidate)."""
    reach = {k: set(r["items"]) & required for k, r in results.items() if "items" in r}
    chosen = [k for k in reach if k.startswith("x")]
    left = required - set().union(*[reach[k] for k in chosen])
    while True:
        best = max(sorted(reach), key=lambda k: (len(reach[k] & left), -len(results[k]["case"]["evidence"])))
        if not reach[best] & left:
            return chosen
        chosen.append(best)
        left -= reach[best]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1500)
    ap.add_argument("--rows", type=int, default=300)
    args = ap.parse_args()
    from sorobn_b200 import engine

    results = {}
    cases = candidates(args.n)
    for lo in range(0, len(cases), 50):
        batch, runs = [], []
        for case in cases[lo:lo + 50]:
            try:
                spec, net, dn, plan, query, evidence = kernel_corpus.build(case)
            except ValueError as e:
                results[case["name"]] = {"case": case, "error": str(e)}
                continue
            if plan.max_factor_per_row() > 100_000:  # small cases only: the corpus runs at every row count
                continue
            codes = kernel_corpus.evidence_rows(spec, evidence, args.rows)
            default = engine.Program(plan)
            plain = engine.Program(plan)
            plain.set_tiled(False)
            unpaired = engine.Program(plan)
            unpaired.set_tiled(10)
            runs += [(default, codes, args.rows), (plain, codes, args.rows), (unpaired, codes, args.rows)]
            batch.append((case, plan, (default, plain, unpaired)))
        seen = kernel_census.census_many(runs)
        for k, (case, plan, progs) in enumerate(batch):
            items = set().union(*[kernel_census.variants(s) for s in seen[3 * k:3 * k + 3]])
            results[case["name"]] = {"case": case, "items": sorted(items | kernel_corpus.plan_items(plan))}
            for prog in progs:
                prog.close()
        print(f"{lo + len(batch)} / {len(cases)}", flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "variant_search.json"), "w") as f:
        json.dump(results, f)
    required = kernel_corpus.required_items() - kernel_corpus.ALWAYS
    chosen = cover(results, required)
    with open(os.path.join(args.out, "corpus_cases.py"), "w") as f:
        f.write("CASES = [\n")
        for k in chosen:
            case = {key: v for key, v in results[k]["case"].items() if key != "name"}
            case = {"name": kernel_corpus.case_name(case), **case,
                    "claims": sorted(set(results[k]["items"]) & kernel_corpus.required_items())}
            f.write(f"    {case!r},\n")
        f.write("]\n")
    union = set().union(*[set(r.get("items", ())) for r in results.values()])
    missing = sorted(required - union)
    print("chosen", len(chosen), "reached", len(union), "missing", len(missing))
    for m in missing:
        print("  ", m)


if __name__ == "__main__":
    main()
