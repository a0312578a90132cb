"""Small networks aimed at the step-kernel variants the engine dispatches.

Each case is plain data: a generator of `sorobn_b200.synthetic` with its arguments, optional
post-processing of the spec (variables cut to a single state, structural zeros in the CPTs),
the query and evidence variables (indices into `spec.nodes`), and `claims`: coverage items of
`tests/kernel_census.variants` that the case must reach on the GPU.  The cases were picked from
a seeded search on an H100 (tools/variant_search.py); nothing is searched at test time.

Runtime features that do not show in a kernel name (pre-multiplied factors of paired steps, the
padding of 4-state variables to the pair tile, the number of evidence columns one canonical array
gathers) are exercised by how the cases are built (mixed 4/5-state lattices, evidence next to the
paired frontier); the census cannot confirm them.
"""
from __future__ import annotations

import itertools

import numpy as np

from sorobn_b200 import planner, synthetic
from oracle import ve_oracle


def make_spec(case):
    """The network of a case: generator output, then the post-processing the case asks for."""
    gen = getattr(synthetic, case["gen"])
    spec = gen(*case["args"], seed=case["seed"], **case.get("kwargs", {}))
    for k in case.get("single", ()):
        _make_single_state(spec, spec.nodes[k])
    if case.get("zeros"):
        _add_structural_zeros(spec, case["zeros"], case["seed"])
    return spec


def _make_single_state(spec, node):
    """Cut `node` to one state: its CPT becomes ones, and every child keeps the slice of its
    table at that state (still normalised)."""
    ps = spec.parents.get(node, [])
    spec.n_states[node] = 1
    spec.cpt[node] = np.ones((*[spec.n_states[p] for p in ps], 1))
    for child, cps in spec.parents.items():
        if node in cps:
            ax = cps.index(node)
            spec.cpt[child] = np.ascontiguousarray(np.take(spec.cpt[child], [0], axis=ax))


def _add_structural_zeros(spec, frac, seed):
    """Zero about `frac` of every CPT's entries (never the largest of a row) and renormalise."""
    rng = np.random.default_rng(10_000 + seed)
    for n in spec.nodes:
        arr = spec.cpt[n].copy()
        if arr.shape[-1] < 2:
            continue
        flat = arr.reshape(-1, arr.shape[-1])
        keep = flat.argmax(axis=1)
        mask = rng.random(flat.shape) < frac
        mask[np.arange(flat.shape[0]), keep] = False
        flat[mask] = 0.0
        flat /= flat.sum(axis=1, keepdims=True)
        spec.cpt[n] = flat.reshape(arr.shape)


def compiled_net(spec):
    """`planner.CompiledNet` of a spec (states 0..card-1, node order = generation order, which is
    topological)."""
    index = {n: i for i, n in enumerate(spec.nodes)}
    return planner.CompiledNet(
        names=list(spec.nodes),
        domains=[list(range(spec.n_states[n])) for n in spec.nodes],
        parents=[[index[p] for p in spec.parents.get(n, [])] for n in spec.nodes],
        cpt=[np.asarray(spec.cpt[n], dtype=np.float64) for n in spec.nodes],
    )


def dense_net(spec):
    """The float64 oracle's view of the same network."""
    dn = ve_oracle.DenseNet(nodes=list(spec.nodes), parents={k: list(v) for k, v in spec.parents.items()},
                            domains={n: list(range(spec.n_states[n])) for n in spec.nodes})
    for n in spec.nodes:
        dn.cpt[n] = np.asarray(spec.cpt[n], dtype=np.float64)
    return dn


def build(case, mode=planner.MODE_BATCHED):
    """(spec, CompiledNet, DenseNet, plan, query names, evidence names) of a case."""
    spec = make_spec(case)
    net = compiled_net(spec)
    query = [spec.nodes[k] for k in case["query"]]
    evidence = [spec.nodes[k] for k in case["evidence"]]
    plan = planner.build_plan(net, [net.index[q] for q in query], [net.index[e] for e in evidence], mode=mode)
    return spec, net, dense_net(spec), plan, query, evidence


def evidence_rows(spec, evidence, n_rows, seed=0):
    """uint8 codes [n_ev, n_rows]: every joint code of the evidence columns first (codes of
    probability zero and codes at card - 1 included), then forward samples.  When the joint codes
    outnumber the rows, the rows are every column at 0, every column at card - 1, each column alone
    at card - 1, and forward samples."""
    if not evidence:
        return np.zeros((0, n_rows), dtype=np.uint8)
    cards = np.array([spec.n_states[v] for v in evidence])
    if np.prod(cards, dtype=np.float64) <= n_rows:
        joint = np.array(list(itertools.product(*[range(c) for c in cards])), dtype=np.uint8).T
    else:
        edges = [np.zeros(len(cards), dtype=np.uint8), (cards - 1).astype(np.uint8)]
        for k in range(len(cards)):
            row = np.zeros(len(cards), dtype=np.uint8)
            row[k] = cards[k] - 1
            edges.append(row)
        joint = np.stack(edges, axis=1)
    if joint.shape[1] < n_rows:
        ev = synthetic.random_events(spec, evidence, n_rows - joint.shape[1], seed=seed)
        joint = np.concatenate([joint, np.stack([ev[v].to_numpy().astype(np.uint8) for v in evidence])], axis=1)
    return np.ascontiguousarray(joint[:, :n_rows])


def naive_bayes(n_children=60, root_states=5, child_states=17, seed=0):
    """A class variable `c` with `n_children` children `f00`, `f01`, ... and no other edge: the shape
    where the product over a variable's children in the Gibbs conditional underflows float32.  The
    CPT entries are float32 values (rows sum to 1 within float32 rounding), so the float64 oracle
    and the device's float32 tables hold the same numbers."""
    rng = np.random.default_rng(seed)
    kids = [f"f{k:02d}" for k in range(n_children)]
    nodes = ["c", *kids]
    cpt = {"c": rng.dirichlet(np.ones(root_states))}
    for k in kids:
        cpt[k] = rng.dirichlet(np.ones(child_states), size=root_states)
    cpt = {n: np.asarray(a, dtype=np.float32).astype(np.float64) for n, a in cpt.items()}
    return synthetic.NetSpec(f"naive{n_children}s{root_states}x{child_states}", nodes, {k: ["c"] for k in kids},
                             {"c": root_states, **{k: child_states for k in kids}}, cpt)


def case_id(case):
    return case["name"]


def case_name(case):
    """A readable, unique name: network, seed, post-processing, query and evidence count."""
    a = case["args"]
    tag = a[-1] if np.isscalar(a[-1]) else "x".join(map(str, a[-1]))
    name = (f"grid{a[0]}x{a[1]}" if case["gen"] == "grid" else f"dag{a[0]}p{a[1]}") + f"s{tag}_seed{case['seed']}"
    if case.get("single"):
        name += "_single" + "-".join(map(str, case["single"]))
    if case.get("zeros"):
        name += "_zeros"
    return name + "_q" + "-".join(map(str, case["query"])) + f"_e{len(case['evidence'])}"


def plan_items(plan):
    """Coverage items read from the plan: a launched step whose tables exceed the shared-memory
    budget is laid out for sliced staging (planner._relayout_big_tables)."""
    size = [n for _, n in plan.table_offsets]
    big = any(sum(size[f.buf] for f, _, _ in st.inputs if not f.is_slot) * 4 > planner.SLICE_MIN_BYTES
              for st in plan.steps if st.kind == planner.KIND_BATCHED)
    return {"tiled sliced staging"} if big else set()


CASES = [
    {'name': 'dag9p2s4x1x4x4_seed54_q1-8_e2', 'gen': 'random_dag', 'args': [9, 2, [4, 1, 4, 4]], 'seed': 54, 'kwargs': {'window': 6}, 'query': [1, 8], 'evidence': [3, 0], 'claims': ['batched CX=1', 'batched N_IN=4', 'tiled (1,1,2,0)', 'tiled T=2 CX=0']},
    {'name': 'dag16p4s5x8_seed63_single8-0_q14_e3', 'gen': 'random_dag', 'args': [16, 4, [5, 8]], 'seed': 63, 'kwargs': {'window': 4}, 'query': [14], 'evidence': [15, 8, 13], 'single': [8, 0], 'claims': ['batched CX=1', 'batched N_IN=4', 'tiled (2,2,0,0)', 'tiled T=5 CX=0']},
    {'name': 'dag14p4s5x8_seed1_zeros_q10-13_e1', 'gen': 'random_dag', 'args': [14, 4, [5, 8]], 'seed': 1, 'kwargs': {'window': 6}, 'query': [10, 13], 'evidence': [0], 'zeros': 0.3, 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=8', 'batched N_IN=1', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'tiled (0,0,0,1)', 'tiled (0,1,1,0)', 'tiled (1,0,0,1)', 'tiled (1,1,1,0)', 'tiled (2,1,1,0)', 'tiled C-side T=2', 'tiled MX cx_inner=8', 'tiled T=2 CX=0', 'tiled T=4 CX=0']},
    {'name': 'dag8p2s37x3x2_seed3_q0-3_e2', 'gen': 'random_dag', 'args': [8, 2, [37, 3, 2]], 'seed': 3, 'kwargs': {'window': 3}, 'query': [0, 3], 'evidence': [1, 2], 'claims': ['batched CX=1', 'batched N_IN=4', 'tiled (2,1,1,0)', 'tiled T=2 CX=0']},
    {'name': 'dag7p2s13x9x4_seed5_q6_e2', 'gen': 'random_dag', 'args': [7, 2, [13, 9, 4]], 'seed': 5, 'kwargs': {'window': 3}, 'query': [6], 'evidence': [1, 2], 'claims': ['batched CX=1', 'batched N_IN=3', 'tiled (2,1,0,0)', 'tiled T=2 CX=0']},
    {'name': 'dag6p2s37x2_seed1_q2_e2', 'gen': 'random_dag', 'args': [6, 2, [37, 2]], 'seed': 1, 'kwargs': {'window': 3}, 'query': [2], 'evidence': [1, 3], 'claims': ['batched CX=1', 'batched N_IN=2', 'tiled (1,1,0,0)', 'tiled T=2 CX=0']},
    {'name': 'grid10x10s5_seed0_q99_e30', 'gen': 'grid', 'args': [10, 10, 5], 'seed': 0, 'query': [99], 'evidence': [2, 7, 10, 12, 19, 21, 22, 24, 30, 31, 33, 34, 36, 43, 47, 50, 54, 55, 62, 68, 69, 73, 76, 77, 79, 84, 88, 90, 91, 96], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=5', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,0)', 'pair (0,1)', 'pair (1,0)', 'pair (1,2)', 'pair (2,0)', 'pair (2,1)', 'pair (4,0)', 'tiled (0,1,1,0)', 'tiled (0,1,2,0)', 'tiled (0,2,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (2,1,0,0)', 'tiled (2,1,1,0)', 'tiled (2,2,0,0)', 'tiled MX cx_inner=5', 'tiled T=5 CX=0', 'tiled T=5 CX=5', 'triple group=5']},
    {'name': 'grid10x10s4_seed0_q99_e30', 'gen': 'grid', 'args': [10, 10, 4], 'seed': 0, 'query': [99], 'evidence': [2, 7, 10, 12, 19, 21, 22, 24, 30, 31, 33, 34, 36, 43, 47, 50, 54, 55, 62, 68, 69, 73, 76, 77, 79, 84, 88, 90, 91, 96], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=4', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,0)', 'pair (0,1)', 'pair (1,0)', 'pair (1,2)', 'pair (2,0)', 'tiled (0,1,1,0)', 'tiled (0,1,2,0)', 'tiled (0,2,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (2,2,0,0)', 'tiled MX cx_inner=4', 'tiled T=4 CX=0', 'tiled T=4 CX=4']},
    {'name': 'grid10x10s3_seed0_q99_e30', 'gen': 'grid', 'args': [10, 10, 3], 'seed': 0, 'query': [99], 'evidence': [2, 7, 10, 12, 19, 21, 22, 24, 30, 31, 33, 34, 36, 43, 47, 50, 54, 55, 62, 68, 69, 73, 76, 77, 79, 84, 88, 90, 91, 96], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=3', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'tiled (0,1,1,0)', 'tiled (0,2,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (2,2,0,0)', 'tiled MX cx_inner=3', 'tiled T=3 CX=0', 'tiled T=3 CX=3']},
    {'name': 'grid10x10s2_seed0_q99_e30', 'gen': 'grid', 'args': [10, 10, 2], 'seed': 0, 'query': [99], 'evidence': [2, 7, 10, 12, 19, 21, 22, 24, 30, 31, 33, 34, 36, 43, 47, 50, 54, 55, 62, 68, 69, 73, 76, 77, 79, 84, 88, 90, 91, 96], 'claims': ['batched CX=1', 'batched CX=2', 'batched CX=4', 'batched CX=8', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'tiled (0,1,1,0)', 'tiled (0,2,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (2,2,0,0)', 'tiled MX cx_inner=2', 'tiled T=2 CX=0', 'tiled T=2 CX=2']},
    {'name': 'dag300p1s17_seed2_q0_e5', 'gen': 'random_dag', 'args': [300, 1, 17], 'seed': 2, 'query': [0], 'evidence': [11, 129, 135, 183, 227], 'claims': ['batched CX=0', 'batched N_IN=5']},
    {'name': 'dag300p1s17_seed5_q0_e6', 'gen': 'random_dag', 'args': [300, 1, 17], 'seed': 5, 'query': [0], 'evidence': [1, 6, 42, 66, 152, 279], 'claims': ['batched CX=0', 'batched N_IN=6']},
    {'name': 'dag300p1s17_seed16_q0_e7', 'gen': 'random_dag', 'args': [300, 1, 17], 'seed': 16, 'query': [0], 'evidence': [1, 2, 3, 9, 13, 65, 196], 'claims': ['batched CX=0', 'batched N_IN=7']},
    {'name': 'dag300p1s17_seed34_q0_e8', 'gen': 'random_dag', 'args': [300, 1, 17], 'seed': 34, 'query': [0], 'evidence': [3, 6, 9, 29, 36, 181, 211, 262], 'claims': ['batched CX=0', 'batched N_IN=8']},
    {'name': 'dag16p4s8_seed0_q15_e2', 'gen': 'random_dag', 'args': [16, 4, 8], 'seed': 0, 'kwargs': {'window': 8}, 'query': [15], 'evidence': [3, 9], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=8', 'batched N_IN=2', 'batched N_IN=3', 'tiled (0,1,1,0)', 'tiled (1,1,0,0)', 'tiled MX cx_inner=8', 'tiled T=4 CX=0', 'tiled T=4 CX=8', 'tiled sliced staging']},
    {'name': 'grid7x7s5_seed39_q48_e18', 'gen': 'grid', 'args': [7, 7, 5], 'seed': 39, 'query': [48], 'evidence': [0, 3, 5, 6, 12, 15, 18, 20, 21, 24, 25, 28, 32, 33, 42, 45, 46, 47], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=5', 'batched N_IN=1', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,0)', 'pair (0,1)', 'pair (1,0)', 'tiled (0,0,1,1)', 'tiled (0,1,0,0)', 'tiled (0,1,0,1)', 'tiled (0,1,1,0)', 'tiled (0,1,1,1)', 'tiled (1,0,0,1)', 'tiled (1,1,0,0)', 'tiled (1,1,0,1)', 'tiled (1,1,1,0)', 'tiled (1,2,0,0)', 'tiled (2,1,0,0)', 'tiled (2,2,0,0)', 'tiled C-side T=5', 'tiled MX cx_inner=5', 'tiled T=5 CX=0', 'tiled T=5 CX=5']},
    {'name': 'grid8x8s4x5_seed10_q63_e9', 'gen': 'grid', 'args': [8, 8, [4, 5]], 'seed': 10, 'query': [63], 'evidence': [4, 8, 28, 32, 35, 48, 49, 54, 61], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=4', 'batched CX=5', 'batched N_IN=1', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,0)', 'pair (1,0)', 'pair (4,0)', 'tiled (0,0,0,1)', 'tiled (0,1,0,0)', 'tiled (0,1,1,0)', 'tiled (0,2,2,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (1,1,2,0)', 'tiled C-side T=2', 'tiled MX cx_inner=5', 'tiled T=2 CX=0', 'tiled T=4 CX=0', 'tiled T=5 CX=0', 'tiled T=5 CX=5']},
    {'name': 'dag15p4s6_seed79_q7_e2', 'gen': 'random_dag', 'args': [15, 4, 6], 'seed': 79, 'kwargs': {'window': 6}, 'query': [7], 'evidence': [4, 9], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=6', 'batched N_IN=2', 'tiled (0,2,0,0)', 'tiled (1,0,0,1)', 'tiled (1,1,0,0)', 'tiled C-side T=3', 'tiled T=3 CX=0']},
    {'name': 'grid10x10s5_seed60_q99_e26', 'gen': 'grid', 'args': [10, 10, 5], 'seed': 60, 'query': [99], 'evidence': [0, 5, 8, 10, 20, 22, 31, 34, 36, 40, 41, 44, 45, 47, 48, 53, 55, 60, 71, 75, 83, 84, 88, 91, 92, 98], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=5', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,1)', 'pair (1,0)', 'pair (2,0)', 'pair (3,0)', 'pair (3,1)', 'pair (4,0)', 'pair (4,1)', 'tiled (0,1,0,1)', 'tiled (0,1,1,0)', 'tiled (0,1,1,1)', 'tiled (1,1,0,0)', 'tiled (1,1,0,1)', 'tiled (1,1,1,0)', 'tiled (2,2,0,0)', 'tiled C-side T=5', 'tiled MX cx_inner=5', 'tiled T=5 CX=0', 'tiled T=5 CX=5']},
    {'name': 'grid10x10s4x5_seed76_q99_e29', 'gen': 'grid', 'args': [10, 10, [4, 5]], 'seed': 76, 'query': [99], 'evidence': [1, 3, 7, 9, 23, 25, 26, 30, 35, 38, 42, 49, 51, 53, 56, 57, 58, 59, 62, 67, 68, 69, 70, 71, 74, 83, 89, 90, 92], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=4', 'batched CX=5', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'pair (0,0)', 'pair (0,1)', 'pair (1,0)', 'tiled (0,1,1,0)', 'tiled (0,2,1,0)', 'tiled (1,0,1,1)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (1,1,1,1)', 'tiled (2,2,0,0)', 'tiled C-side T=2', 'tiled C-side T=4', 'tiled C-side T=5', 'tiled MX cx_inner=5', 'tiled T=2 CX=0', 'tiled T=4 CX=0', 'tiled T=4 CX=4', 'tiled T=5 CX=0', 'tiled T=5 CX=5']},
    {'name': 'grid8x8s5_seed74_q63_e11', 'gen': 'grid', 'args': [8, 8, 5], 'seed': 74, 'query': [63], 'evidence': [2, 15, 18, 20, 21, 27, 35, 36, 54, 61, 62], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=5', 'batched N_IN=2', 'batched N_IN=3', 'pair (0,0)', 'pair (0,1)', 'pair (0,2)', 'pair (1,0)', 'pair (1,1)', 'pair (4,0)', 'tiled (0,1,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (2,1,0,0)', 'tiled MX cx_inner=5', 'tiled T=5 CX=0', 'tiled T=5 CX=5']},
    {'name': 'dag19p7s3_seed93_q12_e3', 'gen': 'random_dag', 'args': [19, 7, 3], 'seed': 93, 'kwargs': {'window': 8}, 'query': [12], 'evidence': [8, 5, 2], 'claims': ['batched CX=0', 'batched CX=1', 'batched CX=3', 'batched N_IN=1', 'batched N_IN=2', 'batched N_IN=3', 'batched N_IN=4', 'tiled (0,0,0,1)', 'tiled (0,1,0,0)', 'tiled (0,2,1,0)', 'tiled (1,1,0,0)', 'tiled (1,1,1,0)', 'tiled (1,2,1,0)', 'tiled C-side T=3', 'tiled MX cx_inner=3', 'tiled T=3 CX=0', 'tiled T=3 CX=3']},
]

# Coverage items no network can reach, with the reason.  The GPU test asserts that no case ever
# produces one of them.
_NO_PRELOAD_4 = "launch_tiled (sbn_api.cu) turns preload off for 4-input steps other than (2,1,1,0)"
UNREACHABLE = {
    f"tiled ({c}) T={t} CX={cx}{mx}": _NO_PRELOAD_4
    for c in ("0,2,2,0", "1,2,1,0", "1,1,2,0", "2,2,0,0")
    for t, cx in ((2, 2), (3, 3), (4, 4), (4, 8), (5, 5))
    for mx in ("", " MX")
}
# plan_slab (sbn_api.cu) takes a step only when the slab has >= 512 floats (c0 x private states of A
# x eliminated states), and only when 512 rows of that slab fit kSlabSmemMax = 96 KB, i.e. <= 192 floats
_SLAB = "plan_slab asks for >= 512 slab floats but fits at most 192 in kSlabSmemMax: it never takes a step"
UNREACHABLE.update({f"slab NU={nu} T={t} CX={t}": _SLAB for nu in (0, 1) for t in (2, 3, 4, 5)})
UNREACHABLE["slab NU=0 T=4 CX=8"] = _SLAB

# Reachable as far as the dispatch code shows, but no network of the seeded search reaches them.
# The GPU test fails when a case starts to reach one, so that it moves into that case's claims.
OPEN = {
    "pair (2,2)": "CE coefficients in both steps: no searched network forms it",
    "pair (3,2)": "GB first step with CE coefficients in the second: no searched network forms it",
    "pair (4,2)": "GC first step with CE coefficients in the second: no searched network forms it",
    "triple group=1": "every searched triple had a 5-state tile axis only its first operand carries (group 5)",
}

# Items every case reaches: the test always runs the single-event programs and the float64 batch.
ALWAYS = {"flat<float>", "flat<double>", "batched_f64"}


def required_items():
    """Every coverage item the corpus must reach (tests/kernel_census.variants spells them)."""
    req = set()
    combos = [(0, 1, 0, 0), (0, 1, 1, 0), (0, 1, 2, 0), (0, 2, 0, 0), (0, 2, 1, 0), (0, 2, 2, 0), (1, 1, 0, 0),
              (1, 1, 1, 0), (1, 1, 2, 0), (1, 2, 0, 0), (1, 2, 1, 0), (2, 1, 0, 0), (2, 1, 1, 0), (2, 2, 0, 0),
              (0, 0, 0, 1), (0, 0, 1, 1), (0, 1, 0, 1), (0, 1, 1, 1), (1, 0, 0, 1), (1, 0, 1, 1), (1, 1, 0, 1),
              (1, 1, 1, 1)]
    for c in combos:
        req.add("tiled ({},{},{},{})".format(*c))
    for t in (2, 3, 4, 5):
        req.add(f"tiled T={t} CX=0")
        req.add(f"tiled T={t} CX={t}")
        req.add(f"tiled C-side T={t}")
        for nu in (0, 1):
            req.add(f"slab NU={nu} T={t} CX={t}")
    req.add("tiled T=4 CX=8")
    req.add("tiled sliced staging")
    req.add("slab NU=0 T=4 CX=8")
    for k in (2, 3, 4, 5, 8):
        req.add(f"tiled MX cx_inner={k}")
    # the preload instantiations (with and without MX) of the 4-input combinations
    for c in ((0, 2, 2, 0), (1, 2, 1, 0), (1, 1, 2, 0), (2, 2, 0, 0)):
        for t in (2, 3, 4, 5):
            req.add("tiled ({},{},{},{}) T={t} CX={t}".format(*c, t=t))
            req.add("tiled ({},{},{},{}) T={t} CX={t} MX".format(*c, t=t))
        req.add("tiled ({},{},{},{}) T=4 CX=8".format(*c))
        req.add("tiled ({},{},{},{}) T=4 CX=8 MX".format(*c))
    for n in range(1, 9):
        req.add(f"batched N_IN={n}")
    for cx in (0, 1, 2, 3, 4, 5, 6, 8):
        req.add(f"batched CX={cx}")
    for m1 in range(5):
        for m2 in range(3):
            req.add(f"pair ({m1},{m2})")
    req.add("triple group=1")
    req.add("triple group=5")
    req.update({"flat<float>", "flat<double>", "batched_f64"})
    return req
