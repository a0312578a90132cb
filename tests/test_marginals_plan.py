"""Marginals plans (planner.build_marginals_plan, version-5 programs), checked on the CPU.

oracle/program_interp.py executes the serialised words with numpy, so a pass here means the
bucket tree (upward messages, downward messages, readouts), the strides, the evidence gathers and
the slot reuse the device will see are right: every target's segment must equal the reference's
single-variable answers (tests/golden) and oracle.ve_oracle.query."""
import hashlib

import numpy as np
import pytest

from conftest import build_network, case_event, dense_answer, golden_names, load_golden
from oracle import program_interp, ve_oracle
from sorobn_b200 import BayesNet, planner, synthetic, workloads


def oracle_net(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def segments(plan, net, post):
    """{target name: [card, B] slice of the posterior}."""
    out, q = {}, 0
    for t in plan.targets:
        c = int(net.card[t])
        out[net.names[t]] = post[q:q + c]
        q += c
    assert q == plan.Q == post.shape[0]
    return out


def patterns(golden):
    """Evidence patterns of a golden file: {evidence vars: [(row values, {single query var: case})]}."""
    out = {}
    for case in golden["cases"]:
        ev = case_event(case)
        out.setdefault(tuple(ev), []).append(case)
    return out


@pytest.mark.parametrize("name", golden_names())
def test_marginals_plan_matches_reference_goldens(name):
    golden = load_golden(name)
    bn = build_network(golden)
    net = bn._compiled
    dn = oracle_net(bn)
    checked = 0
    for ev_vars, cases in patterns(golden).items():
        if not ev_vars and len(net.names) > 40:
            continue  # no evidence on the benchmark grid: every variable is relevant, covered with evidence below
        rows = []
        for case in cases:
            ev = case_event(case)
            rows.append(tuple(ev[v] for v in ev_vars))
        rows = sorted(set(rows), key=repr)
        codes = np.array([[net.domains[net.index[v]].index(r[i]) for r in rows] for i, v in enumerate(ev_vars)],
                         dtype=np.uint8).reshape(len(ev_vars), len(rows))
        for mode in (planner.MODE_BATCHED, planner.MODE_FLAT):
            plan = planner.build_marginals_plan(net, [net.index[e] for e in ev_vars], mode=mode)
            assert plan.version == 5 and plan.words[1] == 5
            for b, row in enumerate(rows):
                if mode == planner.MODE_FLAT and b >= 2:
                    break
                sub = codes[:, b:b + 1] if mode == planner.MODE_FLAT else codes
                got = program_interp.run_marginals(plan.words, plan.table_blob64, sub, n_rows=1 if mode == planner.MODE_FLAT else len(rows))
                col = 0 if mode == planner.MODE_FLAT else b
                seg = segments(plan, net, got)
                for case in cases:
                    ev = case_event(case)
                    if tuple(ev[v] for v in ev_vars) != row:
                        continue
                    if len(case["query"]) == 1:
                        want = dense_answer(case, dn.domains)
                        got_t = seg[case["query"][0]][:, col]
                        if want.sum() == 0:  # impossible evidence: the reference's answer is empty
                            assert np.isnan(got_t).all(), case
                        else:
                            assert np.allclose(got_t, want, rtol=1e-12, atol=1e-300), case
                        checked += 1
                if len(net.names) <= 40 or b == 0:
                    ev = {v: row[i] for i, v in enumerate(ev_vars)}
                    for t, values in seg.items():
                        want = ve_oracle.query(dn, t, event=ev)[1].reshape(-1)
                        if not np.isfinite(want).all() or want.sum() == 0:
                            assert np.isnan(values[:, col]).all(), (t, ev)
                        else:
                            assert np.allclose(values[:, col], want, rtol=1e-12, atol=1e-300), (t, ev)
    assert checked > 0


def test_float32_interpretation_on_the_benchmark_grid():
    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    n = 256  # a float32 readout accumulator is off by 1.8e-6 on one of these rows: the check must see that
    codes = wl.codes(bn, n, seed=3)
    plan = planner.build_marginals_plan(net, [net.index[e] for e in wl.evidence])
    got64 = program_interp.run_marginals(plan.words, plan.table_blob64, codes)
    got32 = program_interp.run_marginals(plan.words, plan.table_blob, codes, dtype=np.float32)
    assert np.isfinite(got32).all()
    assert np.max(np.abs(got32 - got64) / np.maximum(got64, 1e-300) * (got64 > 1e-12)) < 1e-6
    assert np.allclose(got32.sum(axis=0), 70, rtol=1e-5)
    # every targetless grid variable's marginal equals its own query plan
    for t in (net.names[plan.targets[0]], net.names[plan.targets[35]], net.names[plan.targets[-1]]):
        p4 = planner.build_plan(net, [net.index[t]], [net.index[e] for e in wl.evidence])
        want = marginals_interp_v4(p4, codes)
        assert np.allclose(segments(plan, net, got64)[t], want, rtol=1e-10)


def marginals_interp_v4(plan, codes):
    return program_interp.run(plan.words, plan.table_blob64, codes)


def _check_against_oracle(bn, ev_vars, targets, B, seed):
    net = bn._compiled
    dn = oracle_net(bn)
    rng = np.random.default_rng(seed)
    codes = np.stack([rng.integers(0, net.card[net.index[v]], B) for v in ev_vars]).astype(np.uint8) if ev_vars \
        else np.zeros((0, B), np.uint8)
    plan = planner.build_marginals_plan(net, [net.index[e] for e in ev_vars],
                                        targets=None if targets is None else [net.index[t] for t in targets])
    got = program_interp.run_marginals(plan.words, plan.table_blob64, codes, n_rows=B)
    seg = segments(plan, net, got)
    if targets is not None:
        assert sorted(seg) == sorted(targets)
    for b in range(B):
        ev = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(ev_vars)}
        for t, values in seg.items():
            _, want, _ = ve_oracle.query(dn, t, event=ev)
            want = want.reshape(-1)
            if not np.isfinite(want).all() or want.sum() == 0:
                assert np.isnan(values[:, b]).all()
            else:
                assert np.allclose(values[:, b], want, rtol=1e-12, atol=1e-300), (t, ev)
    return plan


@pytest.mark.parametrize("trial", range(12))
def test_random_networks_targets_and_evidence(trial):
    rng = np.random.default_rng(100 + trial)
    n = int(rng.integers(3, 14))
    spec = synthetic.random_dag(n, 3, int(rng.integers(2, 5)), seed=trial)
    bn = synthetic.load(spec, BayesNet)
    perm = [spec.nodes[i] for i in rng.permutation(n)]
    ne = int(rng.integers(0, n - 1))
    ev_vars, rest = perm[:ne], perm[ne:]
    targets = None if trial % 2 == 0 else rest[:max(1, len(rest) // 2)]
    _check_against_oracle(bn, ev_vars, targets, 5, trial)


def test_no_evidence():
    bn = synthetic.load(synthetic.random_dag(9, 3, 3, seed=4), BayesNet)
    _check_against_oracle(bn, [], None, 1, 0)


def test_disconnected_network():
    """Two components plus a lone node: every root bucket's pi carries the other components' constants."""
    bn = BayesNet(("a", "b"), ("b", "c"), ("x", "y"), "z")
    rng = np.random.default_rng(5)
    import pandas as pd

    for node, parents in (("a", []), ("b", ["a"]), ("c", ["b"]), ("x", []), ("y", ["x"]), ("z", [])):
        scope = [*parents, node]
        idx = pd.MultiIndex.from_product([[0, 1, 2]] * len(scope), names=scope) if len(scope) > 1 \
            else pd.Index([0, 1, 2], name=node)
        raw = rng.random((3,) * len(scope)) + 0.05
        raw /= raw.sum(axis=-1, keepdims=True)
        bn.P[node] = pd.Series(raw.reshape(-1), index=idx)
    bn.prepare()
    _check_against_oracle(bn, ["c", "y"], None, 6, 1)
    _check_against_oracle(bn, ["c"], ["b", "z"], 4, 2)
    _check_against_oracle(bn, [], None, 1, 3)


def test_impossible_rows_are_nan():
    from sorobn_b200 import examples

    bn = examples.build(examples.NETWORKS["asia"])
    net = bn._compiled
    # "TB or cancer" is a deterministic OR: yes without either cause is impossible
    ev = ["Tuberculosis", "Lung cancer", "TB or cancer"]
    plan = planner.build_marginals_plan(net, [net.index[e] for e in ev])
    dom = {v: net.domains[net.index[v]] for v in ev}
    rows = [(False, False, True), (True, False, True)]
    codes = np.array([[dom[v].index(r[i]) for r in rows] for i, v in enumerate(ev)], dtype=np.uint8)
    got = program_interp.run_marginals(plan.words, plan.table_blob64, codes)
    assert np.isnan(got[:, 0]).all()
    assert np.isfinite(got[:, 1]).all()


@pytest.mark.parametrize("name", ["alarm", "grid10x10s5_bench", "dag20p4s4"])
def test_plan_structure(name):
    bn = build_network(load_golden(name))
    net = bn._compiled
    case = load_golden(name)["cases"][-1]
    ev_vars = [net.index[v] for v, _ in case["event"]]
    for mode in (planner.MODE_BATCHED, planner.MODE_FLAT):
        plan = planner.build_marginals_plan(net, ev_vars, mode=mode)
        names = [net.names[t] for t in plan.targets]
        assert names == sorted(names)
        assert set(plan.targets) == set(range(len(net.names))) - set(ev_vars)
        offsets = []
        for st in plan.steps:
            slots_in = [f.buf for f, _, _ in st.inputs if f.is_slot]
            assert st.out_slot not in slots_in, "a step's output aliases one of its inputs"
            assert len(st.inputs) <= planner.MAX_IN
            if st.kind == planner.KIND_MARGINAL:
                assert len(st.out_vars) == 1 and st.out_slot == -1
                offsets.append((st.q_offset, net.names[st.out_vars[0]]))
            else:
                assert len(st.elims) <= planner.MAX_ELIM and st.cx <= planner.MAX_Z
                assert len(st.cards) <= planner.MAX_AXES
        # segments in target order, back to back
        assert [n for _, n in sorted(offsets)] == names
        assert plan.bytes_per_row() > 0 and sum(plan.step_bytes_per_row()) > 0 or mode == planner.MODE_FLAT


# sha256 (first 16 hex digits) of build_plan's words + float64 table blob, computed at the commit that
# introduced marginals plans: build_plan's version-4 programs must not change by a single bit.
FROZEN = [
    ('alarm', ('Burglary',), (), 0, '402e4e4c537ebc3d'),
    ('alarm', ('Burglary',), (), 1, '045aaa8b90a89c14'),
    ('alarm', ('Burglary',), ('Earthquake',), 0, 'bfcdd408085b44a5'),
    ('alarm', ('Burglary',), ('Earthquake',), 1, '3aedb87847c787f8'),
    ('alarm', ('Burglary',), ('Alarm',), 0, 'f8cf3590ad6bd38b'),
    ('alarm', ('Burglary',), ('Alarm',), 1, '3f58290df3da6d82'),
    ('asia', ('Visit to Asia',), (), 0, '1b88b822b054129f'),
    ('asia', ('Visit to Asia',), (), 1, '6d67d38fbd79fed1'),
    ('asia', ('Visit to Asia',), ('Tuberculosis',), 0, 'f4ed31400c8efb7e'),
    ('asia', ('Visit to Asia',), ('Tuberculosis',), 1, '3a507e931dbf044f'),
    ('asia', ('Visit to Asia',), ('Smoker',), 0, 'effdcedcbf23c41d'),
    ('asia', ('Visit to Asia',), ('Smoker',), 1, '3e3887cce889c403'),
    ('chain9s4', ('c5', 'c3'), ('c4', 'c1', 'c0', 'c7', 'c6'), 0, 'e34712178813ae16'),
    ('chain9s4', ('c5', 'c3'), ('c4', 'c1', 'c0', 'c7', 'c6'), 1, '25f1eb825d05698e'),
    ('chain9s4', ('c5', 'c6'), (), 0, '6dc93af2c42e5748'),
    ('chain9s4', ('c5', 'c6'), (), 1, '0daa1f06a5e07809'),
    ('chain9s4', ('c1', 'c2'), ('c3', 'c5', 'c0', 'c8', 'c6'), 0, '18ff39f9064bd50a'),
    ('chain9s4', ('c1', 'c2'), ('c3', 'c5', 'c0', 'c8', 'c6'), 1, 'c6812f1fa347f99c'),
    ('dag12p3s3', ('v03', 'v06'), ('v09', 'v04', 'v05', 'v07', 'v08', 'v01', 'v00'), 0, '1d2a5cc2535719de'),
    ('dag12p3s3', ('v03', 'v06'), ('v09', 'v04', 'v05', 'v07', 'v08', 'v01', 'v00'), 1, '2913c75bc815ab53'),
    ('dag12p3s3', ('v01',), ('v02', 'v03', 'v08', 'v00', 'v05'), 0, '0aa067a8f9e110f9'),
    ('dag12p3s3', ('v01',), ('v02', 'v03', 'v08', 'v00', 'v05'), 1, '4aaf5a623d1c9e7b'),
    ('dag12p3s3', ('v02',), ('v00', 'v08', 'v11', 'v07', 'v04', 'v10'), 0, '1c43d4cce68dd71c'),
    ('dag12p3s3', ('v02',), ('v00', 'v08', 'v11', 'v07', 'v04', 'v10'), 1, 'f22411217f0e06da'),
    ('dag20p4s4', ('v05', 'v06'), ('v04', 'v03', 'v17', 'v14', 'v16', 'v09', 'v12', 'v08', 'v19', 'v07', 'v01'), 0, 'ad3577b775f44faf'),
    ('dag20p4s4', ('v05', 'v06'), ('v04', 'v03', 'v17', 'v14', 'v16', 'v09', 'v12', 'v08', 'v19', 'v07', 'v01'), 1, 'b18b9bf6dc32d0b6'),
    ('dag20p4s4', ('v02', 'v16'), ('v13', 'v11', 'v07', 'v14', 'v10', 'v01', 'v06', 'v19', 'v03', 'v18', 'v09', 'v15'), 0, '9d8b15cd0c0c885e'),
    ('dag20p4s4', ('v02', 'v16'), ('v13', 'v11', 'v07', 'v14', 'v10', 'v01', 'v06', 'v19', 'v03', 'v18', 'v09', 'v15'), 1, '2560c23cc6b07919'),
    ('dag20p4s4', ('v11', 'v03'), ('v04', 'v15', 'v10', 'v01', 'v18', 'v19', 'v14'), 0, '5b94065b5b6984b6'),
    ('dag20p4s4', ('v11', 'v03'), ('v04', 'v15', 'v10', 'v01', 'v18', 'v19', 'v14'), 1, '54f63fd31f6788a1'),
    ('grades', ('Difficulty',), (), 0, 'c53965731ee5d184'),
    ('grades', ('Difficulty',), (), 1, '847b053fd705e67d'),
    ('grades', ('Difficulty',), ('Intelligence',), 0, '589d01fb9b593096'),
    ('grades', ('Difficulty',), ('Intelligence',), 1, 'de393d1a33eed37f'),
    ('grades', ('Difficulty',), ('Grade',), 0, '0cee7077151fa2ca'),
    ('grades', ('Difficulty',), ('Grade',), 1, '0c985df7b89e3bc0'),
    ('grid10x10s5_bench', ('g0909',), ('g0002', 'g0007', 'g0100', 'g0102', 'g0109', 'g0201', 'g0202', 'g0204', 'g0300', 'g0301', 'g0303', 'g0304', 'g0306', 'g0403', 'g0407', 'g0500', 'g0504', 'g0505', 'g0602', 'g0608', 'g0609', 'g0703', 'g0706', 'g0707', 'g0709', 'g0804', 'g0808', 'g0900', 'g0901', 'g0906'), 0, '08150d9a76dc19d7'),
    ('grid10x10s5_bench', ('g0909',), ('g0002', 'g0007', 'g0100', 'g0102', 'g0109', 'g0201', 'g0202', 'g0204', 'g0300', 'g0301', 'g0303', 'g0304', 'g0306', 'g0403', 'g0407', 'g0500', 'g0504', 'g0505', 'g0602', 'g0608', 'g0609', 'g0703', 'g0706', 'g0707', 'g0709', 'g0804', 'g0808', 'g0900', 'g0901', 'g0906'), 1, 'e6bce0a503ffb65b'),
    ('grid4x4s3', ('g0100', 'g0200'), ('g0300', 'g0003', 'g0101', 'g0102', 'g0301', 'g0303', 'g0201'), 0, '7e70a55de9f4bfac'),
    ('grid4x4s3', ('g0100', 'g0200'), ('g0300', 'g0003', 'g0101', 'g0102', 'g0301', 'g0303', 'g0201'), 1, '5beeaf6b5e283bc5'),
    ('grid4x4s3', ('g0303',), ('g0002', 'g0003', 'g0001', 'g0102', 'g0203'), 0, 'e2908d2e90476827'),
    ('grid4x4s3', ('g0303',), ('g0002', 'g0003', 'g0001', 'g0102', 'g0203'), 1, '8aaadce18a3fad7d'),
    ('grid4x4s3', ('g0200',), ('g0003', 'g0300', 'g0101', 'g0000', 'g0102'), 0, '923dca708161dc29'),
    ('grid4x4s3', ('g0200',), ('g0003', 'g0300', 'g0101', 'g0000', 'g0102'), 1, '3a7559e2a992c075'),
    ('sprinkler', ('Cloudy',), (), 0, '88b4788194e05d62'),
    ('sprinkler', ('Cloudy',), (), 1, 'f2ef6bcd7e564f0a'),
    ('sprinkler', ('Cloudy',), ('Sprinkler',), 0, '0136b487f6fb8127'),
    ('sprinkler', ('Cloudy',), ('Sprinkler',), 1, '70432707cf8f6a53'),
    ('sprinkler', ('Cloudy',), ('Rain',), 0, '5d19f118d36944fc'),
    ('sprinkler', ('Cloudy',), ('Rain',), 1, '5c863144fb993a77'),
]


@pytest.mark.parametrize("name,query,evidence,mode,digest", FROZEN)
def test_build_plan_words_are_frozen(name, query, evidence, mode, digest):
    bn = build_network(load_golden(name))
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in query], [net.index[e] for e in evidence], mode=mode)
    assert plan.words[1] == 4
    assert hashlib.sha256(plan.words.tobytes() + plan.table_blob64.tobytes()).hexdigest()[:16] == digest
