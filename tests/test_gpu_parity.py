"""Parity of the CUDA path with the reference (golden vectors) and the oracle.

Every test here calls through the C ABI (ctypes -> libsorobn_b200.so).  Tolerance:
1e-6 relative on every posterior entry (BASELINE.json's north_star); the arithmetic is
fp32 on the device against float64 in the reference.
"""
import numpy as np
import pandas as pd
import pytest

from conftest import build_network, case_event, dense_answer, golden_names, load_golden  # noqa: F401

pytestmark = pytest.mark.gpu

RTOL = 1e-6


def rel_err(got, want):
    got = np.asarray(got, dtype=np.float64).reshape(-1)
    want = np.asarray(want, dtype=np.float64).reshape(-1)
    mask = want > 0
    err = 0.0
    if mask.any():
        err = float(np.max(np.abs(got[mask] - want[mask]) / want[mask]))
    if (~mask).any():
        err = max(err, float(np.max(np.abs(got[~mask]))))  # exact zeros must stay zero
    return err


@pytest.mark.parametrize("name", golden_names())
def test_query_matches_reference_goldens(name):
    """BayesNet.query (flat kernels, one event) against the reference's own answers:
    same index (zero rows dropped), same values."""
    golden = load_golden(name)
    bn = build_network(golden)
    worst = 0.0
    for case in golden["cases"]:
        ans = bn.query(*case["query"], event=case_event(case))
        assert list(ans.index.names) == case["names"]
        got_idx = [list(k) if isinstance(k, tuple) else [k] for k in ans.index.tolist()]
        assert got_idx == case["index"], (case["query"], case["event"])
        assert ans.name == f"P({', '.join(case['query'])})"
        if case["values"]:
            worst = max(worst, rel_err(ans.to_numpy(), case["values"]))
    assert worst < RTOL, worst


@pytest.mark.parametrize("name", golden_names())
def test_query_many_matches_reference_goldens(name):
    """The batched kernels on the same cases: golden cases that share (query, evidence
    variables) are answered together as one batch."""
    golden = load_golden(name)
    bn = build_network(golden)
    net = bn._compiled
    groups = {}
    for case in golden["cases"]:
        key = (tuple(case["query"]), tuple(k for k, _ in case["event"]))
        groups.setdefault(key, []).append(case)
    worst = 0.0
    for (query, ev_vars), cases in groups.items():
        events = pd.DataFrame([case_event(c) for c in cases], columns=list(ev_vars), index=range(len(cases)))
        got = bn.query_many(*query, events=events)
        assert got.shape[0] == len(cases)
        domains = {n: net.domains[net.index[n]] for n in cases[0]["names"]}
        for row, case in zip(got.to_numpy(), cases):
            want = dense_answer(case, domains).reshape(-1)
            if not case["values"]:  # impossible evidence: reference returns an empty Series
                assert np.isnan(row).all()
                continue
            worst = max(worst, rel_err(row, want))
    assert worst < RTOL, worst


def test_reference_doctests_on_device():
    from sorobn_b200 import examples

    bn = examples.sprinkler()
    assert np.allclose(bn.query("Rain", event={"Sprinkler": True}).to_numpy(), [0.7, 0.3], rtol=RTOL)
    bn = examples.asia()
    ans = bn.query("Lung cancer", "Tuberculosis", event={"Visit to Asia": True, "Smoker": True})
    assert ans.index.names == ["Lung cancer", "Tuberculosis"]
    assert np.allclose(ans.to_numpy(), [0.855, 0.045, 0.095, 0.005], rtol=RTOL)
    assert np.allclose(bn.query("Lung cancer", event={"Visit to Asia": True, "Smoker": False}).to_numpy(),
                       [0.99, 0.01], rtol=RTOL)
    bn = examples.alarm()
    ans = bn.query("John calls", "Mary calls", event={"Burglary": True, "Earthquake": False})
    assert np.allclose(ans.to_numpy(), [0.08463, 0.06637, 0.25677, 0.59223], rtol=1e-5)
    # BASELINE.json configs[0]
    ans = bn.query("Burglary", event={"John calls": True, "Mary calls": True})
    assert np.allclose(ans.to_numpy(), [0.715828, 0.284172], atol=1e-6)
    bn = examples.grades()
    ans = bn.query("Letter", "SAT", event={"Intelligence": "Smart"})
    assert np.allclose(ans.to_numpy(), [0.153544, 0.614176, 0.046456, 0.185824], atol=1e-6)


def test_independent_variables_and_no_evidence():
    # reference test_indep_vars (test_bayes_net.py:121-165)
    from sorobn_b200 import BayesNet

    bn = BayesNet("A", "B")
    bn.P["A"] = pd.Series({1: 0.2, 2: 0.3, 3: 0.5})
    bn.P["B"] = pd.Series({1: 0.4, 2: 0.2, 3: 0.4})
    bn.prepare()
    for b in (1, 2, 3):
        ans = bn.query("A", event={"B": b})
        assert ans.index.tolist() == [1, 2, 3]
        assert np.allclose(ans.to_numpy(), [0.2, 0.3, 0.5], rtol=RTOL)
    assert np.allclose(bn.query("A", event={}).to_numpy(), [0.2, 0.3, 0.5], rtol=RTOL)
    many = bn.query_many("B", events=pd.DataFrame({"A": [1, 3, 2, 1, 1]}))
    assert np.allclose(many.to_numpy(), np.tile([0.4, 0.2, 0.4], (5, 1)), rtol=RTOL)


def test_cpt_forms_and_impute():
    # reference test_cpt_with_index_names / test_cpt_dataframe (test_bayes_net.py:168-233)
    from sorobn_b200 import BayesNet, examples

    bn = BayesNet(("A", "C"), ("B", "C"))
    bn.P["A"] = pd.Series({True: 0.7, False: 0.3})
    bn.P["B"] = pd.Series({True: 0.4, False: 0.6})
    pc = pd.DataFrame({
        "B": [True, True, True, True, False, False, False, False],
        "A": [True, True, False, False, True, True, False, False],
        "C": [True, False, True, False, True, False, True, False],
        "p": [1, 0, 0, 1, 0.5, 0.5, 0.001, 0.999],
    })
    bn.P["C"] = pc.set_index(["B", "A", "C"])["p"]
    bn.prepare()
    pd.testing.assert_series_equal(
        bn.query("C", event={"B": False, "A": True}),
        pd.Series([0.5, 0.5], name="P(C)", index=pd.Index([False, True], name="C")),
        rtol=RTOL,
    )
    # impute (bayes_net.py:877-908)
    bn = examples.asia()
    sample = {"Smoker": True, "Dispnea": True, "Lung cancer": None, "Bronchitis": None}
    filled = bn.impute(sample)
    post = bn.query("Lung cancer", "Bronchitis", event={"Smoker": True, "Dispnea": True})
    best = post.idxmax()
    assert filled["Bronchitis"] == best[0] and filled["Lung cancer"] == best[1]
    assert filled["Smoker"] is True or filled["Smoker"] == True  # noqa: E712


def test_impossible_and_unknown_evidence():
    from sorobn_b200 import examples

    bn = examples.asia()
    # P(TB or cancer = False, Lung cancer = True) == 0: the reference returns an empty Series
    ans = bn.query("Smoker", event={"TB or cancer": False, "Lung cancer": True})
    assert len(ans) == 0
    ans = bn.query("Smoker", event={"Dispnea": "maybe"})
    assert len(ans) == 0
    many = bn.query_many("Smoker", events=pd.DataFrame({"TB or cancer": [False, True], "Lung cancer": [True, True]}))
    assert np.isnan(many.iloc[0]).all() and np.isclose(many.iloc[1].sum(), 1.0)


@pytest.mark.parametrize("n_rows", [1, 3, 4, 5, 31, 32, 33, 511, 512, 513, 1027])
def test_ragged_batch_sizes(n_rows):
    """Row counts around the float4 / warp / CTA boundaries."""
    from oracle import ve_oracle
    from sorobn_b200 import workloads

    wl = workloads.asia_1m()
    bn = wl.build()
    events = wl.events(n_rows, seed=n_rows, bn=bn)
    got = bn.query_many(*wl.query, events=events).to_numpy()
    net = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    cache = {}
    for b in range(n_rows):
        key = tuple(events.iloc[b])
        if key not in cache:
            cache[key] = ve_oracle.query(net, *wl.query, event=dict(zip(wl.evidence, key)))[1].reshape(-1)
        assert rel_err(got[b], cache[key]) < RTOL


def test_random_networks_batched_vs_oracle():
    """Random DAGs with mixed cardinalities, random query / evidence sets."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet, synthetic

    rng = np.random.default_rng(2024)
    worst = 0.0
    for trial in range(12):
        n = int(rng.integers(4, 14))
        spec = synthetic.random_dag(n, 3, int(rng.integers(2, 5)), seed=100 + trial)
        bn = synthetic.load(spec, BayesNet)
        net = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
        perm = rng.permutation(n)
        nq = int(rng.integers(1, 3))
        ne = int(rng.integers(0, n - nq))
        query = [spec.nodes[i] for i in perm[:nq]]
        evs = [spec.nodes[i] for i in perm[nq:nq + ne]]
        B = 70
        events = synthetic.random_events(spec, evs, B, seed=trial)
        if not evs:
            events = pd.DataFrame(index=range(B))
        got = bn.query_many(*query, events=events).to_numpy()
        assert got.shape[0] == B
        for b in range(0, B, 7):
            ev = {v: int(events[v].iloc[b]) for v in evs}
            want = ve_oracle.query(net, *query, event=ev)[1].reshape(-1)
            worst = max(worst, rel_err(got[b], want))
    assert worst < RTOL, worst


@pytest.mark.parametrize("cards", [2, 3, 4, 5, 6, 7, 8, (2, 5, 3), (8, 2, 4, 3), (5, 7)])
def test_tiled_and_plain_kernels_agree_with_oracle(cards):
    """Every tile edge of sbn_step_tiled (2..5, with partial tiles for 6, 7, 8 states) and
    the plain sbn_step_batched kernel, on the same programs, against the oracle."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet, engine, planner, synthetic

    import zlib

    rng = np.random.default_rng(zlib.crc32(str(cards).encode()))  # stable across processes, unlike hash()
    worst = 0.0
    for trial in range(3):
        spec = synthetic.random_dag(14, 3, cards, seed=40 + trial, window=5)
        bn = synthetic.load(spec, BayesNet)
        net = bn._compiled
        dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
        perm = rng.permutation(14)
        query = [spec.nodes[i] for i in perm[:1 + trial % 2]]
        evs = [spec.nodes[i] for i in perm[2:2 + 3 + trial]]
        plan = planner.build_plan(net, [net.index[q] for q in query], [net.index[e] for e in evs])
        B = 301
        events = synthetic.random_events(spec, evs, B, seed=trial)
        codes = np.stack([events[v].to_numpy().astype(np.uint8) for v in evs])
        prog = engine.Program(plan)
        tiled = prog.run(codes, B).copy()
        prog.set_tiled(False)
        plain = prog.run(codes, B).copy()
        assert np.allclose(tiled, plain, rtol=5e-6, atol=1e-30)
        order = [net.names[v] for v in plan.order]
        for b in range(0, B, 29):
            ev = {v: int(events[v].iloc[b]) for v in evs}
            want = ve_oracle.query(dn, *query, event=ev, order=order)[1].reshape(-1)
            worst = max(worst, rel_err(tiled[:, b], want), rel_err(plain[:, b], want))
    assert worst < RTOL, worst


def test_full_size_grid_properties():
    """BASELINE.json configs[2] at full size (10x10 grid, 5 states, 100k rows):
    size-independent properties + an oracle sample."""
    from oracle import ve_oracle
    from sorobn_b200 import planner, workloads
    from sorobn_b200 import engine

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    B = 100_000
    codes = wl.codes(bn, B, seed=5)
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    prog = engine.Program(plan)
    out = prog.run(codes, B)
    assert out.shape == (5, B)
    assert np.isfinite(out).all() and (out >= 0).all()
    # every posterior sums to one
    assert np.allclose(out.sum(axis=0), 1.0, atol=2e-6)
    # determinism: same call, same bits
    again = prog.run(codes, B)
    assert np.array_equal(out, again)
    # permutation equivariance: shuffled evidence rows give shuffled posteriors (bitwise)
    perm = np.random.default_rng(0).permutation(B)
    shuffled = prog.run(np.ascontiguousarray(codes[:, perm]), B)
    assert np.array_equal(shuffled, out[:, perm])
    # chunking invariance: the batch run as 4096-row pieces (the last one partial) agrees bitwise.  (A
    # reservation alone does not chunk: a run grows it to the batch when device memory allows.)
    small = engine.Program(plan)
    pieces = [small.run(np.ascontiguousarray(codes[:, lo:lo + 4096]), min(4096, B - lo)) for lo in range(0, B, 4096)]
    assert np.array_equal(np.concatenate(pieces, axis=1), out)
    # oracle on a sample of rows
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    worst = 0.0
    for b in range(0, B, B // 16):
        ev = {v: int(net.domains[net.index[v]][codes[i, b]]) for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        worst = max(worst, rel_err(out[:, b], want))
    assert worst < RTOL, worst


def test_device_pointer_api_matches_host_api():
    """sbn_program_run_device on caller-owned device buffers (torch as the allocator)."""
    import torch

    from sorobn_b200 import engine, planner, workloads

    wl = workloads.asia_1m()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    prog = engine.Program(plan)
    B = 10_007
    codes = wl.codes(bn, B, seed=3)
    want = prog.run(codes, B)
    d_ev = torch.from_numpy(codes).cuda()
    d_out = torch.full((prog.Q, B), -1.0, dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for use_graph in (True, False, True):
        prog.set_graph(use_graph)
        d_out.fill_(-1.0)
        prog.run_device(d_ev.data_ptr(), B, B, d_out.data_ptr(), B, stream)
        torch.cuda.synchronize()
        assert np.array_equal(d_out.cpu().numpy(), want)
    info = prog.info()
    assert info["launches"] > 0 and info["Q"] == 2 and info["n_ev"] == 4


def test_single_queries_run_in_float64():
    """`query()` programs are float64 on the device: reference-grade precision (1e-12 here,
    against 1e-6 for the float32 batch path) on every example golden."""
    golden = load_golden("asia")
    bn = build_network(golden)
    worst = 0.0
    for case in golden["cases"][::7]:
        ans = bn.query(*case["query"], event=case_event(case))
        if case["values"]:
            worst = max(worst, rel_err(ans.to_numpy(), case["values"]))
    assert worst < 1e-12, worst


def test_extremely_unlikely_evidence_is_rescued_in_float64():
    """A 120-node chain observed at 119 nodes with near-deterministic CPTs: the evidence has
    probability ~1e-240, far below float32.  The float32 batch flags the row (normaliser <
    1e-24) and query_many settles it with the float64 program; the reference (float64) and
    the oracle agree with the result."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet

    n = 120
    names = [f"c{k:03d}" for k in range(n)]
    bn = BayesNet(*[(names[k - 1], names[k]) for k in range(1, n)])
    bn.P[names[0]] = pd.Series({0: 0.5, 1: 0.5})
    for k in range(1, n):
        bn.P[names[k]] = pd.DataFrame({names[k - 1]: [0, 0, 1, 1], names[k]: [0, 1, 0, 1],
                                       "p": [0.99, 0.01, 0.02, 0.98]})
    bn.prepare()
    # alternate the observed states: every transition is the unlikely one
    ev_vars = names[1:]
    rows = pd.DataFrame([[k % 2 for k in range(1, n)], [0] * (n - 1)], columns=ev_vars)
    got = bn.query_many(names[0], events=rows).to_numpy()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for b in range(2):
        ev = {v: int(rows[v].iloc[b]) for v in ev_vars}
        want = ve_oracle.query(dn, names[0], event=ev)[1].reshape(-1)
        assert np.isfinite(got[b]).all()
        # row 0 (P(event) ~ 1e-240) was settled in float64, row 1 stayed in float32
        assert rel_err(got[b], want) < (1e-9 if b == 0 else RTOL), (b, got[b], want)
    single = bn.query(names[0], event={v: int(rows[v].iloc[0]) for v in ev_vars})
    assert rel_err(single.to_numpy(), ve_oracle.query(dn, names[0], event={v: int(rows[v].iloc[0]) for v in ev_vars})[1]) < 1e-12


def test_tiny_posterior_entry_next_to_a_representable_normaliser_is_rescued():
    """The float32 range check is per ENTRY (VERDICT r1): P(event) ~ 1e-28 is above the 1e-30
    threshold on the normaliser, but the un-normalised entry of the unlikely query state is
    ~4e-40 (a float32 denormal: two or three digits).  The row must be flagged and settled in
    float64 so that EVERY posterior entry -- also the one at ~4e-12 -- is within 1e-6 relative."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet

    evs = ["E1", "E2", "E3", "E4"]
    bn = BayesNet(("Q", evs))
    bn.P["Q"] = pd.Series({0: 1.0 - 1e-13, 1: 1e-13})
    for e in evs:
        bn.P[e] = pd.DataFrame({"Q": [0, 0, 1, 1], e: [0, 1, 0, 1], "p": [1 - 1e-7, 1e-7, 1 - 2.5e-7, 2.5e-7]})
    bn.prepare()
    rows = pd.DataFrame([[1, 1, 1, 1], [0, 0, 0, 0], [1, 1, 0, 0]], columns=evs)
    got = bn.query_many("Q", events=rows).to_numpy()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    for b in range(len(rows)):
        ev = {v: int(rows[v].iloc[b]) for v in evs}
        want = ve_oracle.query(dn, "Q", event=ev)[1].reshape(-1)
        assert (want > 0).all() and np.isfinite(got[b]).all()
        assert np.max(np.abs(got[b] - want) / want) < RTOL, (b, got[b], want)
    # the raw float32 program really flags row 0 (normaliser 1e-28 >= 1e-30, entry 4e-40 < 1e-30)
    plan, program = bn._plan(("Q",), tuple(evs), 1)
    codes = np.ascontiguousarray(rows.to_numpy().T.astype(np.uint8))
    raw = program.run(codes, len(rows))
    assert np.isnan(raw[:, 0]).all() and np.isfinite(raw[:, 1]).all()


def test_graph_branches_match_linear_replay_and_plain_launches():
    """The branched CUDA graph (independent elimination sub-trees in parallel, slot-reuse
    hazards as edges) must give bitwise the same posteriors as the linear graph and as
    plain launches, repeatedly (a missing edge would show up as a race)."""
    from sorobn_b200 import engine, planner, workloads

    for wl, B in ((workloads.grid10x10(), 20_000), (workloads.dag50(), 5_000), (workloads.asia_1m(), 50_000)):
        bn = wl.build()
        net = bn._compiled
        plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
        prog = engine.Program(plan)
        prog.set_tiled(10)  # the branched capture issues one launch per step: compare like with like (no paired steps)
        codes = wl.codes(bn, B, seed=21)
        prog.set_graph(0)
        want = prog.run(codes, B).copy()
        assert np.isfinite(want).all()
        for mode in (1, 3, 1):
            prog.set_graph(mode)
            for _ in range(3):
                assert np.array_equal(prog.run(codes, B), want), (wl.name, mode)


def test_merged_sum_outs_match_unmerged_program_on_device():
    """Launches that sum out several variables at once (joint-state offset tables) against
    the one-variable-per-launch program, on the benchmark grid and a random DAG."""
    from sorobn_b200 import BayesNet, engine, planner, synthetic, workloads

    wl = workloads.grid10x10()
    cases = [(wl.build(), wl.query, wl.evidence, None)]
    spec = synthetic.random_dag(16, 3, (3, 4, 2), seed=77, window=6)
    cases.append((synthetic.load(spec, BayesNet), (spec.nodes[-1],), tuple(spec.nodes[2:12:3]), spec))
    for bn, query, evidence, spec in cases:
        net = bn._compiled
        q, e = [net.index[v] for v in query], [net.index[v] for v in evidence]
        merged = planner.build_plan(net, q, e, merge_sum_outs=True)
        plain = planner.build_plan(net, q, e, merge_sum_outs=False)
        B = 4099
        if spec is None:
            codes = wl.codes(bn, B, seed=8)
        else:
            ev = synthetic.random_events(spec, list(evidence), B, seed=8)
            codes = np.stack([ev[v].to_numpy().astype(np.uint8) for v in evidence])
        a = engine.Program(merged).run(codes, B)
        b = engine.Program(plain).run(codes, B)
        assert np.isfinite(a).all()
        assert np.allclose(a, b, rtol=2e-6, atol=1e-30)
        # single-event float64 programs use the same merged plan
        fm = planner.build_plan(net, q, e, mode=planner.MODE_FLAT, merge_sum_outs=True)
        fp = planner.build_plan(net, q, e, mode=planner.MODE_FLAT, merge_sum_outs=False)
        one = np.ascontiguousarray(codes[:, :1])
        assert np.allclose(engine.Program(fm, f64=True).run(one, 1), engine.Program(fp, f64=True).run(one, 1), rtol=1e-12)


def test_slab_variant_matches_plain_tile_walk():
    """Expanding products (both batched operands have private axes) run through the
    shared-memory slab variant; with it switched off (mode 5) the same program must give the
    same posteriors to float32 rounding, and both must match the oracle."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet, engine, planner, synthetic, workloads

    wl = workloads.grid10x10()
    jobs = [(wl.build(), wl.query, wl.evidence, None, 6000)]
    for cards, seed in ((4, 5), (3, 6), ((2, 5, 3), 7)):
        spec = synthetic.grid(5, 5, cards if isinstance(cards, int) else 3, seed=seed)
        jobs.append((synthetic.load(spec, BayesNet), (spec.nodes[-1],), tuple(spec.nodes[1:9:4]), spec, 900))
    for bn, query, evidence, spec, B in jobs:
        net = bn._compiled
        plan = planner.build_plan(net, [net.index[q] for q in query], [net.index[e] for e in evidence])
        if spec is None:
            codes = wl.codes(bn, B, seed=31)
        else:
            ev = synthetic.random_events(spec, list(evidence), B, seed=31)
            codes = np.stack([ev[v].to_numpy().astype(np.uint8) for v in evidence])
        prog = engine.Program(plan)
        with_slab = prog.run(codes, B).copy()
        prog.set_tiled(5)
        without = prog.run(codes, B).copy()
        assert np.isfinite(with_slab).all()
        assert np.allclose(with_slab, without, rtol=2e-6, atol=1e-30)
        dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
        order = [net.names[v] for v in plan.order]
        for b in range(0, B, B // 7):
            evd = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(evidence)}
            want = ve_oracle.query(dn, *query, event=evd, order=order)[1].reshape(-1)
            assert rel_err(with_slab[:, b], want) < RTOL


@pytest.mark.parametrize("name", golden_names(kinds=("predict_proba",)))
def test_predict_proba_matches_reference(name):
    """Row likelihoods on the device (normaliser of an elimination with the row as evidence,
    no query variable) against the reference's predict_proba on its example networks."""
    from sorobn_b200 import examples

    golden = load_golden(name)
    bn = examples.build(examples.NETWORKS[golden["network"]])
    worst = 0.0
    for case in golden["cases"]:
        X = pd.DataFrame(case["rows"], columns=case["columns"])
        got = bn.predict_proba(X)
        assert list(got.index.names) == sorted(case["columns"])
        worst = max(worst, rel_err(got.to_numpy(), case["prob"]))
        row = dict(zip(case["columns"], case["rows"][0]))
        assert abs(bn.predict_proba(row) - case["prob"][0]) <= RTOL * case["prob"][0]
    assert worst < RTOL, worst
    # log-likelihood and the joint itself
    X = pd.DataFrame(golden["cases"][0]["rows"], columns=golden["cases"][0]["columns"])
    assert np.allclose(bn.predict_log_proba(X).to_numpy(), np.log(golden["cases"][0]["prob"]), rtol=1e-5, atol=1e-6)
    fjd = bn.full_joint_dist()
    assert np.isclose(fjd.sum(), 1.0) and len(fjd) == len(golden["cases"][0]["rows"])
    assert np.allclose(np.sort(fjd.to_numpy()), np.sort(golden["cases"][0]["prob"]), rtol=1e-9)


def test_predict_proba_order_and_zero_rows():
    # reference test_predict_proba_order_doesnt_matter (test_bayes_net.py:340-354)
    import itertools
    import math

    from sorobn_b200 import examples

    bn = examples.alarm()
    event = {"Alarm": False, "Burglary": False, "Earthquake": True, "John calls": False, "Mary calls": False}
    base = bn.predict_proba(event)
    for order in list(itertools.permutations(event))[:24]:
        assert math.isclose(bn.predict_proba({v: event[v] for v in order}), base, rel_tol=1e-6)
    # a combination the reference's joint does not contain (probability zero) gives 0.0
    asia = examples.asia()
    assert asia.predict_proba({"TB or cancer": False, "Lung cancer": True}) == 0.0
    many = asia.predict_proba(pd.DataFrame({"TB or cancer": [False, True], "Lung cancer": [True, True]}))
    assert many.iloc[0] == 0.0 and many.iloc[1] > 0


def test_batch_of_unlikely_rows_goes_through_the_batched_float64_program():
    """Most variables observed on a 60-node chain: every row has P(event) around 1e-40..1e-60,
    below the float32 threshold, so query_many / predict_proba re-run the whole batch with the
    batched float64 program (plain kernel in double).  Answers match the oracle to 1e-9."""
    from oracle import ve_oracle
    from sorobn_b200 import BayesNet, engine, planner

    n = 60
    names = [f"h{k:02d}" for k in range(n)]
    bn = BayesNet(*[(names[k - 1], names[k]) for k in range(1, n)])
    rng = np.random.default_rng(5)
    bn.P[names[0]] = pd.Series({0: 0.3, 1: 0.3, 2: 0.4})
    for k in range(1, n):
        t = rng.dirichlet(np.ones(3) * 0.3, size=3)
        bn.P[names[k]] = pd.DataFrame([(a, b, t[a, b]) for a in range(3) for b in range(3)], columns=[names[k - 1], names[k], "p"])
    bn.prepare()
    ev_vars = names[1:]
    B = 40
    rows = pd.DataFrame(rng.integers(0, 3, size=(B, n - 1)), columns=ev_vars)
    got = bn.query_many(names[0], events=rows).to_numpy()
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    lik = bn.predict_proba(rows).to_numpy()
    assert (lik < 1e-25).all() and (lik > 0).all()
    for b in range(0, B, 3):
        ev = {v: int(rows[v].iloc[b]) for v in ev_vars}
        want = ve_oracle.query(dn, names[0], event=ev)[1].reshape(-1)
        assert rel_err(got[b], want) < 1e-9
        assert abs(lik[b] - ve_oracle.evidence_probability(dn, ev)) <= 1e-9 * lik[b]
    # the float32 program does flag these rows (that is what routed them to float64)
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[names[0]]], [net.index[v] for v in ev_vars])
    codes = np.stack([rows[v].to_numpy().astype(np.uint8) for v in ev_vars])
    assert np.isnan(engine.Program(plan).run(codes, B)).all()
    assert np.isfinite(engine.Program(plan, f64=True).run(codes, B)).all()


def test_impute_many_agrees_with_row_by_row_impute():
    from sorobn_b200 import examples

    bn = examples.asia(seed=2)
    full = bn.sample(40)
    holes = full.astype(object).copy()
    rng = np.random.default_rng(0)
    for i in range(len(holes)):
        for c in rng.choice(holes.columns, size=rng.integers(0, 4), replace=False):
            holes.loc[i, c] = None
    filled = bn.impute_many(holes)
    assert not filled.isna().any().any() and list(filled.columns) == list(holes.columns)
    for i in range(len(holes)):
        row = {c: (None if pd.isna(holes.loc[i, c]) else holes.loc[i, c]) for c in holes.columns}
        if all(v is not None for v in row.values()):
            assert (filled.loc[i] == full.loc[i]).all()
            continue
        want = bn.impute(row)
        for c in holes.columns:
            assert filled.loc[i, c] == want[c], (i, c)


def test_sliced_staging_of_big_cpts_matches_the_oracle():
    """dag50 has 8^5-entry CPTs (128 KB): the planner lays them out for their consumer and the
    tiled kernel stages, per chunk of tiles, only the slice those tiles touch.  Against the oracle,
    and against the plain kernel that gathers the same tables from L1/L2."""
    from oracle import ve_oracle
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.dag50()
    bn = wl.build()
    net = bn._compiled
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    assert any(sum(net.cpt[plan.tables[f.buf]].size for f, _, _ in st.inputs if not f.is_slot) * 4 > planner.SLICE_MIN_BYTES
               for st in plan.steps if st.kind == planner.KIND_BATCHED)
    B = 2_000
    codes = wl.codes(bn, B, seed=31)
    prog = engine.Program(plan)
    tiled = prog.run(codes, B).copy()
    prog.set_tiled(False)
    plain = prog.run(codes, B).copy()
    assert np.allclose(tiled, plain, rtol=5e-6, atol=1e-30)
    order = [net.names[v] for v in plan.order]
    worst = 0.0
    for b in range(0, B, 211):
        ev = {v: net.domains[net.index[v]][int(codes[k, b])] for k, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        worst = max(worst, rel_err(tiled[:, b], want))
    assert worst < RTOL, worst


@pytest.mark.parametrize("name", golden_names(("impute",)))
def test_impute_matches_reference_goldens(name):
    """`impute` (bayes_net.py:877-908) pinned to the reference's own results (2-3 missing values
    per sample), one sample at a time and as one `impute_many` batch (mixed missing patterns)."""
    from sorobn_b200 import examples

    golden = load_golden(name)
    bn = examples.build(examples.NETWORKS[golden["network"]])
    rows = []
    for case in golden["cases"]:
        sample = {k: v for k, v in case["sample"]}
        want = {k: v for k, v in case["filled"]}
        got = bn.impute(dict(sample))
        assert {k: got[k] for k in want} == want, (sample, dict(got), want)
        rows.append(sample)
    frame = pd.DataFrame(rows, dtype=object)
    filled = bn.impute_many(frame)
    for b, case in enumerate(golden["cases"]):
        want = {k: v for k, v in case["filled"]}
        assert {k: filled[k].iloc[b] for k in want} == want, (b, filled.iloc[b].to_dict(), want)


def test_query_many_over_a_device_list_equals_the_single_device_answer():
    """`query_many(devices=[...])` shards the rows over the listed GPUs from one process (one
    thread and one program per device); with every visible device it must return exactly what
    the default single-device call returns -- ragged shards, float64 rescue included."""
    from sorobn_b200 import engine, workloads

    wl = workloads.asia_1m()
    bn = wl.build()
    events = wl.events(10_007, seed=3, bn=bn)
    want = bn.query_many(*wl.query, events=events)
    n_dev = engine.device_count()
    for devices in ([0], list(range(n_dev)), [0] * 3):  # the same GPU three times: three programs, three threads
        got = bn.query_many(*wl.query, events=events, devices=devices)
        pd.testing.assert_frame_equal(got, want, check_exact=True)


def test_program_chunk_capacity_grows_with_the_batch():
    """A cached program first used for ONE row must not answer a later large batch one row at a
    time (ADVICE r1): the reservation follows the largest batch seen."""
    from sorobn_b200 import workloads

    wl = workloads.asia_1m()
    bn = wl.build()
    events = wl.events(50_000, seed=5, bn=bn)
    first = bn.query_many(*wl.query, events=events.iloc[:1])
    _, program = bn._plan(wl.query, tuple(events.columns), 1)
    assert program.info()["reserved_rows"] >= 1
    full = bn.query_many(*wl.query, events=events)
    assert program.info()["reserved_rows"] >= 50_000
    assert np.array_equal(full.iloc[:1].to_numpy(), first.to_numpy())
    launches = program.info()["launches"]
    bn.query_many(*wl.query, events=events)
    per_call = program.info()["launches"] - launches
    assert per_call <= 4, per_call  # one chunk: a couple of launches, not 50,000 rounds


@pytest.mark.parametrize("workload,rows", [("grid10x10", 4099), ("asia_1m", 10_001), ("dag50", 3001)])
def test_on_chip_segments_match_classic_launches_and_the_oracle(workload, rows):
    """The segment kernel (csrc/sbn_chain.cu: runs of steps executed on chip for 32 rows at a time,
    intermediates in shared memory / L2-resident scratch, fused normalisation) against the classic
    one-launch-per-step path on the same program, at a ragged row count (partial row block, more
    row blocks than CTAs), and against the oracle on a sample of rows."""
    from oracle import ve_oracle
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.WORKLOADS[workload]()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    codes = wl.codes(bn, rows, seed=21)
    prog = engine.Program(plan)
    assert prog.info()["segments"] == 0  # opt-in: the default is one launch per step
    prog.set_tiled(7)
    info = prog.info()
    if workload == "grid10x10":
        assert info["segments"] >= 1 and info["segment_steps"] >= 40 and info["segment_hbm_bytes_per_row"] == 0, info
    chained = prog.run(codes, rows).copy()
    again = prog.run(codes, rows)
    # (not bitwise: a step with few tiles and many eliminated states splits them over warps whose
    # partial sums meet through atomic adds, in arrival order)
    assert np.allclose(chained, again, rtol=1e-6, atol=1e-30)
    prog.set_tiled(6)
    assert prog.info()["segments"] == 0
    classic = prog.run(codes, rows)
    assert np.isfinite(classic).all()
    assert np.allclose(chained, classic, rtol=3e-6, atol=1e-30)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    for b in list(range(0, rows, max(1, rows // 7))) + [rows - 1]:
        ev = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        assert rel_err(chained[:, b], want) < RTOL, (b, chained[:, b], want)
    # P(event) per row comes out of the fused normalisation too
    prog.set_tiled(7)
    p_chain = prog.evidence(codes, rows)
    prog.set_tiled(6)
    p_classic = prog.evidence(codes, rows)
    assert np.allclose(p_chain, p_classic, rtol=3e-6, atol=0)


def test_pipelined_host_path_equals_the_device_path():
    """`sbn_program_run_host` pipelines transfer-bound programs (Asia: one batched launch for
    megabytes of codes and posteriors): column ranges on three streams.  The answer must be
    bitwise the one of a single device-resident run, also for a ragged row count."""
    import torch

    from sorobn_b200 import engine, planner, workloads

    wl = workloads.asia_1m()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    prog = engine.Program(plan)
    rows = 400_003
    codes = wl.codes(bn, rows, seed=9)
    host = prog.run(codes, rows)  # >= 4 x 32768 rows and >= 2 MB of copies: pipelined
    d_ev = torch.from_numpy(codes).cuda()
    d_out = torch.empty((prog.Q, rows), dtype=torch.float32, device="cuda")
    prog.run_device(d_ev.data_ptr(), rows, rows, d_out.data_ptr(), rows, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert np.array_equal(host, d_out.cpu().numpy())
    assert np.allclose(host.sum(axis=0), 1.0, atol=1e-5)
    again = prog.run(codes, rows)
    assert np.array_equal(host, again)
    small = prog.run(np.ascontiguousarray(codes[:, :1000]), 1000)  # below the threshold: single-stream path
    assert np.array_equal(small, host[:, :1000])


@pytest.mark.parametrize("workload,rows", [("grid10x10", 5003), ("dag50", 2049)])
def test_tensor_map_tma_kernel_matches_the_default_kernels(workload, rows):
    """`sbn_step_tma` (csrc/sbn_tma.cu: the batched operands of a tile arrive as cp.async.bulk.tensor
    boxes in a shared-memory ring, producer warp + four consumer warps, persistent CTAs) against the
    register-preload kernels on the same program, at a ragged row count (the last row block's boxes
    reach past `ld`: zero-filled by the tensor map), and against the oracle on a sample of rows."""
    from oracle import ve_oracle
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.WORKLOADS[workload]()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    codes = wl.codes(bn, rows, seed=23)
    prog = engine.Program(plan)
    default = prog.run(codes, rows).copy()
    prog.set_tiled(9)
    tma = prog.run(codes, rows).copy()
    assert np.array_equal(tma, prog.run(codes, rows))  # deterministic
    assert np.allclose(tma, default, rtol=3e-6, atol=1e-30)
    if workload == "grid10x10":
        assert not np.array_equal(tma, default)  # the other kernel really ran (different rounding order)
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    for b in (0, rows // 3, rows - 1):
        ev = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        assert rel_err(tma[:, b], want) < RTOL, (b, tma[:, b], want)


@pytest.mark.parametrize("workload,rows", [("grid10x10", 5003), ("grid10x10", 257), ("dag50", 2049), ("asia_1m", 3001)])
def test_paired_steps_match_single_step_launches_and_the_oracle(workload, rows):
    """`sbn_pair_kernel` (csrc/sbn_pair.cu: a step and its consumer as ONE launch, the intermediate
    factor in registers, the tables of both steps pre-multiplied into canonical coefficient arrays)
    against one launch per step on the same program, at a ragged row count, and against the oracle
    on a sample of rows."""
    from oracle import ve_oracle
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.WORKLOADS[workload]()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    codes = wl.codes(bn, rows, seed=29)
    prog = engine.Program(plan)
    prog.set_graph(False)

    def run():
        before = prog.info()["launches"]
        out = prog.run(codes, rows).copy()
        return out, prog.info()["launches"] - before

    paired, n_paired = run()
    assert np.array_equal(paired, run()[0])  # deterministic
    prog.set_tiled(10)
    single, n_single = run()
    prog.set_tiled(11)
    assert np.isfinite(single).all()
    assert np.allclose(paired, single, rtol=3e-6, atol=1e-30)
    assert prog.info()["pairs"] == n_single - n_paired and prog.info()["pair_bytes_saved_per_row"] >= 8 * prog.info()["pairs"]
    if workload == "grid10x10":
        assert n_single - n_paired >= 8, (n_single, n_paired)  # the frontier chains of the grid pair up
        # ... and the expanding product 3125 <- B625 x B625 runs inside its consumer: 25,000 B per row on its own
        assert prog.info()["pair_bytes_saved_per_row"] >= 8 * 3125 + 7 * 8 * 625, prog.info()
        assert not np.array_equal(paired, single)
    prog.set_graph(True)
    assert np.array_equal(prog.run(codes, rows), paired)  # the captured graph replays the same launches
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)
    order = [net.names[v] for v in plan.order]
    for b in sorted({0, rows // 3, rows // 2, rows - 1}):
        ev = {v: net.domains[net.index[v]][codes[i, b]] for i, v in enumerate(wl.evidence)}
        want = ve_oracle.query(dn, *wl.query, event=ev, order=order)[1].reshape(-1)
        assert rel_err(paired[:, b], want) < RTOL, (b, paired[:, b], want)
    p_pair = prog.evidence(codes, rows)
    prog.set_tiled(10)
    assert np.allclose(p_pair, prog.evidence(codes, rows), rtol=3e-6, atol=0)


def test_step_roles_and_the_fallback_when_offsets_do_not_fit_32_bits(monkeypatch):
    """`sbn_program_step_roles` names how each step runs; on the benchmark grid: pairs, one expanding
    product fused with its consumer, table steps hoisted to creation.  A program whose `entries x row
    pitch` exceeds the fused kernels' 32-bit element offsets must fall back to one launch per step
    (here forced with SOROBN_B200_PAIR_IDX_LIMIT) and give the numbers of `set_tiled(10)`."""
    from sorobn_b200 import engine, planner, workloads

    wl = workloads.grid10x10()
    bn = wl.build()
    net = bn._compiled
    plan = planner.build_plan(net, [net.index[q] for q in wl.query], [net.index[e] for e in wl.evidence])
    rows = 3001
    codes = wl.codes(bn, rows, seed=31)
    prog = engine.Program(plan)
    prog.set_graph(False)
    roles = prog.step_roles()
    kinds = np.array([st.kind for st in plan.steps])
    assert (roles[kinds == planner.KIND_FLAT] == 0).all() and (roles[kinds == planner.KIND_BATCHED] > 0).all()
    assert (roles == 2).sum() == (roles == 3).sum() >= 8 and (roles == 4).sum() == (roles == 5).sum() == 1
    firsts = np.flatnonzero((roles == 2) | (roles == 4))
    launched = np.flatnonzero(roles > 0)
    for i in firsts:  # the second step of a fused launch is the next launched step
        nxt = launched[np.searchsorted(launched, i) + 1]
        assert roles[nxt] == roles[i] + 1
    assert prog.info()["pairs"] == len(firsts)
    fused = prog.run(codes, rows).copy()
    before = prog.info()["launches"]
    prog.run(codes, rows)
    n_fused = prog.info()["launches"] - before

    monkeypatch.setenv("SOROBN_B200_PAIR_IDX_LIMIT", "1000")
    assert set(prog.step_roles().tolist()) == {0, 1}
    before = prog.info()["launches"]
    single = prog.run(codes, rows).copy()
    n_single = prog.info()["launches"] - before
    assert n_single == n_fused + len(firsts)
    monkeypatch.delenv("SOROBN_B200_PAIR_IDX_LIMIT")
    prog.set_tiled(10)
    assert np.array_equal(single, prog.run(codes, rows))
    assert np.allclose(fused, single, rtol=3e-6, atol=1e-30)
