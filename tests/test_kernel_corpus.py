"""The variant corpus (tests/kernel_corpus.py) through the planner and the CPU interpreter of the
device program, against the float64 oracle: corpus and generator mistakes show up without a GPU."""
import numpy as np
import pytest

import kernel_corpus
from oracle import program_interp, ve_oracle


@pytest.mark.parametrize("case", kernel_corpus.CASES, ids=kernel_corpus.case_id)
def test_variant_case_through_the_interpreter(case):
    spec, net, dn, plan, query, evidence = kernel_corpus.build(case)
    n = 40
    codes = kernel_corpus.evidence_rows(spec, evidence, n, seed=case["seed"])
    got = program_interp.run(plan.words, plan.table_blob64, codes, n_rows=n)
    order = [net.names[v] for v in plan.order]
    for b in range(n):
        ev = {v: int(codes[i, b]) for i, v in enumerate(evidence)}
        want = ve_oracle.query(dn, *query, event=ev, order=order)[1].reshape(-1)
        if np.isnan(want).all():
            assert np.isnan(got[:, b]).all()
            continue
        assert np.allclose(got[:, b], want, rtol=1e-12, atol=0), (b, got[:, b], want)


def test_corpus_reaches_the_shapes_it_is_meant_for():
    """Shapes the census cannot see, checked on the specs themselves."""
    specs = [(c, kernel_corpus.make_spec(c)) for c in kernel_corpus.CASES]
    card = lambda spec, ks: [spec.n_states[spec.nodes[k]] for k in ks]  # noqa: E731
    assert any(1 in card(s, c["query"]) for c, s in specs), "a query variable with one state"
    assert any(1 in card(s, c["evidence"]) for c, s in specs), "an evidence variable with one state"
    assert any(any(s.n_states[p] == 1 for p in s.parents.get(n, [])) for c, s in specs for n in s.nodes), \
        "a single-state parent"
    hidden_single = False
    for c in kernel_corpus.CASES:
        spec, net, _, plan, _, _ = kernel_corpus.build(c)
        hidden_single |= any(spec.n_states[net.names[v]] == 1 for v in plan.order)
    assert hidden_single, "a single-state hidden variable"
    assert any(c.get("zeros") for c, _ in specs), "structural zeros"
    for big in (9, 13, 37):
        assert any(big in s.n_states.values() for _, s in specs), big
    assert any(len(c["query"]) == 2 and np.prod(card(s, c["query"])) >= 400 for c, s in specs), "two query variables, Q >= 400"
    assert {4, 5} <= set().union(*[set(s.n_states.values()) for c, s in specs if c["gen"] == "grid"])


def test_grid_accepts_a_cardinality_sequence():
    from sorobn_b200 import synthetic

    a, b = synthetic.grid(3, 3, 4, seed=2), synthetic.grid(3, 3, [4], seed=2)
    assert synthetic.grid(3, 3, np.int64(4), seed=2).name == a.name == "grid3x3s4"
    assert a.nodes == b.nodes and all(np.array_equal(a.cpt[n], b.cpt[n]) for n in a.nodes)
    mixed = synthetic.grid(3, 3, [4, 5], seed=2)
    assert [mixed.n_states[n] for n in mixed.nodes] == [4, 5, 4, 5, 4, 5, 4, 5, 4]
    assert all(mixed.cpt[n].shape == (*[mixed.n_states[p] for p in mixed.parents.get(n, [])], mixed.n_states[n])
               for n in mixed.nodes)
