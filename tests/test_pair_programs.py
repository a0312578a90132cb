"""The hand-built programs of tests/pair_programs.py, on the CPU: the float64 interpreter of the words
equals a direct einsum of the same factor graph, and the words meet the pairing preconditions each
case is built for.  A GPU failure of tests/test_gpu_pair_programs.py is then a device bug, not a
builder bug."""
import numpy as np
import pytest

import pair_programs as pp
from oracle import program_interp

N_ROWS = 64


def _built(case):
    built = pp.build(case)
    codes = pp.evidence_rows(built, N_ROWS)
    return built, pp.unique_rows(codes)[0]


@pytest.mark.parametrize("case", pp.CASES, ids=pp.case_id)
def test_interpreter_equals_einsum(case):
    built, codes = _built(case)
    plan = built.plan
    got, totals = program_interp.run(plan.words, plan.table_blob64, codes, n_rows=codes.shape[1], return_totals=True)
    want, want_totals = pp.einsum_posterior(built, codes)
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.allclose(got, want, rtol=1e-12, atol=0, equal_nan=True)
    assert np.allclose(totals, want_totals, rtol=1e-12, atol=0)
    assert np.array_equal(plan.table_blob64, plan.table_blob.astype(np.float64))  # float32 values
    assert (plan.table_blob64 == 0).any()  # structural zeros
    if plan.evidence:
        assert (want_totals == 0).any() and (want_totals > 0).any()  # impossible rows beside possible ones
        # every column has codes at and above the largest card - 1, 255 included
        cards = pp.ev_cards(built)
        for k, c in enumerate(cards):
            assert (codes[k] == c - 1).any() and (codes[k] == c).any() and (codes[k] == 255).any()


@pytest.mark.parametrize("case", [c for c in pp.PAIR_CASES if c["census"] is not None or c["name"].startswith("smem")],
                         ids=pp.case_id)
def test_pair_preconditions_hold(case):
    plan = pp.build(case).plan
    conds = pp.pair_conditions(plan.words, *case["pair"], [s for _, s in plan.slots])
    assert all(conds.values()), conds


@pytest.mark.parametrize("case,broken", [("refuse_F_is_out2", "F apart from step 2's output"),
                                         ("refuse_out1_is_post", "step 1's output is not the posterior")])
def test_refusal_cases_break_exactly_one_precondition(case, broken):
    case = next(c for c in pp.PAIR_CASES if c["name"] == case)
    plan = pp.build(case).plan
    conds = pp.pair_conditions(plan.words, *case["pair"], [s for _, s in plan.slots])
    assert [k for k, v in conds.items() if not v] == [broken], conds


@pytest.mark.parametrize("case", pp.TRIPLE_CASES, ids=pp.case_id)
def test_triple_preconditions_hold(case):
    plan = pp.build(case).plan
    conds = pp.triple_conditions(plan.words, *case["pair"])
    assert all(conds.values()), conds


def test_cases_cover_every_mode_pair_and_triple_group():
    claimed = {c["census"] for c in pp.CASES if c["census"]}
    want = {f"pair ({m1},{m2})" for m1 in range(5) for m2 in range(3)} | {"triple group=1", "triple group=5"}
    assert want <= claimed, sorted(want - claimed)


def test_canonical_arrays_around_the_shared_memory_limit():
    """The two smem cases: B over one column (5 or 6 states) + CE over two (8 x 10), laid out as
    spec_step / size_canon do (B slab T x 8 + 4 floats, CE slab T^3), rounded up to 4 floats."""
    def floats(slab, n):
        return -(-slab * n // 4) * 4
    under = floats(pp.T * 8 + 4, 5) + floats(pp.T ** 3, 80)
    over = floats(pp.T * 8 + 4, 6) + floats(pp.T ** 3, 80)
    assert under * 4 <= pp.PAIR_SMEM_MAX < over * 4
    assert floats(pp.T ** 3, 80) * 4 <= pp.PAIR_SMEM_MAX  # each array alone fits: the total decides


def test_multi_chunk_rows():
    """The row count of the multi-chunk case gives tiles_per_cta > 1 and a partial last chunk."""
    for n_sms in (114, 132):
        n = pp.multi_chunk_rows(125, n_sms)
        n_rblocks = -(-n // pp.PAIR_ROWS)
        chunks = max(1, min(125, 8 * n_sms * 6 // n_rblocks))
        tpc = -(-125 // chunks)
        assert tpc > 1 and 125 % tpc, (n_sms, n, tpc)
