"""The host side of `BayesNet.joint_marginals_many` on the CPU: the device programs are replaced by the CPU replay
of their words (tests/joint_interp.py), and only the public entry point is driven.  Ground truth is
`ve_oracle.query` per row and group (test_joint_plan.oracle_group), and `expected_counts` of the same frame."""
import numpy as np
import pandas as pd
import pytest

import joint_interp
import soft_pattern_interp as spi
import soft_oracle
from interpreted_program import InterpretedProgram
from sorobn_b200 import engine, examples, workloads
from test_joint_plan import oracle_group


class JointProgram(InterpretedProgram):
    """InterpretedProgram with the joint call, and counts runs that take likelihoods."""

    def _lik(self, lik):
        return None if lik is None else np.asarray(lik.cpu().numpy() if hasattr(lik, "cpu") else lik, dtype=self.dtype)

    def joint(self, codes, n_rows, lik=None):
        self._start(n_rows)
        assert (lik is None) == (not self.plan.soft)
        out, prob, _ = joint_interp.run_joint(self.plan.words, self.blob, codes, lik=self._lik(lik), n_rows=n_rows,
                                              dtype=self.dtype, min_total=self._min_total())
        return out, prob

    def counts(self, codes, n_rows, lik=None, log_evidence=False):
        if lik is None:
            return super().counts(codes, n_rows)
        self._start(n_rows)
        c, prob, log_ev = spi.run_counts(self.plan.words, self.blob, codes, self._lik(lik), n_rows=n_rows,
                                         dtype=self.dtype, min_total=self._min_total())
        return (c, prob, log_ev) if log_evidence else (c, prob)


@pytest.fixture
def interpreted(monkeypatch):
    monkeypatch.setattr(InterpretedProgram, "live", [])
    monkeypatch.setattr(InterpretedProgram, "calls", [])
    monkeypatch.setattr(InterpretedProgram, "flag_below", None)
    monkeypatch.setattr(engine, "Program", JointProgram)
    return JointProgram


def frame(bn, n, seed, cols, frac=0.35):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed)
    out = {}
    for c in cols:
        vals = np.asarray(net.domains[net.index[c]], dtype=object)[codes[net.index[c]]].copy()
        vals[rng.random(n) < frac] = None
        out[c] = vals
    return pd.DataFrame(out, index=pd.RangeIndex(3, 3 + n, name="row"))


ASIA_COLS = ("Smoker", "Visit to Asia", "Positive X-ray", "Dispnea")


def check_against_oracle(bn, X, got, lik=None):
    net = bn._compiled
    dn = soft_oracle.dense(net)
    for entry, df in got.items():
        names = list(df.columns.names)
        assert df.index.equals(X.index)
        for b, (label, row) in enumerate(X.iterrows()):
            hard = {c: v for c, v in row.items() if v is not None and v == v}
            soft = {} if lik is None else {k: np.asarray(v)[b] for k, v in lik.items()}
            M = [n for n in names if n not in hard]
            vals = df.loc[label].to_numpy().reshape([len(net.domains[net.index[n]]) for n in names])
            if not M:
                want_arr = np.zeros_like(vals)
                want_arr[tuple(net.domains[net.index[n]].index(hard[n]) for n in names)] = 1.0
            else:
                want = oracle_group(net, dn, [net.index[n] for n in M], hard, soft)
                if np.isnan(want).all():
                    assert np.isnan(vals).all()
                    continue
                sub = want.reshape([len(net.domains[net.index[n]]) for n in reversed(M)]).transpose()
                want_arr = np.zeros_like(vals)
                index = tuple(net.domains[net.index[n]].index(hard[n]) if n in hard else slice(None) for n in names)
                want_arr[index] = sub
            assert np.allclose(vals, want_arr, rtol=1e-6, atol=1e-7), (entry, label, vals, want_arr)
            assert abs(vals.sum() - 1.0) < 1e-6


def test_families_match_the_oracle_and_sum_to_the_expected_counts(interpreted):
    bn = examples.asia()
    X = frame(bn, 25, 1, ASIA_COLS)
    got = bn.joint_marginals_many(X)
    assert list(got) == bn.nodes
    check_against_oracle(bn, X, got)
    counts = bn.expected_counts(X)
    for node, df in got.items():
        want = counts[node]
        summed = df.sum(axis=0)
        assert np.allclose(summed.to_numpy(), want.to_numpy(), rtol=1e-6, atol=1e-6), node
    # axes are [*parents, node], as the dense CPTs of cpt_tensors
    net = bn._compiled
    for v, node in enumerate(net.names):
        assert list(got[node].columns.names) == [net.names[u] for u in net.scope(v)]


def test_family_frames_sum_down_to_marginals_many(interpreted):
    bn = examples.asia()
    X = frame(bn, 12, 4, ("Smoker", "Positive X-ray"), frac=0.0)
    got = bn.joint_marginals_many(X, groups=["Lung cancer", "Dispnea"])
    net = bn._compiled
    for node in ("Lung cancer", "Dispnea"):
        dn = soft_oracle.dense(net)
        summed = got[node].T.groupby(level=node).sum().T
        for b, (label, row) in enumerate(X.iterrows()):
            want = oracle_group(net, dn, [net.index[node]], dict(row), {})
            assert np.allclose(summed.loc[label].to_numpy(), want, rtol=1e-6)


def test_observed_members_are_one_hot_and_groups_keep_their_order(interpreted):
    bn = examples.asia()
    X = frame(bn, 20, 2, ASIA_COLS, frac=0.5)
    groups = [("Dispnea", "Smoker"), ("Smoker", "Dispnea"), "Bronchitis", ("Positive X-ray",),
              ("Visit to Asia", "Lung cancer", "Smoker")]
    got = bn.joint_marginals_many(X, groups=groups)
    assert list(got) == groups
    assert list(got[("Dispnea", "Smoker")].columns.names) == ["Dispnea", "Smoker"]
    assert list(got[("Dispnea", "Smoker")].columns) == [(a, b) for a in (False, True) for b in (False, True)]
    check_against_oracle(bn, X, got)
    a, b = got[("Dispnea", "Smoker")], got[("Smoker", "Dispnea")]
    assert np.allclose(a.to_numpy(), b.T.reorder_levels(["Dispnea", "Smoker"]).sort_index().T.to_numpy())
    # a row that observes Smoker has all its mass on that state
    obs = X["Smoker"].notna()
    for label in X.index[obs]:
        row = got[("Visit to Asia", "Lung cancer", "Smoker")].loc[label]
        assert row.xs(not X.loc[label, "Smoker"], level="Smoker").sum() == 0.0


def test_soft_evidence_and_latent_nodes(interpreted):
    bn = examples.asia()
    X = frame(bn, 16, 3, ("Smoker", "Positive X-ray"))
    rng = np.random.default_rng(0)
    lik = {"Lung cancer": rng.random((16, 2)), "Dispnea": rng.random((16, 2)) * 1e-3}
    lik["Lung cancer"][5] = 0.0  # an impossible row
    got = bn.joint_marginals_many(X, groups=["TB or cancer", ("Lung cancer", "Bronchitis")], likelihoods=lik)
    check_against_oracle(bn, X, got, lik)
    for df in got.values():
        assert np.isnan(df.iloc[5]).all() and not np.isnan(df.drop(index=X.index[5])).any().any()


def test_impossible_rows_are_nan_everywhere(interpreted):
    bn2 = examples.sprinkler()
    node = bn2.nodes[-1]
    parents = bn2.parents.get(node, [])
    table = bn2.P[node].copy()
    table[:] = 0.0
    table.loc[table.index[::2]] = 1.0  # one state only per parent configuration: the others are impossible
    bn2.P[node] = table
    bn2.prepare()
    net2 = bn2._compiled
    v = net2.index[node]
    X = pd.DataFrame({node: [net2.domains[v][0], net2.domains[v][1], None]}, index=[7, 8, 9])
    got = bn2.joint_marginals_many(X, groups=[node, parents[0] if parents else node])
    impossible = [i for i, val in enumerate(X[node]) if val is not None and not bn2.joint_marginals_many(
        X.iloc[[i]]).get(node).notna().all().all()]
    for df in got.values():
        for i in range(3):
            assert np.isnan(df.iloc[i]).all() == (i in impossible)
    assert impossible, "the test network has no impossible row"


def test_rescued_rows_rerun_in_float64(interpreted, monkeypatch):
    bn = examples.asia()
    X = frame(bn, 10, 5, ASIA_COLS)
    want = bn.joint_marginals_many(X)
    monkeypatch.setattr(JointProgram, "flag_below", 2.0)  # every float32 row is flagged
    InterpretedProgram.calls.clear()
    bn._engine_cache.clear()
    got = bn.joint_marginals_many(X)
    assert any(f64 for _, _, f64, _ in InterpretedProgram.calls)
    for k in want:
        assert np.allclose(got[k].to_numpy(), want[k].to_numpy(), rtol=1e-6)


def test_errors(interpreted):
    bn = examples.asia()
    X = frame(bn, 5, 1, ASIA_COLS)
    with pytest.raises(ValueError, match="not nodes"):
        bn.joint_marginals_many(X, groups=["Smokers"])
    with pytest.raises(ValueError, match="not nodes"):
        bn.joint_marginals_many(X, groups=[("Smoker", "nope")])
    with pytest.raises(ValueError, match="duplicate"):
        bn.joint_marginals_many(X, groups=[("Smoker", "Smoker")])
    bad = X.copy()
    bad.loc[bad.index[0], "Smoker"] = "maybe"
    with pytest.raises(ValueError, match="not a state"):
        bn.joint_marginals_many(bad)


def test_empty_frame_and_fully_observed_patterns(interpreted):
    bn = examples.asia()
    empty = frame(bn, 0, 1, ASIA_COLS)
    got = bn.joint_marginals_many(empty, groups=["Smoker", ("Smoker", "Dispnea")])
    assert got["Smoker"].shape == (0, 2) and got[("Smoker", "Dispnea")].shape == (0, 4)
    X = frame(bn, 6, 2, ("Smoker", "Dispnea"), frac=0.0)
    got = bn.joint_marginals_many(X, groups=[("Smoker", "Dispnea")])  # observed completely: a counts program decides
    df = got[("Smoker", "Dispnea")]
    assert ((df == 0) | (df == 1)).all().all() and (df.sum(axis=1) == 1).all()


def test_groups_subsets_and_the_cache_key(interpreted):
    bn = examples.asia()
    X = frame(bn, 8, 6, ("Smoker",), frac=0.0)  # one pattern
    bn.joint_marginals_many(X, groups=["Dispnea"])
    n = len(InterpretedProgram.live)
    bn.joint_marginals_many(X, groups=["Dispnea"])
    assert len(InterpretedProgram.live) == n  # the same program
    bn.joint_marginals_many(X, groups=["Dispnea", "Bronchitis"])
    assert len(InterpretedProgram.live) == n + 1  # another group set is another program
    keys = [k for k in bn._engine_cache if k[0] == "joint"]
    assert len(keys) == 2 and all(len(k[2]) in (1, 2) for k in keys)
    got = bn.joint_marginals_many(X, groups="Dispnea")
    assert list(got) == ["Dispnea"]


def joint_golden_check(bn, name, rtol=1e-6):
    """Every case of tests/golden/joint_<name>.json (the reference's `query` of each group's unobserved members given
    the row's hard cells) through `joint_marginals_many`: the answer sits at the row's observed codes, the states
    the reference leaves out (probability zero) hold nothing, and its empty answers (impossible hard cells) are NaN.  Returns the number of answers checked."""
    from conftest import load_golden

    g = load_golden(f"joint_{name}")
    assert g["kind"] == "joint"
    n = 0
    for case in g["cases"]:
        hard = {k: v for k, v in case["hard"]}
        # (a row without a hard cell: one missing cell)
        X = pd.DataFrame([hard], columns=sorted(hard)) if hard else pd.DataFrame({case["answers"][0]["group"][0]: [None]})
        groups = [tuple(a["group"]) for a in case["answers"]]
        got = bn.joint_marginals_many(X, groups=groups)
        for a in case["answers"]:
            row = got[tuple(a["group"])].iloc[0]
            n += 1
            if not a["values"]:  # the reference's empty answer: hard cells of probability zero
                assert row.isna().all(), (name, case["hard"], a["group"])
                continue
            for key, value in zip(a["index"], a["values"]):
                full = tuple(hard[m] if m in hard else key[a["names"].index(m)] for m in a["group"])
                assert abs(row[full] - value) <= rtol * value + 1e-7, (name, case["hard"], a["group"], full)
            assert abs(row.sum() - 1.0) < 1e-6 and abs(sum(a["values"]) - 1.0) < 1e-9
    return n


@pytest.mark.parametrize("name", ["alarm", "asia", "grades", "sprinkler"])
def test_reference_joint_goldens(interpreted, name):
    assert joint_golden_check(getattr(examples, name)(), name) > 50
