"""Sample plans (planner.build_sample_plan, version-7 programs) and BayesNet.sample_many, checked on the CPU.

oracle/program_interp.py executes the serialised words with numpy.  Every sample step's normalised
conditional must equal the oracle's posterior of the step's variables given the row's observed cells
and the variables drawn before them (`ve_oracle.query`), and seeded draws must follow the oracle's
joint posterior.  The host side of `sample_many` runs with the device programs replaced by the
interpreter."""
import numpy as np
import pandas as pd
import pytest
from scipy import stats

from conftest import build_network, load_golden
from interpreted_program import InterpretedProgram
from oracle import program_interp, ve_oracle
from sorobn_b200 import engine, examples, planner, workloads

EXAMPLES = ["alarm", "asia", "sprinkler", "grades"]


def oracle_net(bn):
    return ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def network(name):
    if name in EXAMPLES:
        return getattr(examples, name)()
    return build_network(load_golden(name))


def check_against_oracle(bn, observed, n_rows=3, n_draws=2, seed=1):
    net = bn._compiled
    dn = oracle_net(bn)
    plan = planner.build_sample_plan(net, observed)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, n_rows, seed)[list(observed)])
    drawn, prob, info = program_interp.run_sample(plan.words, plan.table_blob64, codes, n_rows=n_rows, n_draws=n_draws, seed=seed)
    assert not np.isnan(prob).any()
    worst = 0.0
    for st in info:
        X = [plan.sampled[st["d_first"] + j] for j in range(len(st["cards"]))]
        names = [net.names[x] for x in X]
        for b in range(n_rows):
            for d in range(n_draws):
                ev = {net.names[v]: net.domains[v][codes[i, b]] for i, v in enumerate(observed)}
                for j in range(st["d_first"]):
                    u = plan.sampled[j]
                    ev[net.names[u]] = net.domains[u][drawn[j, d, b]]
                vs, want, _ = ve_oracle.query(dn, *names, event=ev)
                # z runs first variable fastest: the flat conditional is C-ordered over reversed(X)
                got = st["cond"][:, d, b].reshape(tuple(reversed(st["cards"])))
                got = np.transpose(got, [len(X) - 1 - names.index(v) for v in vs])
                worst = max(worst, float(np.max(np.abs(got - want))))
    assert worst < 1e-12, (observed, worst)
    return plan


def test_every_unobserved_node_is_drawn_once_after_its_separator():
    for name in EXAMPLES + ["grid4x4s3", "dag20p4s4"]:
        bn = network(name)
        net = bn._compiled
        observed = (0, len(net.names) - 1)
        plan = planner.build_sample_plan(net, observed)
        assert plan.version == planner.VERSION_SAMPLE and plan.words[1] == 7
        assert sorted(plan.sampled) == [v for v in range(len(net.names)) if v not in observed]
        assert plan.words[10] == len(plan.sampled)
        samples = [st for st in plan.steps if st.kind == planner.KIND_SAMPLE]
        assert plan.steps[-len(samples):] == samples  # the sample steps run last
        done = set()
        for st in samples:
            assert st.q_offset == len(done) and tuple(plan.sampled[st.q_offset:st.q_offset + len(st.elims)]) == st.elims
            for f, es, _ in st.inputs:
                for col, _, _ in f.ev:
                    assert col < len(observed) or plan.sampled[col - len(observed)] in done
                assert set(f.vars) <= set(st.elims) | done
            done |= set(st.elims)
        words = plan.words.copy()
        planner._serialise(plan, [plan.table_blob64[o:o + s].reshape(-1) for o, s in plan.table_offsets])
        assert np.array_equal(words, plan.words)


@pytest.mark.parametrize("name", EXAMPLES + ["grid4x4s3", "dag20p4s4"])
def test_every_step_conditional_equals_the_oracle(name):
    bn = network(name)
    n_vars = len(bn.nodes)
    rng = np.random.default_rng(3)
    for k in range(4):  # 0 .. 3 observed columns, the other nodes latent
        observed = tuple(sorted(rng.choice(n_vars, size=k, replace=False).tolist()))
        check_against_oracle(bn, observed, seed=k)


@pytest.mark.parametrize("name,observed", [("sprinkler", ("Wet grass",)), ("asia", ("Dispnea", "Positive X-ray"))])
def test_seeded_joint_frequencies_follow_the_posterior(name, observed):
    bn = getattr(examples, name)()
    net = bn._compiled
    dn = oracle_net(bn)
    obs = tuple(sorted(net.index[o] for o in observed))
    plan = planner.build_sample_plan(net, obs)
    codes = np.ascontiguousarray(workloads.forward_sample_codes(net, 3, 9)[list(obs)])
    n = 20000
    drawn, prob, _ = program_interp.run_sample(plan.words, plan.table_blob64, codes, n_draws=n, seed=12345)
    names = [net.names[v] for v in plan.sampled]
    for b in range(codes.shape[1]):
        ev = {net.names[v]: net.domains[v][codes[i, b]] for i, v in enumerate(obs)}
        vs, want, _ = ve_oracle.query(dn, *names, event=ev)
        order = [names.index(v) for v in vs]
        flat = np.ravel_multi_index(tuple(drawn[j, :, b].astype(np.int64) for j in order), want.shape)
        freq = np.bincount(flat, minlength=want.size)
        expect = want.reshape(-1) * n
        assert freq[expect == 0].sum() == 0
        keep = expect > 0
        # merge the rare joint states into one cell, so that every expected count is at least 5
        rare = keep & (expect < 5)
        f = np.r_[freq[keep & ~rare], freq[rare].sum()]
        e = np.r_[expect[keep & ~rare], expect[rare].sum()]
        f, e = (f[:-1], e[:-1]) if e[-1] == 0 else (f, e)
        assert stats.chisquare(f, e).pvalue > 1e-4, (name, b)


def test_a_sample_step_past_the_bounds_is_refused(monkeypatch):
    net = examples.asia()._compiled
    planner.build_sample_plan(net, [0])
    monkeypatch.setattr(planner, "SAMPLE_MAX_CARD", 1)
    with pytest.raises(ValueError, match="uint8"):
        planner.build_sample_plan(net, [0])
    monkeypatch.undo()
    monkeypatch.setattr(planner, "SAMPLE_MAX_TERMS", 1)
    with pytest.raises(ValueError, match="gathers at most 1"):
        planner.build_sample_plan(net, [0])
    monkeypatch.undo()
    # a bucket of more than MAX_Z joint states (MAX_Z also bounds the fused buckets, so none forms at 1)
    monkeypatch.setattr(planner, "MAX_Z", 1)
    with pytest.raises(ValueError, match="draws from at most 1"):
        planner.build_sample_plan(net, [0])


def test_version_4_to_6_words_are_unchanged_by_the_sample_planner():
    net = examples.asia()._compiled
    assert planner.build_plan(net, [1], [0]).words[1] == 4
    assert planner.build_marginals_plan(net, [0]).words[1] == 5
    assert planner.build_counts_plan(net, [0]).words[1] == 6


# ---------------------------------------------------------------- sample_many on the interpreter
@pytest.fixture
def interpreted(monkeypatch):
    InterpretedProgram.live = []
    InterpretedProgram.calls = []
    InterpretedProgram.flag_below = None
    monkeypatch.setattr(engine, "Program", InterpretedProgram)
    return InterpretedProgram


def frame(bn, n, seed, frac, latent=()):
    net = bn._compiled
    codes = workloads.forward_sample_codes(net, n, seed)
    rng = np.random.default_rng(seed + 1)
    cols = {}
    for v, name in enumerate(net.names):
        if name in latent:
            continue
        values = np.asarray(net.domains[v], dtype=object)[codes[v]]
        values[rng.random(n) < frac] = None
        cols[name] = values
    return pd.DataFrame(cols)


def test_more_patterns_than_cached_programs(interpreted):
    bn = examples.asia()
    bn.max_cached_programs = 4
    X = frame(bn, 120, 3, 0.3)
    assert len(bn._count_patterns(X)) > 3 * bn.max_cached_programs
    got = bn.sample_many(X, n=2, seed=7)
    assert got.shape == (240, len(bn.nodes)) and list(got.columns) == sorted(bn.nodes)
    assert list(got.index.get_level_values(0)) == list(np.repeat(X.index, 2))
    assert list(got.index.get_level_values("draw")) == [0, 1] * 120
    assert len(bn._engine_cache) <= bn.max_cached_programs
    # the observed cells are copied through
    for c in X.columns:
        obs = X[c].notna().to_numpy()
        assert (got[c].to_numpy().reshape(120, 2)[obs] == X[c].to_numpy()[obs][:, None]).all()
    again = bn.sample_many(X, n=2, seed=7)
    assert again.equals(got)
    assert not bn.sample_many(X, n=2, seed=8).equals(got)


def alone(bn, X, b, n, seed):
    """{node: the n draws of row b of X} of the row run on its own by the interpreter, with row_base = b."""
    net = bn._compiled
    ev = tuple(sorted(net.index[c] for c in X.columns if pd.notna(X[c].iloc[b])))
    plan = planner.build_sample_plan(net, ev)
    codes = np.array([[net.domains[v].index(X[net.names[v]].iloc[b])] for v in ev], dtype=np.uint8).reshape(len(ev), 1)
    drawn, _, _ = program_interp.run_sample(plan.words, plan.table_blob64, codes, n_rows=1, n_draws=n, seed=seed, row_base=b)
    return {net.names[v]: list(np.asarray(net.domains[v], dtype=object)[drawn[j, :, 0]]) for j, v in enumerate(plan.sampled)}


def test_draws_follow_the_row_position_not_the_grouping(interpreted):
    """A row's draws depend on (seed, its position, draw): every row of a frame gets the draws it gets when
    run alone with row_base = its position, whatever the other rows (and so its pattern's grouping) are;
    relabelling the frame changes nothing."""
    bn = examples.asia()
    X = frame(bn, 60, 4, 0.4, latent=["Tuberculosis"])
    got = bn.sample_many(X, n=3, seed=11)
    # a permutation of the rows: each pattern's rows now sit at other positions, in other runs
    shuffled = X.iloc[np.random.default_rng(0).permutation(len(X))]
    got_s = bn.sample_many(shuffled, n=3, seed=11)
    assert list(got_s.index.get_level_values(0)) == list(np.repeat(shuffled.index, 3))
    for frame_, res in ((X, got), (shuffled, got_s)):
        for b in range(len(frame_)):
            for node, want in alone(bn, frame_, b, 3, 11).items():
                assert list(res[node].iloc[3 * b:3 * b + 3]) == want, (b, node)
    # the even positions keep their rows, the odd ones get other rows (other patterns): the even rows' draws stay
    other = X.copy()
    odd = np.arange(1, len(X), 2)
    other.iloc[odd] = shuffled.iloc[odd].to_numpy()
    got2 = bn.sample_many(other, n=3, seed=11)
    rows_even = np.concatenate([np.arange(3 * p, 3 * p + 3) for p in range(0, len(X), 2)])
    assert got2.iloc[rows_even].equals(got.iloc[rows_even])
    # labels do not enter the stream
    relabelled = X.set_axis([f"r{i}" for i in range(len(X))])
    assert np.array_equal(bn.sample_many(relabelled, n=3, seed=11).to_numpy(), got.to_numpy())


def test_errors(interpreted):
    bn = examples.sprinkler()
    X = pd.DataFrame({"Rain": [False, True], "Sprinkler": [False, True], "Wet grass": [True, True]})
    with pytest.raises(ValueError, match="probability zero"):
        bn.sample_many(X)
    with pytest.raises(ValueError, match="not a state"):
        bn.sample_many(pd.DataFrame({"Rain": ["maybe"]}))
    with pytest.raises(ValueError, match="at least 1"):
        bn.sample_many(X.iloc[1:], n=0)


def test_rows_the_float32_program_flags_are_drawn_by_the_float64_program(interpreted):
    bn = examples.asia()
    X = frame(bn, 50, 6, 0.0)[["Dispnea", "Smoker", "Positive X-ray"]]
    net = bn._compiled
    ev = tuple(sorted(net.index[c] for c in X.columns))
    plan = planner.build_sample_plan(net, ev)
    codes = np.array([[net.domains[v].index(x) for x in X[net.names[v]]] for v in ev], dtype=np.uint8)
    want, p, _ = program_interp.run_sample(plan.words, plan.table_blob64, codes, n_draws=2, seed=3)
    interpreted.flag_below = float(np.median(p))
    got = bn.sample_many(X, n=2, seed=3)
    assert any(f64 for _, _, f64, _ in interpreted.calls) and any(not f64 for _, _, f64, _ in interpreted.calls)
    assert sum(n for _, _, f64, n in interpreted.calls if f64) == int((p < np.median(p)).sum())
    for j, v in enumerate(plan.sampled):
        assert list(got[net.names[v]]) == list(np.asarray(net.domains[v], dtype=object)[want[j].T.reshape(-1)])


def test_the_counts_and_sample_pattern_programs_share_the_cache(monkeypatch):
    """`_pattern_runner("counts", ...)` (used by tools/em_bench.py) and `_pattern_runner("sample", ...)` share the
    program cache under their own keys."""
    class FakeProgram:
        def __init__(self, plan, device=None, f64=False):
            self.plan = plan

        def close(self):
            pass

    monkeypatch.setattr(engine, "Program", FakeProgram)
    bn = examples.asia()
    counts = bn._pattern_runner("counts", (0,))
    samples = bn._pattern_runner("sample", (0,))
    assert counts.plan.version == planner.VERSION_COUNTS and samples.plan.version == planner.VERSION_SAMPLE
    assert bn._pattern_runner("counts", (0,)) is counts and bn._pattern_runner("sample", (0,)) is samples
