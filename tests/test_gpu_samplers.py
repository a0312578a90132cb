"""The sampler kernels (csrc/sbn_gibbs.cuh) against an exact CPU replay of their random streams.

Every draw of the samplers comes from Philox-4x32-10 and every comparison is a plain float32
operation, so `oracle/sampler_replay.py` reproduces the Gibbs kernels and rejection sampling bit
for bit, and likelihood weighting up to the order of its float64 sums.  The replay itself is held
to the float64 oracle by tests/test_sampler_replay.py; here the pooled Gibbs frequencies and the
Gibbs conditionals are also checked against the oracle directly.

Which sampler kernel each network and algorithm runs (the dispatch depends on the network and the
algorithm only) is read from the kernel census (tests/kernel_census.py) by
`test_each_network_runs_the_sampler_kernel_it_is_meant_for`, in a fresh interpreter: after many
profiler sessions in one process the profiler stops recording the sampler kernels.  The census cannot
see where the generic kernel reads its tables from; that is asserted on the host from the size of the
table blob.
"""
import itertools
import zlib

import numpy as np
import pytest

import kernel_census
import kernel_corpus
from oracle import sampler_replay as rp
from oracle import ve_oracle

pytestmark = pytest.mark.gpu

FLAT, GEN8, GEN64, FORWARD = ("sbn_gibbs_flat_kernel", "sbn_gibbs_kernel<8>", "sbn_gibbs_kernel<64>",
                              "sbn_forward_kernel")
CHAIN_COUNTS = (1, 63, 64, 65, 777)     # 64 chains per CTA
SAMPLE_COUNTS = (1, 127, 129, 1000)     # 128 threads per evidence row
SMEM_TABLES_MAX = 100 * 1024            # sampler_run stages the tables when they fit beside the chain state


class Net:
    """A network with its query, evidence and Gibbs cycle (non-event variables, sorted by name as
    `BayesNet` orders them), the float64 oracle's view of it, and evidence rows."""

    def __init__(self, name, net, dn, query, evidence, rows, gibbs_kernel, spec=None):
        self.name, self.net, self.dn = name, net, dn
        self.query = sorted((net.index[q] for q in query), key=lambda v: net.names[v])
        self.evidence = [net.index[e] for e in evidence]
        self.cycle = sorted(set(range(len(net.names))) - set(self.evidence), key=lambda v: net.names[v])
        self.rows, self.gibbs_kernel, self.spec = rows, gibbs_kernel, spec

    def sampler(self):
        from sorobn_b200 import engine

        return engine.GibbsSampler(self.net, self.query, self.evidence, self.cycle)

    def event(self, codes, b):
        """Row b of the codes as an oracle event (variable name -> state value)."""
        return {self.net.names[v]: self.net.domains[v][int(codes[k, b])] for k, v in enumerate(self.evidence)}


def _textbook(name, query, event_vars, kernel, codes=None):
    from sorobn_b200 import examples

    bn = getattr(examples, name)(seed=1)
    net = bn._compiled
    dn = ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)

    def rows(n):
        """Every joint code of the evidence columns (probability-zero ones included), repeated."""
        if codes is not None:
            return np.ascontiguousarray(np.repeat(np.array(codes, dtype=np.uint8)[:, None], n, axis=1))
        joint = np.array(list(itertools.product(*[range(int(net.card[net.index[e]])) for e in event_vars])),
                         dtype=np.uint8).T
        return np.ascontiguousarray(np.resize(joint, (len(event_vars), n)))

    return Net(name, net, dn, query, event_vars, rows, kernel)


def _spec(name, spec, query, evidence, kernel):
    net, dn = kernel_corpus.compiled_net(spec), kernel_corpus.dense_net(spec)
    return Net(name, net, dn, query, evidence,
               lambda n: kernel_corpus.evidence_rows(spec, evidence, n, seed=zlib.crc32(name.encode()) % 1000),
               kernel, spec)


def _corpus(name, kernel):
    case = next(c for c in kernel_corpus.CASES if c["name"] == name)
    spec = kernel_corpus.make_spec(case)
    return _spec(name, spec, [spec.nodes[k] for k in case["query"]], [spec.nodes[k] for k in case["evidence"]], kernel)


def _grid():
    from sorobn_b200 import workloads

    wl = workloads.grid10x10()
    return _spec("grid10x10", wl.spec, list(wl.query), list(wl.evidence), FLAT)


def _grid_zeros():
    """A 6x6 3-state grid with about 30 % structural zeros: forward-sampled starts can contradict the
    event, so some conditionals are all zero.  Small enough for the straight-line kernel."""
    from sorobn_b200 import synthetic

    spec = synthetic.grid(6, 6, 3, seed=0)
    kernel_corpus._add_structural_zeros(spec, 0.3, 0)
    return _spec("grid6x6s3_zeros", spec, [spec.nodes[35]], [spec.nodes[k] for k in (3, 10, 17, 28)], FLAT)


def _five_query():
    """Five binary query variables: the generic kernel's n_query > 4 branch (32 joint states)."""
    from sorobn_b200 import synthetic

    spec = synthetic.random_dag(12, 2, 2, seed=0, window=4)
    return _spec("dag12p2s2_q5", spec, [spec.nodes[k] for k in (2, 5, 7, 9, 11)], [spec.nodes[0], spec.nodes[4]], GEN8)


def _naive():
    spec = kernel_corpus.naive_bayes()
    return _spec("naive60s5x17", spec, ["c"], spec.nodes[1:], GEN8)


NETS = {
    "sprinkler": lambda: _textbook("sprinkler", ["Rain"], ["Sprinkler"], FLAT),
    "asia": lambda: _textbook("asia", ["Lung cancer", "Bronchitis"], ["Smoker", "Dispnea"], FLAT),
    "asia_tb_or_cancer_false": lambda: _textbook("asia", ["Smoker"], ["TB or cancer"], FLAT, codes=[0]),
    "alarm": lambda: _textbook("alarm", ["Burglary"], ["John calls", "Mary calls"], FLAT),
    "grid10x10": _grid,
    "dag7p2s13x9x4": lambda: _corpus("dag7p2s13x9x4_seed5_q6_e2", GEN64),
    "dag6p2s37x2": lambda: _corpus("dag6p2s37x2_seed1_q2_e2", GEN64),
    "dag300p1s17": lambda: _corpus("dag300p1s17_seed2_q0_e5", GEN64),
    "dag16p4s8_global_tables": lambda: _corpus("dag16p4s8_seed0_q15_e2", GEN8),
    "dag12p2s2_q5": _five_query,
    "naive60s5x17": _naive,
    "grid6x6s3_zeros": _grid_zeros,
}
_cache = {}


def get(key):
    if key not in _cache:
        _cache[key] = NETS[key]()
    return _cache[key]


class _Run:
    """What kernel_census.census_many expects of a program: `run(codes, n)` (here: one sampler run,
    whose output is kept) and `set_graph` (the samplers launch no graph)."""

    def __init__(self, sampler, n_iterations, seed, algorithm):
        self.sampler, self.n_iterations, self.seed, self.algorithm = sampler, n_iterations, seed, algorithm
        self.out = None

    def set_graph(self, mode):
        pass

    def run(self, codes, n):
        self.out = self.sampler.run(codes, n, self.n_iterations, self.seed, self.algorithm)
        return self.out


def run_jobs(sampler, jobs):
    """jobs: (codes, n_rows, n_iterations, seed, algorithm) -> the outputs."""
    return [sampler.run(codes, n, it, seed, algo) for codes, n, it, seed, algo in jobs]


def census_of_jobs(sampler, jobs):
    """The sampler kernels each job launched (kernel census; every sampler run launches exactly one
    kernel).  The profiler now and then drops the activity records of a session, which says nothing
    about the kernels, so a session that lost records is taken once more."""
    for attempt in (0, 1):
        runs = [(_Run(sampler, it, seed, algo), codes, n) for codes, n, it, seed, algo in jobs]
        try:
            names = kernel_census.census_many(runs)
        except AssertionError:
            if attempt:
                raise
            continue
        out = [sorted({name for name, _ in launched}) for launched in names]
        if attempt or all(out):
            return out


GLOBAL_TABLES = {"dag16p4s8_global_tables", "dag300p1s17"}


def assert_tables_where_expected(key, net, sampler):
    """The generic kernel keeps the tables in global memory when they do not fit beside the chain
    state (sampler_run), and stages them in shared memory otherwise."""
    blob = sampler._tables.nbytes
    if key in GLOBAL_TABLES:
        assert blob > SMEM_TABLES_MAX, blob
    elif net.gibbs_kernel != FLAT:
        assert blob < SMEM_TABLES_MAX // 2, blob


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


GIBBS_KEYS = ["sprinkler", "asia", "asia_tb_or_cancer_false", "alarm", "grid10x10", "dag7p2s13x9x4", "dag6p2s37x2",
              "dag300p1s17", "dag16p4s8_global_tables", "dag12p2s2_q5", "naive60s5x17", "grid6x6s3_zeros"]


@pytest.mark.parametrize("key", GIBBS_KEYS)
def test_gibbs_kernels_equal_the_replay_bit_for_bit(key):
    """Chain counts around the 64-chain CTA; chain c depends only on its own row and the seed, so
    every run must equal the first columns of one replay of 777 chains.  The generic kernel, forced,
    must give the same bits too."""
    net = get(key)
    sampler = net.sampler()
    assert_tables_where_expected(key, net, sampler)
    n_it = max(200, 3 * len(net.cycle) + 17)
    seed = zlib.crc32(key.encode())
    codes = net.rows(max(CHAIN_COUNTS))
    want = rp.gibbs(net.net, net.query, net.evidence, net.cycle, codes, codes.shape[1], n_it, seed)
    jobs = [(np.ascontiguousarray(codes[:, :n]), n, n_it, seed, "gibbs") for n in CHAIN_COUNTS]
    jobs.append((codes, codes.shape[1], n_it, seed, "gibbs_generic"))
    results = run_jobs(sampler, jobs)
    for (codes_n, n, _, _, algo), got in zip(jobs, results):
        assert got.shape == (want.shape[0], n)
        assert np.array_equal(bits(got), bits(want[:, :n])), (algo, n, np.argwhere(bits(got) != bits(want[:, :n]))[:5])
    sampler.close()


@pytest.mark.parametrize("key", ["asia_tb_or_cancer_false", "grid6x6s3_zeros"])
def test_straight_line_and_generic_gibbs_agree_when_conditionals_are_all_zero(key):
    """A forward-sampled start can contradict the event under deterministic or zero CPT entries, and
    the first update of such a chain then has an all-zero conditional: the chain keeps its value, and
    both kernels must still consume one draw so that their streams stay together."""
    net = get(key)
    codes = net.rows(777)
    stats = {}
    rp.gibbs(net.net, net.query, net.evidence, net.cycle, codes, 777, 3001, 99, stats=stats)
    assert stats["all_zero"] > 0, "no chain meets an all-zero conditional: the case tests nothing"
    sampler = net.sampler()
    flat, generic = run_jobs(sampler, [(codes, 777, 3001, 99, "gibbs"), (codes, 777, 3001, 99, "gibbs_generic")])
    assert np.array_equal(bits(flat), bits(generic)), np.argwhere(bits(flat) != bits(generic))[:5]
    sampler.close()


FORWARD_KEYS = ["sprinkler", "asia", "alarm", "grid10x10", "dag7p2s13x9x4", "dag6p2s37x2", "dag16p4s8_global_tables",
                "dag12p2s2_q5", "naive60s5x17"]


@pytest.mark.parametrize("key", FORWARD_KEYS)
@pytest.mark.parametrize("algorithm", ["rejection", "likelihood"])
def test_forward_kernel_equals_the_replay(key, algorithm):
    """Rejection sampling: bit for bit, NaN rows (no sample kept) included.  Likelihood weighting:
    the kernel adds the float64 likelihoods in the order its atomics land, then rounds to float32, so
    within 3e-7 relative, and two runs of one seed within one float32 ulp."""
    net = get(key)
    sampler = net.sampler()
    rows = 5
    codes = net.rows(rows)
    seed = zlib.crc32((key + algorithm).encode())
    jobs = [(codes, rows, n_it, seed, algorithm) for n_it in SAMPLE_COUNTS]
    if algorithm == "likelihood":
        jobs.append(jobs[-1])
    results = run_jobs(sampler, jobs)
    for (_, _, n_it, _, _), got in zip(jobs, results):
        want = rp.forward(net.net, net.query, net.evidence, codes, rows, n_it, seed, algorithm)
        if algorithm == "rejection":
            assert np.array_equal(bits(got), bits(want)), (n_it, got, want)
            continue
        assert np.array_equal(np.isnan(got), np.isnan(want)), (n_it, got, want)
        ok = ~np.isnan(want)
        assert np.all(np.abs(got[ok] - want[ok]) <= 3e-7 * np.abs(want[ok])), (n_it, got, want)
    if algorithm == "likelihood":
        a, b = results[-2], results[-1]
        assert np.array_equal(np.isnan(a), np.isnan(b))
        ok = ~np.isnan(a)
        assert np.all(np.abs(bits(a)[ok].astype(np.int64) - bits(b)[ok].astype(np.int64)) <= 1)
        if key in ("grid10x10", "naive60s5x17"):  # every evidence row is possible: an answer for each
            assert np.isfinite(a).all(), a
            assert np.allclose(a.sum(axis=0), 1.0, atol=1e-5), a.sum(axis=0)
    sampler.close()


@pytest.mark.parametrize("key", ["asia", "grid10x10", "dag6p2s37x2", "naive60s5x17"])
def test_pooled_gibbs_chains_track_the_exact_posterior(key):
    """4096 chains of one event, pooled: the error of the pooled frequencies shrinks with the number
    of chains (they are independent), so a wrong blanket term or a stuck chain shows as a bias far
    above the standard error.  Asia's event is on root variables only: its deterministic OR makes the
    chain reducible, but a forward sample clamped on roots is an exact posterior sample."""
    net = get(key)
    if key == "asia":
        net = Net("asia_roots", net.net, net.dn, ["Lung cancer", "Bronchitis"], ["Smoker"], None, FLAT)
        codes = np.ones((1, 1), dtype=np.uint8)
    else:
        codes = net.rows(200)[:, -1:]  # a forward-sampled event
    n = 4096
    sampler = net.sampler()
    (freq,) = run_jobs(sampler, [(np.ascontiguousarray(np.repeat(codes, n, axis=1)), n, 400 * len(net.cycle), 2024, "gibbs")])
    assert np.allclose(freq.sum(axis=0), 1.0, atol=1e-5)
    want = ve_oracle.query(net.dn, *[net.net.names[v] for v in net.query], event=net.event(codes, 0))[1].reshape(-1)
    pooled = freq.mean(axis=1)
    sem = freq.std(axis=1, ddof=1) / np.sqrt(n)
    assert np.all(np.abs(pooled - want) < 6 * sem + 2e-3), (pooled, want, sem)
    sampler.close()


@pytest.mark.parametrize("key", ["naive60s5x17", "dag7p2s13x9x4", "dag6p2s37x2"])
def test_gibbs_conditional_kernel_matches_the_oracle(key):
    """P(v | Markov blanket) as the chains evaluate it (the same device function), for a sample of
    joint states, against the float64 conditional: every state of the naive-Bayes class variable,
    whose float32 product over 60 children underflows without rescaling, and every cycle variable
    of the >8-state corpus networks."""
    net = get(key)
    sampler = net.sampler()
    rng = np.random.default_rng(zlib.crc32(key.encode()))
    card = [int(c) for c in net.net.card]
    checked = 0
    for v in net.cycle:
        for _ in range(64 if key.startswith("naive") else 12):
            joint = np.array([rng.integers(0, c) for c in card], dtype=np.uint8)
            got = sampler.conditional(v, joint)
            want = ve_oracle.gibbs_conditional_at(net.dn, net.net.names[v],
                                                  {net.net.names[u]: net.net.domains[u][x] for u, x in enumerate(joint)})
            if np.isnan(want).all():
                assert np.isnan(got).all(), got
                continue
            assert np.all(np.abs(got - want) <= 2e-6 * np.maximum(want, 1e-30)), (net.net.names[v], joint, got, want)
            checked += 1
    assert checked >= 40
    sampler.close()


_CENSUS_SCRIPT = """
import json, sys
import test_gpu_samplers as T
out = {}
for key in T.GIBBS_KEYS:
    net = T.get(key)
    sampler = net.sampler()
    codes = net.rows(65)
    jobs = [(codes, 65, 50, 1, algo) for algo in ("gibbs", "gibbs_generic", "likelihood", "rejection")]
    out[key] = T.census_of_jobs(sampler, jobs)
    sampler.close()
json.dump(out, sys.stdout)
"""


def test_each_network_runs_the_sampler_kernel_it_is_meant_for():
    """The kernel census of every network under every algorithm, taken in a fresh interpreter: the
    straight-line kernel, `sbn_gibbs_kernel<8>` and `<64>` (a cycle variable with more than 8 states)
    for Gibbs, the generic kernel when it is forced, and `sbn_forward_kernel` for both forward
    samplers.  The benchmark grid must stay on the straight-line kernel."""
    import json
    import os
    import subprocess
    import sys

    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([here, os.path.dirname(here), os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", _CENSUS_SCRIPT], capture_output=True, text=True, env=env, cwd=here,
                         timeout=600)
    assert res.returncode == 0, res.stderr[-3000:]
    census = json.loads(res.stdout)
    seen = set()
    for key in GIBBS_KEYS:
        net = get(key)
        generic = GEN64 if max(int(net.net.card[v]) for v in net.cycle) > 8 else GEN8
        assert census[key] == [[net.gibbs_kernel], [generic], [FORWARD], [FORWARD]], (key, census[key])
        seen.update(k for ks in census[key] for k in ks)
    assert census["grid10x10"][0] == [FLAT]
    assert seen == {FLAT, GEN8, GEN64, FORWARD}, seen
