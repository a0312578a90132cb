"""The CPU replay of the sampler kernels (oracle/sampler_replay.py), checked without a GPU.

The GPU tests compare the kernels with this replay bit for bit, so a replay that shared a
misreading of the algorithm with a kernel would hide it.  Here the replay's random stream is
pinned to the Philox-4x32-10 known-answer vectors, and its estimates are checked against the
float64 oracle: Gibbs and rejection frequencies against the exact posterior, likelihood weighting
against the exact expectation of the reference's estimator, each within a few standard errors."""
import numpy as np
import pytest

import kernel_corpus
from oracle import sampler_replay as rp
from oracle import ve_oracle


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    """Random123's known-answer vectors for Philox-4x32-10."""
    got = rp.philox4x32([np.array([c], dtype=np.uint32) for c in ctr], key)
    assert [int(w[0]) for w in got] == list(want)


def test_stream_block_layout_and_word_order():
    """Seed -> key (low, high), chain -> counter words 2 and 3, block counter in word 0, and the
    four words of a block used last first."""
    s = rp.Stream(0, [0])
    words = (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    for w in reversed(words):
        assert s.uniform()[0] == np.float32(((w >> 8) + 1) * 2.0 ** -24)
    # the second block: counter 1; chain ids in words 2 and 3; seed split into (low, high)
    s = rp.Stream(0x299F31D0_A4093822, [(0x03707344 << 32) | 0x13198A2E])
    first = rp.philox4x32([np.array([0], np.uint32), np.array([0], np.uint32), np.array([0x13198A2E], np.uint32),
                           np.array([0x03707344], np.uint32)], (0xA4093822, 0x299F31D0))
    second = rp.philox4x32([np.array([1], np.uint32), np.array([0], np.uint32), np.array([0x13198A2E], np.uint32),
                            np.array([0x03707344], np.uint32)], (0xA4093822, 0x299F31D0))
    for w in [*reversed(first), *reversed(second)]:
        assert s.uniform()[0] == np.float32(((int(w[0]) >> 8) + 1) * 2.0 ** -24)
    u = rp.Stream(7, np.arange(1000)).uniform()
    assert u.dtype == np.float32 and (u > 0).all() and (u <= 1).all()


def _example(name, seed):
    from sorobn_b200 import examples

    bn = getattr(examples, name)(seed=seed)
    return bn._compiled, ve_oracle.dense_from_pandas(bn.P, bn.parents, bn.nodes)


def _ids(net, names):
    return [net.index[n] for n in names]


def _codes(net, event, n):
    return np.array([[net.domains[net.index[k]].index(v)] * n for k, v in event.items()], dtype=np.uint8).reshape(len(event), n)


def _exact(dn, query, event):
    return ve_oracle.query(dn, *query, event=event)[1].reshape(-1)


# Asia's "TB or cancer" is a deterministic OR, so its Gibbs chain is not irreducible: a chain can
# stay where its forward-sampled start put it.  With evidence on root variables only, that start is an
# exact posterior sample, so the chains pooled still track the posterior.
CASES = [
    ("sprinkler", ("Rain",), {"Sprinkler": True}),
    ("sprinkler", ("Cloudy", "Rain"), {"Wet grass": False}),
    ("asia", ("Dispnea", "Lung cancer"), {"Smoker": True}),
    ("asia", ("Bronchitis", "Tuberculosis"), {"Visit to Asia": True, "Smoker": False}),
]


@pytest.mark.parametrize("name,query,event", CASES)
def test_replayed_gibbs_converges_to_the_exact_posterior(name, query, event):
    net, dn = _example(name, 3)
    q = sorted(_ids(net, query), key=lambda v: net.names[v])
    ev = _ids(net, event)
    cycle = sorted(set(range(len(net.names))) - set(ev), key=lambda v: net.names[v])
    n = 2000
    freq = rp.gibbs(net, q, ev, cycle, _codes(net, event, n), n, 400 * len(cycle), seed=11)
    assert np.allclose(freq.sum(axis=0), 1.0, atol=1e-5)
    pooled, sem = freq.mean(axis=1), freq.std(axis=1, ddof=1) / np.sqrt(n)
    want = _exact(dn, query, event)
    assert np.all(np.abs(pooled - want) < 5 * sem + 1e-3), (pooled, want, sem)


@pytest.mark.parametrize("name,query,event", CASES)
def test_replayed_rejection_sampling_converges_to_the_exact_posterior(name, query, event):
    net, dn = _example(name, 3)
    q = sorted(_ids(net, query), key=lambda v: net.names[v])
    n_it = 200_000
    got = rp.forward(net, q, _ids(net, event), _codes(net, event, 1), 1, n_it, seed=5, algorithm="rejection")[:, 0]
    want = _exact(dn, query, event)
    kept = n_it * ve_oracle.evidence_probability(dn, event)
    sem = np.sqrt(want * (1 - want) / kept)
    assert np.isclose(got.sum(), 1.0, atol=1e-5)
    assert np.all(np.abs(got - want) < 5 * sem + 1e-6), (got, want, sem)


def test_replayed_rejection_sampling_returns_nan_when_nothing_is_kept():
    net, _ = _example("asia", 1)
    event = {"TB or cancer": False, "Lung cancer": True}  # impossible: TB or cancer is a deterministic OR
    got = rp.forward(net, _ids(net, ["Smoker"]), _ids(net, event), _codes(net, event, 2), 2, 5000, seed=1,
                     algorithm="rejection")
    assert np.isnan(got).all()


@pytest.mark.parametrize("name,query,event", [
    ("sprinkler", ("Rain",), {"Sprinkler": True}),
    ("alarm", ("Burglary",), {"John calls": True, "Mary calls": True}),
    ("grades", ("Letter", "SAT"), {"Intelligence": "Smart"}),
])
def test_replayed_likelihood_weighting_converges_to_the_reference_estimator(name, query, event):
    """20 rows of the same event are 20 independent estimates: their spread gives the standard error."""
    net, _ = _example(name, 5)
    q = sorted(_ids(net, query), key=lambda v: net.names[v])
    rows = 20
    got = rp.forward(net, q, _ids(net, event), _codes(net, event, rows), rows, 20_000, seed=9, algorithm="likelihood")
    assert np.allclose(got.sum(axis=0), 1.0, atol=1e-5)
    want = np.zeros(got.shape[0])
    for key, p in rp.lw_expectation(net, query, event).items():
        want[np.ravel_multi_index(key, [int(net.card[v]) for v in q])] = p
    pooled, sem = got.mean(axis=1), got.std(axis=1, ddof=1) / np.sqrt(rows)
    assert np.all(np.abs(pooled - want) < 6 * sem + 1e-6), (pooled, want, sem)


def test_replayed_gibbs_weights_equal_the_oracle_conditional():
    """The replay's float32 weights, rescaled, against the float64 conditional: on the naive-Bayes
    class variable, where the plain float32 product underflows, and on every variable of Alarm."""
    spec = kernel_corpus.naive_bayes()
    net, dn = kernel_corpus.compiled_net(spec), kernel_corpus.dense_net(spec)
    tabs = rp._Tables(net)
    rng = np.random.default_rng(0)
    n = 64
    state = np.stack([rng.integers(0, int(c), n) for c in net.card])
    w = rp.gibbs_weights(tabs, 0, state).astype(np.float64)
    got = w / w.sum(axis=0)
    plain = np.repeat(tabs.flat[0][:, None], n, axis=1)  # the same product without rescaling
    for v in range(1, len(net.names)):
        plain = plain * tabs.flat[v].reshape(5, 17)[:, state[v]]
    assert (plain.max(axis=0) == 0).mean() > 0.5, "the case no longer underflows float32"
    for b in range(n):
        want = ve_oracle.gibbs_conditional_at(dn, "c", {u: int(state[k, b]) for k, u in enumerate(spec.nodes)})
        assert np.allclose(got[:, b], want, rtol=2e-6, atol=1e-30), (b, got[:, b], want)

    net, dn = _example("alarm", 2)
    tabs = rp._Tables(net)
    for v in range(len(net.names)):
        boundary, table = ve_oracle.gibbs_conditional(dn, net.names[v])
        for joint in np.ndindex(*[int(c) for c in net.card]):
            st = np.array(joint)[:, None]
            w = rp.gibbs_weights(tabs, v, st)[:, 0].astype(np.float64)
            want = table[tuple(joint[net.index[u]] for u in boundary)]
            if w.sum() == 0:
                assert np.isnan(want).all()
                continue
            assert np.allclose(w / w.sum(), want, rtol=2e-6, atol=0), (net.names[v], joint, w, want)
            at = ve_oracle.gibbs_conditional_at(dn, net.names[v], {net.names[u]: net.domains[u][x] for u, x in enumerate(joint)})
            assert np.allclose(at, want, rtol=1e-12, atol=0)
