import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with `-m gpu`)")


def load_golden(name):
    with open(os.path.join(GOLDEN, f"{name}.json")) as f:
        return json.load(f)


def golden_names(kinds=("example", "synthetic", "workload")):
    """Golden files of the given kinds (query goldens by default; "predict_proba" for the
    row-likelihood vectors)."""
    out = []
    for fn in sorted(os.listdir(GOLDEN)):
        if fn.endswith(".json"):
            with open(os.path.join(GOLDEN, fn)) as f:
                g = json.load(f)
            if g["kind"] in kinds:
                out.append(fn[:-5])
    return out


def build_network(golden, cls=None):
    """Rebuild the network a golden file was generated on, with this package's classes."""
    from sorobn_b200 import BayesNet, examples, synthetic, workloads

    cls = cls or BayesNet
    if golden["kind"] == "example":
        return examples.build(examples.NETWORKS[golden["network"]], cls=cls)
    if golden["kind"] == "synthetic":
        spec = getattr(synthetic, golden["generator"])(**golden["kwargs"])
    else:
        spec = workloads.WORKLOADS[golden["workload"]]().spec
    assert spec_digest(spec) == golden["digest"], "synthetic generator drifted: regenerate tests/golden"
    return synthetic.load(spec, cls)


def spec_digest(spec):
    import hashlib

    h = hashlib.sha256()
    for n in spec.nodes:
        h.update(n.encode())
        h.update(np.ascontiguousarray(spec.cpt[n], dtype=np.float64).tobytes())
    return h.hexdigest()


def case_event(case):
    return {k: v for k, v in case["event"]}


def dense_answer(case, domains):
    """Golden answer as a dense array over the (sorted) query variables' domains;
    rows the reference dropped (zero posterior) are 0."""
    names = case["names"]
    shape = [len(domains[n]) for n in names]
    arr = np.zeros(shape)
    pos = [{v: i for i, v in enumerate(domains[n])} for n in names]
    for key, val in zip(case["index"], case["values"]):
        arr[tuple(pos[i][k] for i, k in enumerate(key))] = val
    return arr
