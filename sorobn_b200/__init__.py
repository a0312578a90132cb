"""sorobn_b200: GPU-native exact inference for Bayesian networks on the NVIDIA H100.

A drop-in for the exact-inference path of MaxHalford/sorobn
(`BayesNet.query(..., algorithm="exact")`, `BayesNet.impute`), with the
factor-product / sum-out loop running as hand-written sm_90a CUDA kernels.
"""
from . import examples, planner, sharding, structure, synthetic, workloads
from .bayes_net import BayesNet

__version__ = "0.1.0"
__all__ = ["BayesNet", "examples", "planner", "sharding", "structure", "synthetic", "workloads"]
