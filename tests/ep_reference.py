"""TEST INFRASTRUCTURE (build container only): the reference's own EP (expectation_propagation.py) on top of
oracle/ref_gpy.py, which installs a stand-in for that module (its exact-GP path never reaches EP).

`load_reference_ep()` replaces the stand-in with the reference's module, executed verbatim. Not the reference's code on
this path: the two names the module imports from its package (ExactGaussianInference, VarDTC) are set on the stub package
from the reference's own modules, and the paramz stand-in gets paramz's `num_params` (the number of a parameterized
object's parameters, which Likelihood.ep_gradients reads for a likelihood without parameters). Y has to be passed as an
ObsAr (expectation_propagation.py:286 reads Y.values). Used by tests/golden/make_ep.py, tests/test_ep_cpu.py and
tools/ep_bench.py --reference-host; never by the product or by GPU-side tests.
"""
import importlib
import sys

from oracle import ref_gpy


def load_reference_ep():
    """-> (EP class, Bernoulli class, ObsAr) of the reference"""
    ref_gpy.load_sparse_models()
    ref_gpy.load_combination()
    lfi = sys.modules["GPy.inference.latent_function_inference"]
    lfi.ExactGaussianInference = sys.modules[
        "GPy.inference.latent_function_inference.exact_gaussian_inference"].ExactGaussianInference
    lfi.VarDTC = ref_gpy.load().VarDTC
    import paramz
    from paramz import parameterized
    if not hasattr(parameterized.Parameterized, "num_params"):
        parameterized.Parameterized.num_params = property(lambda self: len(self.parameters))
    name = "GPy.inference.latent_function_inference.expectation_propagation"
    sys.modules.pop(name, None)
    ep = importlib.import_module(name)
    lfi.expectation_propagation = ep
    return ep.EP, importlib.import_module("GPy.likelihoods.bernoulli").Bernoulli, paramz.ObsAr
