"""TEST INFRASTRUCTURE (build container only): the reference's own EPDTC, from the module tests/ep_reference.py loads
(expectation_propagation.py, executed verbatim). Used by tests/golden/make_epdtc.py and tests/test_epdtc_cpu.py; never by
the product or by GPU-side tests."""
import importlib
import sys

from ep_reference import load_reference_ep


def load_reference_epdtc():
    """-> (EPDTC class, Bernoulli class, ObsAr) of the reference"""
    _, Bern, ObsAr = load_reference_ep()
    ep = sys.modules["GPy.inference.latent_function_inference.expectation_propagation"]
    importlib.import_module("GPy.inference.latent_function_inference.posterior")
    return ep.EPDTC, Bern, ObsAr
