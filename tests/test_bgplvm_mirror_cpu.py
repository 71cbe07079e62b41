"""gpy_b200.BayesianGPLVM on a host double of the engine (its gpx_sparse_eval_psi restated by tests/bgplvm_oracle.py):
the bound and gradient order against the reference fixtures, the seeded draws, the optimiser space and the errors it
raises. No GPU needed."""
import os

import numpy as np
import pytest

import bgplvm_oracle as bo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bgplvm")


class HostEngine(object):
    """the sparse entries BayesianGPLVM calls, on the host"""

    def __init__(self):
        self.sparse_serial, self.calls = 0, 0

    def set_option(self, name, value):
        pass

    def sparse_set_data(self, X, Y):
        self.X, self.Y = np.array(X, dtype=np.float64), np.array(Y, dtype=np.float64)

    def sparse_eval_psi(self, rbf, S, Z, noise):
        kind, ard, term, dims, variance, ls = rbf
        assert kind == "rbf" and list(dims) == list(range(self.X.shape[1]))
        r = bo.vardtc_psi(variance, np.atleast_1d(ls), ard, np.asarray(Z), self.X, np.asarray(S), self.Y, noise)
        self.sparse_serial += 1
        self.calls += 1
        return r["lml"], r["grad"], r["dZ"], r["dmu"], r["dS"]


def _model(name, **kw):
    import gpy_b200
    f = np.load(os.path.join(GOLD, name + ".npz"))
    Q = f["mu"].shape[1]
    ard = bool(f["ard"])
    kern = gpy_b200.RBF(Q, variance=float(f["variance"]), lengthscale=f["ls"] if ard else float(f["ls"][0]), ARD=ard)
    m = gpy_b200.BayesianGPLVM(f["Y"], Q, X=f["mu"], X_variance=f["S"], Z=f["Z"], kernel=kern, engine=HostEngine(), **kw)
    m.likelihood.variance[:] = float(f["noise"])
    return m, f


@pytest.mark.parametrize("name", ["default_p1", "iso", "default_p12"])
def test_mirror_bound_and_gradient_order(name):
    m, f = _model(name)
    assert abs(m.log_likelihood() - float(f["bound"])) <= 1e-8 * max(1.0, abs(float(f["bound"])))
    ref = np.concatenate([(f["dmu"] + f["kl_mu"]).ravel(), (f["dS"] + f["kl_S"]).ravel(), f["dZ"].ravel(), f["grad"]])
    g = m.gradient
    assert g.shape == ref.shape
    assert np.max(np.abs(g - ref)) <= 1e-6 * np.max(np.abs(ref))
    names = [p.name for p in m.flattened_parameters()]
    assert names[:3] == ["latent space mean", "latent space variance", "inducing inputs"]


def test_seeded_draws_follow_the_reference_order():
    import gpy_b200
    from gpy_b200.gplvm import initialize_latent
    Y = np.load(os.path.join(GOLD, "default_p8.npz"))["Y"]
    np.random.seed(5)
    X, fracs = initialize_latent("PCA", 3, Y)
    S = np.random.uniform(0, .1, X.shape)
    Z = np.random.permutation(X.copy())[:7]
    np.random.seed(5)
    m = gpy_b200.BayesianGPLVM(Y, 3, num_inducing=7, engine=HostEngine())
    np.testing.assert_array_equal(m.latent_mean.values, X)
    np.testing.assert_array_equal(m.latent_variance.values, S)
    np.testing.assert_array_equal(m.Z.values, Z)
    np.testing.assert_allclose(m.kern.lengthscale.values, 1.0 / fracs)


def test_checkgrad_and_a_few_optimiser_steps():
    import gpy_b200
    Y = np.load(os.path.join(GOLD, "default_p1.npz"))["Y"][:25]
    np.random.seed(2)
    m = gpy_b200.BayesianGPLVM(Y, 2, num_inducing=5, engine=HostEngine())
    assert m.checkgrad(tolerance=1e-4)
    b0 = -m.log_likelihood()
    m.optimize(max_iters=5)
    assert -m.log_likelihood() < b0
    assert np.all(m.latent_variance.values > 0)


def test_unsupported_kernels_and_uncertain_test_points():
    import gpy_b200
    Y = np.load(os.path.join(GOLD, "default_p1.npz"))["Y"][:20]
    with pytest.raises(NotImplementedError):
        gpy_b200.BayesianGPLVM(Y, 2, num_inducing=4, kernel=gpy_b200.Matern32(2), engine=HostEngine())
    with pytest.raises(NotImplementedError):
        gpy_b200.BayesianGPLVM(Y, 2, num_inducing=4, kernel=gpy_b200.RBF(2) + gpy_b200.Bias(2), engine=HostEngine())
    m = gpy_b200.BayesianGPLVM(Y, 2, num_inducing=4, engine=HostEngine())

    class NormalPosterior(object):
        mean = np.zeros((3, 2))
        variance = np.ones((3, 2))
    with pytest.raises(NotImplementedError):
        m.predict(NormalPosterior())
