"""Bayesian GPLVM (GPy/models/bayesian_gplvm.py:20-101) on the device.

The latent inputs are the Gaussians q(x_n) = N(mu_n, diag(S_n)). One evaluation is one gpx_sparse_eval_psi call: the RBF
psi-statistics, the uncertain-input VarDTC bound and its gradients w.r.t. the kernel, the noise, Z, mu and S. The
NormalPrior KL term (variational.py:29-37) is O(N Q) and is formed on the host.
"""
import numpy as np

from .gplvm import initialize_latent
from .kern import RBF, part_descriptor
from .param import Logexp, Param
from .sparse import LazySparsePosterior, SparseGPRegression


def normal_prior_kl(mu, S):
    """NormalPrior.KL_divergence (variational.py:29-32) and the gradients it adds to the bound's (:34-37)"""
    kl = 0.5 * (np.square(mu).sum() + (S - np.log(S)).sum()) - 0.5 * mu.size
    return kl, -mu, -0.5 * (1.0 - 1.0 / S)


class BayesianGPLVM(SparseGPRegression):
    """GPy.models.BayesianGPLVM with a Gaussian likelihood and one RBF kernel on all latent columns. The seeded draws
    follow the reference: initialize_latent's, then uniform(0, .1) for X_variance, then the permutation for Z. The default
    kernel is RBF(input_dim, lengthscale=1/fracs, ARD=True). Parameter and gradient order: [latent space mean, latent
    space variance (Logexp), inducing inputs, rbf.., noise]."""

    def __init__(self, Y, input_dim, X=None, X_variance=None, init="PCA", num_inducing=10, Z=None, kernel=None,
                 device=0, engine=None):
        Y = np.asarray(Y, dtype=np.float64)
        if X is None:
            X, fracs = initialize_latent(init, input_dim, Y)
        else:
            fracs = np.ones(input_dim)
        X = np.array(X, dtype=np.float64)
        if X_variance is None:
            X_variance = np.random.uniform(0, .1, X.shape)
        if Z is None:
            Z = np.random.permutation(X.copy())[:num_inducing]
        Z = np.array(Z, dtype=np.float64)
        assert Z.shape[1] == X.shape[1]
        if kernel is None:
            kernel = RBF(input_dim, lengthscale=1. / fracs, ARD=True)
        if type(kernel) is not RBF or not np.array_equal(kernel.active_dims, np.arange(X.shape[1])):
            raise NotImplementedError("gpy_b200.BayesianGPLVM takes one RBF kernel on all latent columns (the device's "
                                      "psi-statistics)")
        self.latent_mean = Param("latent space mean", X, transform=None)
        self.latent_mean.values = X
        self.latent_mean.gradient = np.zeros_like(X)
        S = np.array(X_variance, dtype=np.float64)
        self.latent_variance = Param("latent space variance", S)
        self.latent_variance.values = S
        self.latent_variance.gradient = np.zeros_like(S)
        self._ready = False
        super(BayesianGPLVM, self).__init__(X, Y, kernel=kernel, Z=Z, num_inducing=num_inducing, device=device,
                                            engine=engine, name="bayesian gplvm")
        self._links.insert(0, self.latent_variance)
        self._links.insert(0, self.latent_mean)                      # link_parameter(self.X, index=0)
        for p in (self.latent_mean, self.latent_variance):
            p._observers.append(self._child_changed)
        self._ready = True
        self.parameters_changed()

    def parameters_changed(self):
        """sparse_gp.py:76-107 with uncertain inputs on the device, then bayesian_gplvm.py:86-101 (minus the KL term)"""
        if not self._ready:
            return
        mu, S = self.latent_mean.values, self.latent_variance.values
        self.X = mu
        im = self.inference_method
        eng = im.engine
        if not im._data_key.matches(mu, self.Y):
            if self.Y.shape[1] > 8:
                eng.set_option("sparse_wide", 1)
            eng.sparse_set_data(mu, self.Y)
            im._data_key.remember(mu, self.Y)
        noise = float(np.squeeze(np.asarray(self.likelihood.gaussian_variance(self.Y_metadata))))
        Z = self.Z.values
        lml, grad, dZ, dmu, dS = eng.sparse_eval_psi(part_descriptor(self.kern, 0), S, Z, noise)
        kl, kmu, kS = normal_prior_kl(mu, S)
        self.posterior = LazySparsePosterior(eng, self.kern._state_key(), Z)
        self._log_marginal_likelihood = lml - kl
        self.grad_dict = {"dvariance": grad[0], "dlengthscale": grad[1:-1], "dZ": dZ, "dL_dthetaL": float(grad[-1])}
        self.likelihood.update_gradients(float(grad[-1]))
        self.kern.variance.gradient = np.atleast_1d(grad[0])
        self.kern.lengthscale.gradient = np.atleast_1d(grad[1:-1])
        self.Z.gradient = dZ
        self.latent_mean.gradient = dmu + kmu
        self.latent_variance.gradient = dS + kS

    def _free(self):
        return [self.latent_mean]

    # the optimizer space: mean and Z unconstrained, everything else through Logexp
    def _transformed(self):
        return [p is not self.latent_mean and p is not self.Z for p in self._flat()]

    @property
    def optimizer_array(self):
        return np.concatenate([(Logexp.finv(p.values) if t else p.values).reshape(-1)
                               for p, t in zip(self._flat(), self._transformed())])

    @optimizer_array.setter
    def optimizer_array(self, x):
        i = 0
        for p, t in zip(self._flat(), self._transformed()):
            v = x[i:i + p.values.size].reshape(p.values.shape)
            p.values[...] = Logexp.f(v) if t else v
            i += p.values.size
        self.parameters_changed()

    def _grads_transformed(self):
        g = []
        for p, t in zip(self._flat(), self._transformed()):
            d = np.asarray(p.gradient, dtype=np.float64).reshape(-1)
            g.append(d * Logexp.gradfactor(p.values).reshape(-1) if t else d)
        return -np.concatenate(g)

    def predict(self, Xnew, full_cov=False, include_likelihood=True, Y_metadata=None, kern=None, likelihood=None):
        """gp.py:290-365 at certain latent points through the device's sparse predict"""
        if hasattr(Xnew, "mean") and hasattr(Xnew, "variance") and not isinstance(Xnew, np.ndarray):
            raise NotImplementedError("gpy_b200.BayesianGPLVM predicts at certain latent points only (a NormalPosterior "
                                      "Xnew needs the psi-statistics of the test points)")
        return super(BayesianGPLVM, self).predict(Xnew, full_cov, include_likelihood, Y_metadata, kern, likelihood)
