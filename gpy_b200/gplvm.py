"""The Gaussian-process latent variable model on the device.

Mirrors:
    GPy.models.GPLVM                        GPy/models/gplvm.py:10-49
    GPy.util.initialization.initialize_latent   GPy/util/initialization.py:11-60 ('PCA' and 'random')
    GPy.util.pca.PCA                        GPy/util/pca.py:19-88 (the parts initialize_latent uses)
An evaluation is the exact evaluation of GPRegression plus the input gradient X.gradient = kern.gradients_X(dL_dK, X, None)
(gplvm.py:47-49), which the kernels take from the device (gpx_exact_grad_X) because dL_dK is the evaluation's
DeviceGradient: nothing of size N^2 reaches the host. The latent inputs are a parameter without a transform, linked first,
so the gradient and the optimizer space are ordered [latent_mean, kernel.., noise] as in the reference.

    GPy.models.SparseGPLVM                  GPy/models/sparse_gplvm.py:9-34
is the sparse model (VarDTC) with the latent inputs as a parameter: X.gradient = kern.gradients_X(dL_dKnm, X, Z)
(sparse_gplvm.py:34) is reduced on the device from the dL_dKnm the evaluation left there (gpx_sparse_grad_X); the
gradients_X_diag term of :33 is zero for every kernel the sparse evaluation takes.
"""
import warnings

import numpy as np

from .inference import Gaussian
from .kern import RBF, Bias
from .model import GP
from .param import Param
from .sparse import SparseGPRegression


class PCA(object):
    """GPy.util.pca.PCA (pca.py:19-88): principal components of the standardised data, the primal or the dual eigenproblem
    by shape, eigenvalues in descending order."""

    def __init__(self, X):
        self.mu = None
        self.sigma = None
        X = self.center(X)
        if X.shape[0] >= X.shape[1]:
            self.eigvals, self.eigvectors = np.linalg.eigh(np.einsum("ji,jk->ik", X, X))     # :48-49
        else:
            self.eigvals, self.eigvectors = self._dual_eig(X)
        self.sort = np.argsort(self.eigvals)[::-1]
        self.eigvals = self.eigvals[self.sort]
        self.eigvectors = self.eigvectors[:, self.sort]
        self.fracs = self.eigvals / self.eigvals.sum()
        self.Q = self.eigvals.shape[0]

    def center(self, X):
        """pca.py:34-46: missing values take the column mean, then every column is standardised"""
        X = X.copy()
        inan = np.isnan(X)
        if self.mu is None:
            X_ = np.ma.masked_array(X, inan)
            self.mu = X_.mean(0).base
            self.sigma = X_.std(0).base
        for col, nan, mu in zip(X.T, inan.T, self.mu):
            col[nan] = mu
        X = X - self.mu
        return X / np.where(self.sigma == 0, 1e-30, self.sigma)

    def _dual_eig(self, X):
        """pca.py:51-58"""
        dual_eigvals, dual_eigvects = np.linalg.eigh(np.einsum("ij,kj->ik", X, X))
        relevant = np.argsort(np.abs(dual_eigvals))[-X.shape[1]:]
        eigvals = dual_eigvals[relevant]
        eigvects = dual_eigvects[:, relevant]
        eigvects = (1. / np.sqrt(X.shape[0] * np.abs(eigvals))) * X.T.dot(eigvects)
        eigvects /= np.sqrt(np.diag(eigvects.T.dot(eigvects)))
        return eigvals, eigvects

    def project(self, X, Q=None):
        """pca.py:60-70"""
        if Q is None:
            Q = self.Q
        if Q > X.shape[1]:
            raise IndexError("requested dimension larger then input dimension")
        return self.center(X).dot(self.eigvectors[:, :Q])


def initialize_latent(init, input_dim, Y):
    """initialization.py:11-60 -> (X (N x input_dim), fracs): the random draw comes first, from numpy's global generator,
    then PCA overwrites the leading columns, so a seeded script gets the reference's X. 'empirical_samples' is not served."""
    Xr = np.asfortranarray(np.random.normal(0, 1, (Y.shape[0], input_dim)))
    if init == "PCA":
        p = PCA(Y)
        PC = p.project(Y, min(input_dim, Y.shape[1]))
        Xr[:PC.shape[0], :PC.shape[1]] = PC
        var = 0.1 * p.fracs[:input_dim]
    elif init == "empirical_samples":
        raise NotImplementedError("initialize_latent: 'empirical_samples' (deprecated in the reference) is not served")
    else:
        if init != "random":
            warnings.warn("%s is not a valid initialization method. Supoprt for anything else than 'PCA' or 'random' will "
                          "be removed in the next major release." % init, DeprecationWarning)
        var = Xr.var(0)
    Xr -= Xr.mean(0)
    Xr /= Xr.std(0)
    return Xr, var / var.max()


class GPLVM(GP):
    """GPy.models.GPLVM (gplvm.py:10-49): a GP regression of Y on latent inputs X that are themselves parameters. The
    default kernel is RBF(input_dim, lengthscale=fracs, ARD=input_dim > 1) + Bias(input_dim, exp(-2)); the likelihood is
    Gaussian with unit variance."""

    def __init__(self, Y, input_dim, init="PCA", X=None, kernel=None, name="gplvm", Y_metadata=None, normalizer=False,
                 device=0, engine=None):
        if X is None:
            X, fracs = initialize_latent(init, input_dim, np.asarray(Y, dtype=np.float64))
        else:
            fracs = np.ones(input_dim)
        if kernel is None:
            kernel = RBF(input_dim, lengthscale=fracs, ARD=input_dim > 1) + Bias(input_dim, np.exp(-2))
        X = np.array(X, dtype=np.float64)
        self.latent_mean = Param("latent_mean", X, transform=None)
        super(GPLVM, self).__init__(X, Y, kernel, Gaussian(), name="GPLVM", device=device, engine=engine,
                                    Y_metadata=Y_metadata, normalizer=normalizer)
        self._links.insert(0, self.latent_mean)                   # link_parameter(self.X, index=0)
        self.latent_mean._observers.append(self._child_changed)

    def parameters_changed(self):
        """gplvm.py:46-49: the GP's evaluation, then the input gradient"""
        self.X = self.latent_mean.values
        super(GPLVM, self).parameters_changed()
        self.latent_mean.gradient = self.kern.gradients_X(self.grad_dict["dL_dK"], self.X, None)


class SparseGPLVM(SparseGPRegression):
    """GPy.models.SparseGPLVM (sparse_gplvm.py:9-34): SparseGPRegression of Y on latent inputs X that are themselves a
    parameter ('latent space', linked first, no transform). The seeded draws follow the reference: initialize_latent's,
    then SparseGPRegression's permutation for Z. The default kernel is SparseGPRegression's RBF(input_dim), isotropic.
    Gradient and optimizer order: [latent space, inducing inputs, kernel.., noise]."""

    def __init__(self, Y, input_dim, X=None, kernel=None, init="PCA", num_inducing=10, device=0, engine=None):
        if X is None:
            X, fracs = initialize_latent(init, input_dim, np.asarray(Y, dtype=np.float64))
        X = np.array(X, dtype=np.float64)
        self.latent_space = Param("latent space", X, transform=None)
        self.latent_space.values = X                                   # keep the N x Q shape
        self.latent_space.gradient = np.zeros_like(X)
        super(SparseGPLVM, self).__init__(X, Y, kernel=kernel, num_inducing=num_inducing, device=device, engine=engine)
        self._links.insert(0, self.latent_space)                      # link_parameter(self.X, 0)
        self.latent_space._observers.append(self._child_changed)

    def _free(self):
        return [self.latent_space, self.Z]

    def parameters_changed(self):
        """sparse_gplvm.py:29-34: the sparse evaluation on the current latent inputs, then their gradient"""
        self.X = self.latent_space.values
        super(SparseGPLVM, self).parameters_changed()
        dX = self.inference_method.engine.sparse_grad_X()
        if "part_grads" not in self.grad_dict:                        # a lone kernel saw its active dims only
            full = np.zeros_like(self.X)
            full[:, self.kern.active_dims] = dX
            dX = full
        self.latent_space.gradient = dX
