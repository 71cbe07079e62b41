"""gpy_b200 — H100 exact-GP engine behind GPy's kernel / exact-inference plugin interface.

Host side (Python, mirrors the reference's operator interface for the hot path) over a ctypes C ABI
(include/gpx.h) into hand-written sm_90a CUDA (gpy_b200/csrc). No CPU fallback: importing works everywhere,
computing requires libgpx.so and an H100.
"""
from . import _ffi  # noqa: F401
from ._ffi import Engine, GpxError, kern_K, kern_Kdiag, kern_grad_full  # noqa: F401

from .kern import (RBF, Exponential, Matern32, Matern52, RatQuad, StdPeriodic, Stationary, DeviceGradient,  # noqa: F401
                   Add, Prod, White, Bias, Kern, CombinationKernel)
from .inference import (ExactGaussianInference, Gaussian, HeteroscedasticGaussian, MixedNoise,  # noqa: F401
                        PosteriorExact)
from .model import GP, GPHeteroscedasticRegression, GPRegression  # noqa: F401
from .sparse import FITC, SparseGPRegression, VarDTC  # noqa: F401
from .laplace import Bernoulli, Laplace, PosteriorLaplace, StudentT  # noqa: F401
from .ep import EP, EPDTC, GPClassification, PosteriorEP, SparseGPClassification  # noqa: F401
from .svgp import SVGP, SVGPInference  # noqa: F401
from .gplvm import GPLVM, SparseGPLVM  # noqa: F401
from .bgplvm import BayesianGPLVM  # noqa: F401
from .vargauss import GPVariationalGaussianApproximation, VarGauss  # noqa: F401

__version__ = "0.1.0"
