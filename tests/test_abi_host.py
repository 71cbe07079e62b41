"""CPU tests: the C-ABI library loads and exports every symbol include/gpx.h declares (no compute without a GPU),
host-side logic of the plugin mirror, and loud failure when no device is present."""
import os
import re

import numpy as np
import pytest

import gpy_b200
from gpy_b200 import _ffi
from gpy_b200.param import Logexp, Param

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "gpx.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gpx_[A-Za-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    names = _declared_functions()
    assert len(names) >= 15
    L = _ffi.lib()
    for n in names:
        assert hasattr(L, n), "libgpx.so does not export %s" % n
    assert set(names) == set(_ffi.EXPORTS), "ctypes table and header disagree: %s" % (set(names) ^ set(_ffi.EXPORTS))
    assert b"sm_90a" in L.gpx_version()


def test_built_for_sm_90a_only():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", _ffi.LIB_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout
    assert not re.search(r"sm_(?!90a)\d+", out.stdout)


def test_no_gpu_fails_loudly(have_gpu):
    if have_gpu:
        pytest.skip("a GPU is present")
    with pytest.raises(_ffi.GpxError):
        _ffi.Engine(0)
    with pytest.raises(_ffi.GpxError):
        _ffi.kern_K("rbf", False, 1.0, 1.0, np.zeros((4, 2)))


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "gpy_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), os.path.join(dp, f)


def test_logexp_and_param():
    x = np.linspace(-30, 60, 40)
    np.testing.assert_allclose(Logexp.finv(Logexp.f(x)), x, rtol=1e-9, atol=1e-6)
    p = Param("variance", 2.0)
    assert p.size == 1 and float(p) == 2.0 and (p + 1)[0] == 3.0
    p.gradient = np.array([0.5])
    assert p.gradient[0] == 0.5


def test_kernel_constructor_contract():
    """GPy/kern/src/stationary.py:61-81: lengthscale defaults / shapes, parameter link order variance, lengthscale."""
    k = gpy_b200.RBF(3)
    assert k.lengthscale.size == 1 and not k.ARD and k.parameter_names() == ["rbf.variance", "rbf.lengthscale"]
    k = gpy_b200.Matern52(4, ARD=True)
    assert k.lengthscale.size == 4
    k = gpy_b200.Matern32(4, lengthscale=2.0, ARD=True)
    np.testing.assert_array_equal(k.lengthscale.values, 2.0 * np.ones(4))
    with pytest.raises(AssertionError):
        gpy_b200.RBF(3, lengthscale=[1.0, 2.0])
    with pytest.raises(AssertionError):
        gpy_b200.Exponential(3, lengthscale=[1.0, 2.0], ARD=True)
    k = gpy_b200.RBF(2, active_dims=[0, 2])
    X = np.arange(12.0).reshape(4, 3)
    np.testing.assert_array_equal(k._slice_X(X), X[:, [0, 2]])
    np.testing.assert_array_equal(k.Kdiag(X), np.ones(4))   # host-only entry point (stationary.py:170-173)


def test_device_gradient_handle_shortcut():
    from gpy_b200.kern import DeviceGradient
    k = gpy_b200.RBF(2, variance=1.5, lengthscale=[1.0, 2.0], ARD=True)
    h = DeviceGradient(None, k._state_key(), 0.25, np.array([1.0, -2.0]), 10)
    k.update_gradients_full(h, np.zeros((10, 2)))
    assert k.variance.gradient[0] == 0.25
    np.testing.assert_array_equal(k.lengthscale.gradient, [1.0, -2.0])
    assert h.shape == (10, 10)
    k.update_gradients_diag(np.ones(10), np.zeros((10, 2)))
    assert k.variance.gradient[0] == 10.0 and np.all(k.lengthscale.gradient == 0)
