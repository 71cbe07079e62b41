"""The wide-composite oracle without a GPU: tests/wide_composites_oracle.py against the reference's own numbers in
tests/golden/wide_composites (composites on 64 input columns: RatQuad ARD on 64 dims, StdPeriodic ARD1 + ARD2 on 32 dims x
RBF, eight parts of 8 dims, predictive gradients at sumD 17 and 64 with 8 outputs), so that the GPU tests of
tests/test_gpu_wide_composites.py rest on a checked oracle; and the Python restatement of the device's instantiation
choice against the formulas include/gpx.h documents."""
import glob
import os

import numpy as np
import pytest

import predictive_gradients_oracle as po
import wide_composites_oracle as wo

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "wide_composites", "*.npz")))
TOL = 1e-12


def test_every_fixture_is_there():
    names = {os.path.basename(p)[:-4] for p in FIXTURES}
    assert names == set(wo.fixture_kernels())
    assert sum(os.path.getsize(p) for p in FIXTURES) < 1.2e6


def _rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


@pytest.mark.parametrize("path", FIXTURES, ids=lambda p: os.path.basename(p)[:-4])
def test_oracle_matches_the_reference(path):
    f = np.load(path)
    parts = wo.fixture_kernels()[str(f["kernel"])]
    X, Y, noise = f["X"], f["Y"], float(f["noise"])
    X2, Y2 = wo.data(X.shape[0], X.shape[1], Y.shape[1], int(f["seed"]))
    np.testing.assert_array_equal(X, X2)          # the inputs are those of wo.data
    np.testing.assert_array_equal(Y, Y2)
    if "lml" in f.files:
        lml, g, res = wo.exact_eval(X, Y, parts, noise)
        assert abs(lml - float(f["lml"])) <= TOL * abs(lml)
        assert g.size == f["grad"].size
        np.testing.assert_allclose(g, f["grad"], rtol=1e-10, atol=TOL * np.abs(f["grad"]).max())
        assert _rel(res["alpha"], f["alpha"]) <= 1e-11
        return
    kern = wo.WideOracle(parts)
    wv, wi = po.exact_posterior(kern, X, Y, noise)
    mj, vj = po.jacobians(kern, wv, wi, f["Xnew"], X)
    assert _rel(mj, f["mean_jac"]) <= 1e-11
    assert _rel(vj, f["var_jac"]) <= 1e-11


def test_fixture_routes():
    """what the fixtures exercise on the device: the widest instantiations"""
    k = wo.fixture_kernels()
    assert wo.grad_route(k["ratquad_ard64"], 0) == (64, True) and wo.part_nred(k["ratquad_ard64"][0]) == 67
    assert wo.grad_route(k["periodic32_x_rbf"], 0) == (64, True) and wo.part_nacc(k["periodic32_x_rbf"][0]) == 64
    assert [wo.grad_route(k["eight_parts64"], i) for i in range(8)] == [(8, False)] * 8
    assert wo.sum_dims(k["eight_parts64"]) == 64
    assert wo.pred_grad_route(wo.sum_dims(k["pg_sumd17"])) == (32, 1)
    assert wo.pred_grad_route(wo.sum_dims(k["pg_sumd64"])) == (64, 1)


# ---- the restatement of the instantiation choice ----------------------------------------------------------------------
def _header():
    with open(os.path.join(os.path.dirname(HERE), "include", "gpx.h")) as fh:
        return fh.read()


@pytest.mark.parametrize("sumD", [1, 3, 8, 9, 16, 17, 32, 33, 64])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 7, 8])
def test_channel_groups_follow_the_documented_launch_count(sumD, P):
    """gpx.h: R = ceil((P + 1) / g) + 1 reduction launches, g = 4 channels per launch when the stacked active dims are
    <= 8, 2 when <= 16, else 1; every channel in exactly one group, the variance channel (P) in the last"""
    h = _header()
    assert "R = ceil((P + 1) / g) + 1" in h and "g = 4 channels per launch" in h and "<= 8, 2 when <= 16, else 1" in h
    g = 4 if sumD <= 8 else 2 if sumD <= 16 else 1
    assert wo.pred_grad_launches(sumD, P) == -(-(P + 1) // g) + 1
    groups = wo.channel_groups(sumD, P)
    assert [c for c0, n, _ in groups for c in range(c0, c0 + n)] == list(range(P + 1))
    assert [v for _, _, v in groups] == [False] * (len(groups) - 1) + [True]
    dreg, nch = wo.pred_grad_route(sumD)
    assert nch == g and (dreg * nch <= 32 or nch == 1) and dreg >= sumD


@pytest.mark.parametrize("nrows,ncols,sms,want", [
    (1025, 4097, 132, (43, 96, 65)), (2049, 4097, 132, (26, 160, 97)), (1, 4097, 132, (129, 32, 1)),
    (129, 4097, 132, (129, 32, 1)), (700, 300, 132, (10, 32, 12)), (1025, 4097, 114, (43, 96, 65)),
    (1025, 4097, 16, (8, 544, 289))])
def test_column_chunks(nrows, ncols, sms, want):
    nchunk, mchunk, last = wo.gradx_chunks(nrows, ncols, sms)
    assert (nchunk, mchunk, last) == want
    assert mchunk % 32 == 0 and 0 < last <= mchunk and (nchunk - 1) * mchunk + last == ncols
    ntile = -(-nrows // 128)
    assert nchunk * ntile <= max(4 * sms + ntile, ntile * -(-ncols // 32))   # ~4 waves of CTAs, never more than needed


def test_register_widths():
    assert [wo.width(d) for d in (0, 1, 8, 9, 16, 17, 32, 33, 64)] == [8, 8, 8, 16, 16, 32, 32, 64, 64]
    sp = wo.stdperiodic(list(range(8)), 0, False, False)
    assert wo.part_nacc(sp) == 16 and wo.grad_route([sp], 0) == (16, True)       # the period / lengthscale split needs 2 D
    sp9 = wo.stdperiodic(list(range(9)), 0, True, True)
    assert wo.grad_route([sp9], 0) == (32, True)
    iso = wo.stationary("rbf", list(range(23)), 0, False)
    assert wo.part_nacc(iso) == 0 and wo.grad_route([iso], 0) == (32, False)      # the row point's inputs need D
    with pytest.raises(AssertionError):
        wo.width(65)
