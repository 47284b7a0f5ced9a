"""The discrete Bayes oracle (oracle/discrete_bayes.py) against the reference's golden vectors
(tests/golden/make_golden_discrete_bayes.py): wrap-mode predict, update and normalize bit for bit in fp32 and fp64,
constant mode within the reference's spline roundoff (1e-15 absolute in fp64, 1 ulp in fp32)."""
import numpy as np
import pytest

from oracle import discrete_bayes as odb

CASES = ["db_wrap_k3_f64", "db_wrap_k4_f32", "db_wrap_klong_f64", "db_const_k5_f64", "db_const_k2_f32",
         "db_onebin_f64"]


def const_close(got, want):
    """Within the reference's spline-shift roundoff: 1e-15 absolute in fp64, 1 ulp in fp32 (NaN where it has NaN)."""
    assert got.dtype == want.dtype
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    if want.dtype == np.float32:
        assert np.all(np.abs(got[ok].astype(np.float64) - want[ok]) <= np.spacing(np.abs(want[ok])).astype(np.float64))
    else:
        assert np.all(np.abs(got[ok] - want[ok]) <= 1e-15)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(golden, name):
    g = golden(name)
    mode = "wrap" if int(g["wrap"]) else "constant"
    cval = float(g["cval"])
    prior, _ = odb.step_bank(g["pdf"], g["kernel"], g["offsets"], mode=mode, cval=cval)
    post, sums = odb.step_bank(g["prior"], likelihood=g["lik"], normalize=True)
    norm, _ = odb.step_bank(g["pdf"], normalize=True)
    assert prior.dtype == g["pdf"].dtype
    if mode == "wrap":
        np.testing.assert_array_equal(prior, g["prior"])
    else:
        const_close(prior, g["prior"])
    np.testing.assert_array_equal(post, g["post"])                 # update and normalize: bit for bit, NaN included
    np.testing.assert_array_equal(norm, g["norm"])
    assert sums.shape == (g["pdf"].shape[0],)


def test_goldens_cover_the_issue_cases(golden):
    """The fixtures hold what they are meant to pin: an all-zero row (NaN), an even kernel, K > M with skipped
    weights, offsets beyond the row both ways, both modes and dtypes, a one-bin pdf."""
    g = golden("db_wrap_k3_f64")
    assert np.isnan(g["post"]).any() and np.isnan(g["norm"]).any()
    assert (g["offsets"] < 0).any() and (g["offsets"] >= g["pdf"].shape[1]).any()
    assert golden("db_wrap_k4_f32")["kernel"].shape[1] % 2 == 0
    k = golden("db_wrap_klong_f64")
    assert k["kernel"].shape[1] > k["pdf"].shape[1] and np.isnan(k["kernel"]).any() and (k["kernel"] == 0).any()
    assert golden("db_onebin_f64")["pdf"].shape[1] == 1
    assert not int(golden("db_const_k5_f64")["wrap"]) and golden("db_const_k2_f32")["pdf"].dtype == np.float32


def test_scipy_footprint_rule_is_what_the_oracle_skips():
    """A weight of 1e-17 (below DBL_EPSILON) is not a product of zero: scipy drops it, and so does the oracle.
    Multiplying it in would move a 1e30 bin's neighbours by 1e13."""
    pdf = np.array([1e30, 1.0, 2.0])
    out = odb.predict_row(pdf, 0, [1e-17, 1.0, 0.0])
    np.testing.assert_array_equal(out, pdf)
    out = odb.predict_row(pdf, 0, [np.nextafter(np.finfo(float).eps, 1), 1.0, 0.0])
    assert out[2] > 1e13
