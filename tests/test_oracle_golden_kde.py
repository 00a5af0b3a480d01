"""The oracle's KDEMove branch (``oracle/redblue.py``) vs the unmodified reference's ``KDEMove`` with scipy's
``gaussian_kde`` (golden vectors by ``oracle/gen_golden_kde.py``).  Accept masks and the complement ranks of the
kernel centres are equal bit for bit; coordinates and log-probabilities agree to 1e-12 (the oracle's Cholesky
factor of ``cov * bw**2`` and its log-sum-exp are not the reference's LAPACK / Cython calls)."""
import numpy as np
import pytest

from kde_util import kde_names, kde_oracle, load_kde


def test_every_case_is_there():
    assert len(kde_names()) == 6


@pytest.mark.parametrize("name", kde_names())
def test_oracle_matches_reference(name):
    g = load_kde(name)
    s = kde_oracle(g)
    np.testing.assert_array_equal(s.log_prob, g["lp0"])
    for k in range(g["chain"].shape[0]):
        with np.errstate(invalid="ignore"):
            acc = s.run(1)
        assert np.array_equal(acc, g["accepted"][k]), (name, k)
        np.testing.assert_allclose(s.coords, g["chain"][k], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(s.log_prob, g["log_prob"][k], rtol=1e-12, atol=1e-12)
        # the oracle runs the reference's previous state from here on: no drift between steps
        s.coords, s.log_prob = g["chain"][k].copy(), g["log_prob"][k].copy()


@pytest.mark.parametrize("name", kde_names())
def test_kernel_centres_match_reference(name):
    # complement rank of every proposal's kernel centre, every split of the first three steps
    g = load_kde(name)
    s = kde_oracle(g)
    ranks = []
    orig = s._kde

    def tap(*a, **kw):
        out = orig(*a, **kw)
        ranks.append(s.taps["rank"])
        return out

    s._kde = tap
    with np.errstate(invalid="ignore"):
        for k in range(3):
            s.run(1)
            s.coords, s.log_prob = g["chain"][k].copy(), g["log_prob"][k].copy()
    got = np.concatenate(ranks) if ranks else np.zeros(0, np.int64)
    assert np.array_equal(got, g["trace_kde_choice"])
