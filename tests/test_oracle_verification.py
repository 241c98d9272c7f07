"""The verification oracle (oracle/verification.py) against the live reference where it is present:
every accumulation of CRPS, the rank histogram (with the reference's draws and the random state
after them), the reliability diagram and the ROC curve, bit for bit."""
import warnings

import numpy as np
import pytest

from oracle import verification as ora
from verification_cases import ensemble_cases, prob_cases, reference

ENS = ensemble_cases()
PROB = prob_cases()


@pytest.fixture(scope="module")
def ref():
    r = reference()
    if r is None:
        pytest.skip("the reference is not present")
    return r


def test_pairwise_matches_numpy_sum():
    rng = np.random.default_rng(0)
    for n in list(range(0, 300)) + [1000, 8191, 8192, 8193, 20000]:
        for dt in (np.float32, np.float64):
            x = (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 3, n)).astype(dt)
            assert ora.pairwise(x).tobytes() == np.sum(x).tobytes(), (n, dt)
    A = rng.standard_normal((50, 257))
    assert np.array_equal(ora.pairwise(A), np.sum(A, axis=1))


@pytest.mark.parametrize("name", sorted(ENS))
def test_crps_and_rankhist(ref, name):
    ps, es = ref
    X_f, X_o, X_min = ENS[name]
    d = ps.CRPS_init()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        ps.CRPS_accum(d, X_f, X_o)
    s, n = ora.crps(X_f, X_o)
    if X_f[0].size <= 5000:
        assert ora.crps_loop(X_f, X_o).tobytes() == ora.crps_pixels(X_f, X_o).tobytes()
    assert np.float64(d["CRPS_sum"]).tobytes() == np.float64(s).tobytes() and d["n"] == n
    for xm in (None, X_min):
        counts, pairs = ora.rankhist(X_f, X_o, xm)
        np.random.seed(5)
        h = es.rankhist_init(X_f.shape[0], xm)
        es.rankhist_accum(h, X_f, X_o)
        after = np.random.random()
        np.random.seed(5)
        u = np.random.uniform(size=len(pairs)) if len(pairs) else np.zeros(0)
        assert (np.random.random() == after) == True  # noqa: E712 -- one draw of len(pairs) exactly when tied
        assert np.array_equal(h["n"], ora.rankhist(X_f, X_o, xm, u)), name


@pytest.mark.parametrize("name", sorted(PROB))
def test_reldiag_and_roc(ref, name):
    ps, _ = ref
    P, O, X_min, nb = PROB[name]
    r = ps.reldiag_init(X_min, nb, 0)
    ps.reldiag_accum(r, P, O)
    count, above, sums = ora.reldiag(P, O, X_min, r["bin_edges"])
    assert np.array_equal(r["num_idx"], count) and np.array_equal(r["Y_sum"], above)
    assert r["X_sum"].tobytes() == sums.astype(np.float64).tobytes()
    roc = ps.ROC_curve_init(X_min, nb)
    ps.ROC_curve_accum(roc, P, O)
    got = ora.roc(P, O, X_min, roc["prob_thrs"])
    for key, v in zip(("hits", "misses", "false_alarms", "corr_neg"), got):
        assert np.array_equal(roc[key], v), key
