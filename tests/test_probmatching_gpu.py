"""GPU: probability matching (csrc/probmatching.cu behind postprocessing/probmatching.py) against the
oracle (oracle/probmatching.py) and the reference's stored outputs, warnings and random draws
(tests/golden/probmatching_golden.npz), bit for bit; on cases with tied initial values the stable-order
output bit for bit, and the reference's within every tie group."""
import warnings

import numpy as np
import pytest
import torch

from conftest import assert_bits_equal
from oracle import probmatching as ora
from probmatching_cases import CASES, ERRORS, LARGE, build_case, rain, seed_of
from test_host_logic_probmatching import outcome
from test_oracle_probmatching import check_golden, golden, oracle_call

pytestmark = pytest.mark.gpu


def _pm():
    from pysteps_b200.postprocessing import probmatching
    return probmatching


@pytest.mark.parametrize("name", CASES)
def test_golden_case(name):
    got, warned, nxt = outcome(name)
    g = golden()
    if name in ERRORS:
        assert isinstance(got, Exception) and f"{type(got).__name__}: {got}" == str(g[name + "/error"]), got
    else:
        assert isinstance(got, np.ndarray), got
        check_golden(name, got)
        if name in LARGE:  # the whole output against the oracle
            assert_bits_equal(got, oracle_call(name), name)
    assert warned == list(g[name + "/warnings"]), name
    assert nxt == g[name + "/next"], "the random state after the call differs from the reference's"


@pytest.mark.parametrize("name", ["match_f32_2048_more_target", "match_ignore_mask", "match_nan_target",
                                  "match_ties_small", "resample_nan_first", "resample_f32"])
def test_cuda_tensor_input(name):
    fn, args, kw = build_case(name)
    if fn == "match":
        d = [torch.from_numpy(a).cuda() for a in args]
        if "ignore_indices" in kw:
            kw = dict(kw, ignore_indices=torch.from_numpy(kw["ignore_indices"]).cuda())
        got = _pm().nonparam_match_empirical_cdf(*d, **kw)
    else:
        np.random.seed(seed_of(name))
        got = _pm().resample_distributions(torch.from_numpy(args[0]).cuda(), torch.from_numpy(args[1]).cuda(),
                                           args[2], **kw)
    assert isinstance(got, torch.Tensor) and got.is_cuda
    assert_bits_equal(got.cpu().numpy(), oracle_call(name), name)


@pytest.mark.parametrize("n", [1, 2, 4095, 4096, 4097, 65537, 1000003])
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_sizes_off_the_tile(n, dtype):
    x = rain((n,), n, dtype)
    t = rain((n,), n + 1, dtype, dry=0.3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        assert_bits_equal(_pm().nonparam_match_empirical_cdf(x, t), ora.nonparam_match_empirical_cdf(x, t))
        assert_bits_equal(_pm().nonparam_match_empirical_cdf(t, x), ora.nonparam_match_empirical_cdf(t, x))
    np.random.seed(n)
    got = _pm().resample_distributions(x, t, 0.4)
    np.random.seed(n)
    assert_bits_equal(got, ora.resample_distributions(x, t, np.random.binomial(1, 0.4, n)))


def test_all_wet_and_all_dry():
    x_wet = rain((300, 300), 1, dry=0.0) + 1.0
    x_dry = np.zeros((300, 300))
    t = rain((300, 300), 2)
    for x in (x_wet, x_dry):
        for tt in (t, np.zeros_like(t), rain((300, 300), 3, dry=0.0)):
            assert_bits_equal(_pm().nonparam_match_empirical_cdf(x, tt), ora.nonparam_match_empirical_cdf(x, tt))


def test_repeated_calls_are_bit_identical():
    x = torch.from_numpy(rain((1024, 1024), 4, np.float32)).cuda()
    t = torch.from_numpy(rain((1024, 1024), 5, np.float32, dry=0.4)).cuda()
    first = _pm().nonparam_match_empirical_cdf(x, t)
    for _ in range(3):
        assert torch.equal(_pm().nonparam_match_empirical_cdf(x, t).view(torch.int64), first.view(torch.int64))


def test_non_default_stream():
    x, t = rain((512, 512), 6), rain((512, 512), 7, dry=0.3)
    want = ora.nonparam_match_empirical_cdf(x, t)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dx, dt = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
        got = _pm().nonparam_match_empirical_cdf(dx, dt)
        np.random.seed(1)
        r = _pm().resample_distributions(dx, dt, 0.5)
    s.synchronize()
    assert_bits_equal(got.cpu().numpy(), want)
    np.random.seed(1)
    assert_bits_equal(r.cpu().numpy(), ora.resample_distributions(x, t, np.random.binomial(1, 0.5, x.size)))


def test_resample_feeds_the_match_on_the_device():
    """blending/steps.py's pattern: the resampled distribution is the match's target, with no host copy"""
    x = rain((512, 512), 8)
    a, b = rain((512, 512), 9), rain((512, 512), 10, dry=0.3)
    np.random.seed(2)
    c = _pm().resample_distributions(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda(), 0.3)
    got = _pm().nonparam_match_empirical_cdf(torch.from_numpy(x).cuda(), c)
    np.random.seed(2)
    c_want = ora.resample_distributions(a, b, np.random.binomial(1, 0.3, a.size))
    assert_bits_equal(got.cpu().numpy(), ora.nonparam_match_empirical_cdf(x, c_want))


def test_steps_forecast_with_the_device_match():
    """pysteps.nowcasts.steps.forecast, seeded, once stock and once with its probability matching on
    the device (the module attribute patched inside this test only)"""
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    import contextlib
    import importlib
    import io
    import sys
    from unittest import mock
    from unittest.mock import MagicMock

    from pysteps_b200 import _synthetic as syn
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    steps = importlib.import_module("pysteps.nowcasts.steps")
    m, n = 64, 64
    fr = syn.rain_frames(m, n, 3, 4, dx=2, dy=-1)
    R = np.where(fr > 0.1, 10 * np.log10(np.maximum(fr, 0.1)), -15.0)
    V = 2.0 * syn.velocity_field(m, n, 4)
    kw = dict(timesteps=3, n_ens_members=3, n_cascade_levels=3, precip_thr=-10.0, kmperpixel=1.0, timestep=5.0,
              noise_method="nonparametric", seed=42, num_workers=1, probmatching_method="cdf")
    calls = []

    def device_match(initial, target, ignore_indices=None):
        calls.append(initial.shape)
        return _pm().nonparam_match_empirical_cdf(initial, target, ignore_indices)

    def run():
        with warnings.catch_warnings(), contextlib.redirect_stdout(io.StringIO()):
            warnings.simplefilter("ignore")
            return steps.forecast(R, V, **kw)

    want = run()
    with mock.patch.object(steps.probmatching, "nonparam_match_empirical_cdf", device_match):
        got = run()
    assert calls, "the forecast did not reach the probability matching"
    assert want.shape == got.shape == (3, 3, m, n)
    assert np.array_equal(got, want, equal_nan=True)
