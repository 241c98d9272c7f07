"""Drop-in test at the level the path is actually called from: the UNMODIFIED reference
``pysteps.nowcasts.utils.nowcast_main_loop`` (nowcasts/utils.py:265-533, the loop behind
nowcasts.steps / anvil / linda) run once with the reference's own extrapolator and BPS perturbator
and once with the B200 methods registered into the reference registries (lazy perturbation
handles, displacements resident on the device).  CPU only: the C ABI is emulated by the oracle
(tests/cpu_abi.py), so this checks the plumbing -- registries, kwargs, handle protocol, ensemble
and irregular time steps -- not the kernels.  Needs /root/reference."""
import sys
from unittest.mock import MagicMock

import numpy as np
import pytest

import cpu_abi
import registries
from pysteps_b200 import _synthetic as syn


@pytest.fixture(scope="module")
def ref():
    import _refimport
    if not _refimport.available():
        pytest.skip("/root/reference not present (GPU box)")
    import importlib
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    utils = importlib.import_module("pysteps.nowcasts.utils")
    noise = importlib.import_module("pysteps.noise.interface")
    import pysteps_b200
    with registries.restored():
        pysteps_b200.register()
        yield utils, noise


def _model(state, params):
    """a stand-in nowcast model in Lagrangian coordinates: members drift apart slowly"""
    fields = state["fields"] * params["decay"] + params["bias"][:, None, None]
    return fields, {"fields": fields}


@pytest.mark.parametrize("timesteps", [3, [0.5, 1.0, 2.25, 3.0]])
def test_ensemble_loop_with_b200_methods_equals_the_reference_loop(ref, timesteps):
    utils, noise = ref
    m, n, members = 48, 64, 3
    precip = syn.rain_field(m, n, 5)
    velocity = 2.0 * syn.velocity_field(m, n, 5)
    params = {"decay": 0.97, "bias": np.array([0.0, 0.1, -0.05])}
    state = {"fields": np.stack([precip * (1 + 0.05 * i) for i in range(members)])}
    timestep_min, kmperpixel = 5.0, 1.0

    def run(noise_name, extrap_name, extrap_kwargs):
        init, gen = noise.get_method(noise_name)
        perts = []
        for j in range(members):
            vp = init(velocity, 1.0 / kmperpixel, timestep_min, randstate=np.random.RandomState(100 + j))
            perts.append(lambda t, vp=vp: gen(vp, t * timestep_min))   # nowcasts/steps.py:927-929
        return utils.nowcast_main_loop(precip, velocity, {"fields": state["fields"].copy()}, timesteps, extrap_name,
                                       _model, extrap_kwargs=extrap_kwargs, velocity_pert_gen=perts, params=params,
                                       ensemble=True, num_ensemble_members=members)

    want = run("bps", "semilagrangian", {"allow_nonfinite_values": True})
    with cpu_abi.emulated():
        got = run("bps_b200", "semilagrangian_b200", {"allow_nonfinite_values": True, "b200_resident": True})
    assert len(got) == len(want) == members
    for g_member, w_member in zip(got, want):
        assert len(g_member) == len(w_member)
        for g, w in zip(g_member, w_member):
            assert isinstance(g, np.ndarray) and g.shape == w.shape and g.dtype == w.dtype
            assert np.array_equal(g, w, equal_nan=True)


def test_deterministic_loop(ref):
    utils, _ = ref
    m, n = 40, 56
    precip = syn.rain_field(m, n, 6)
    velocity = syn.velocity_field(m, n, 6, "rotation") * 3.0

    def model(state, params):
        return state["f"], state

    want = utils.nowcast_main_loop(precip, velocity, {"f": precip}, 4, "semilagrangian", model)
    with cpu_abi.emulated():
        got = utils.nowcast_main_loop(precip, velocity, {"f": precip}, 4, "semilagrangian_b200", model)
    assert np.array_equal(np.asarray(got), np.asarray(want), equal_nan=True)


def test_steps_forecast_end_to_end(ref):
    """pysteps.nowcasts.steps.forecast itself (cascade decomposition, AR model, noise, BPS velocity
    perturbations, AR pre-alignment through the extrapolator, the member loop): seeded, once with
    the stock methods and once with extrap_method / vel_pert_method pointing at the B200 ones."""
    import contextlib
    import importlib
    import io
    import warnings
    steps = importlib.import_module("pysteps.nowcasts.steps")
    m, n = 64, 64
    fr = syn.rain_frames(m, n, 3, 4, dx=2, dy=-1)
    R = np.where(fr > 0.1, 10 * np.log10(np.maximum(fr, 0.1)), -15.0)
    V = 2.0 * syn.velocity_field(m, n, 4)
    kw = dict(timesteps=3, n_ens_members=3, n_cascade_levels=3, precip_thr=-10.0, kmperpixel=1.0, timestep=5.0,
              noise_method="nonparametric", seed=42, num_workers=1)

    def run(**extra):
        with warnings.catch_warnings(), contextlib.redirect_stdout(io.StringIO()):
            warnings.simplefilter("ignore")
            return steps.forecast(R, V, **kw, **extra)

    want = run()
    with cpu_abi.emulated():
        got = run(extrap_method="semilagrangian_b200", vel_pert_method="bps_b200",
                  extrap_kwargs={"b200_resident": True})
    assert want.shape == got.shape == (3, 3, m, n)
    assert np.array_equal(want, got, equal_nan=True)
    assert np.isfinite(want).any()
