"""CPU: the registries of this package's subpackages, ``methods()``, and ``register()`` into the
reference's own registries (where the reference is present), with and without override.  Every test
that touches the reference's registries restores all six of them (registries.py)."""
import importlib
import sys
from unittest.mock import MagicMock

import numpy as np
import pytest

import pysteps_b200
import registries
from pysteps_b200.blending.linear_blending import forecast as blend
from pysteps_b200.extrapolation.interface import _do_nothing, eulerian_persistence
from pysteps_b200.extrapolation.semilagrangian import extrapolate
from pysteps_b200.motion.constant import constant
from pysteps_b200.motion.darts import DARTS
from pysteps_b200.motion.lucaskanade import dense_lucaskanade
from pysteps_b200.motion.proesmans import proesmans
from pysteps_b200.motion.vet import vet
from pysteps_b200.noise.motion import generate_bps, initialize_bps
from pysteps_b200.nowcasts.extrapolation import forecast as extrapolation_nowcast
from pysteps_b200.nowcasts.lagrangian_probability import forecast as probability
from pysteps_b200.postprocessing import ensemblestats as es

SALIENT = pysteps_b200.blending.get_method("salient_blending")

# category -> {pysteps' stock name: this package's callable}, for everything this package provides
PROVIDED = {
    "extrapolation": {"semilagrangian": extrapolate},
    "motion": {"lk": dense_lucaskanade, "lucaskanade": dense_lucaskanade, "vet": vet, "proesmans": proesmans,
               "constant": constant, "darts": DARTS},
    "noise": {"bps": (initialize_bps, generate_bps)},
    "nowcasts": {"lagrangian_probability": probability, "probability": probability,
                 "extrapolation": extrapolation_nowcast, "lagrangian": extrapolation_nowcast},
    "ensemblestats": {"mean": es.mean, "excprob": es.excprob, "banddepth": es.banddepth},
    "blending": {"linear_blending": blend, "salient_blending": SALIENT},
}

def _ours(category):
    if category == "ensemblestats":
        return lambda name, method_type="ensemblestats": pysteps_b200.postprocessing.get_method(name, method_type)
    return getattr(pysteps_b200, category).get_method


def _theirs(category):
    module = importlib.import_module(registries.REGISTRIES[category][0])
    if category == "ensemblestats":
        return lambda name: module.get_method(name, "ensemblestats")
    return module.get_method


def _same(got, want):
    """the same callable, or for a noise method the same (initialize, generate) pair"""
    if isinstance(want, tuple):
        return isinstance(got, tuple) and len(got) == len(want) and all(g is w for g, w in zip(got, want))
    return got is want


def _functions(fn):
    """the functions behind a registry entry: a (initialize, generate) pair, a partial, or a function"""
    return [getattr(f, "func", f) for f in (fn if isinstance(fn, tuple) else (fn,))]


def _from_pysteps_b200(fn):
    return any(f.__module__.startswith("pysteps_b200") for f in _functions(fn))


def _check_names(category, names):
    """``names`` (stock name -> callable) resolve in this package's registry under the stock name and the
    "_b200" name, in any case"""
    get = _ours(category)
    for name, fn in names.items():
        for key in (name, name.upper(), name.title(), name + "_b200", name.upper() + "_B200"):
            assert _same(get(key), fn), (category, key)


def test_advection_names():
    _check_names("extrapolation", {"semilagrangian": extrapolate})
    _check_names("motion", {"lk": dense_lucaskanade, "lucaskanade": dense_lucaskanade, "vet": vet,
                            "proesmans": proesmans})
    _check_names("noise", {"bps": (initialize_bps, generate_bps)})
    # the registries' own entries, which are not this package's to publish
    for name, fn in (("eulerian", eulerian_persistence), (None, _do_nothing), ("none", _do_nothing)):
        assert pysteps_b200.extrapolation.get_method(name) is fn, name
    field = pysteps_b200.motion.get_method(None)(np.ones((2, 5, 7)))
    assert field.shape == (2, 5, 7) and not field.any()
    with pytest.raises(ValueError, match="Unknown method farneback"):
        pysteps_b200.motion.get_method("farneback")
    with pytest.raises(NotImplementedError, match="Method brox not implemented"):
        pysteps_b200.motion.get_method("BROX")
    with pytest.raises(ValueError, match="Unknown method lagrangian"):
        pysteps_b200.extrapolation.get_method("lagrangian")
    with pytest.raises(ValueError, match="Unknown method nonparametric"):
        pysteps_b200.noise.get_method("nonparametric")
    with pytest.raises(TypeError, match="Only strings supported"):
        pysteps_b200.noise.get_method(None)


def test_constant_get_method_names():
    _check_names("motion", {"constant": constant})


def test_darts_get_method_names():
    _check_names("motion", {"darts": DARTS})


def test_probability_get_method_names():
    _check_names("nowcasts", {"probability": probability, "lagrangian_probability": probability})
    with pytest.raises(ValueError, match="Unknown nowcasting method steps"):
        pysteps_b200.nowcasts.get_method("steps")
    with pytest.raises(TypeError, match="Only strings supported"):
        pysteps_b200.nowcasts.get_method(None)


def test_nowcast_names():
    _check_names("nowcasts", {"extrapolation": extrapolation_nowcast, "lagrangian": extrapolation_nowcast})
    assert pysteps_b200.nowcasts.get_method("eulerian") is eulerian_persistence


def test_ensemblestats_get_method_names():
    _check_names("ensemblestats", {"mean": es.mean, "excprob": es.excprob, "banddepth": es.banddepth})
    get = pysteps_b200.postprocessing.get_method
    assert get("ExcProb", "EnsembleStats") is es.excprob
    with pytest.raises(ValueError, match="Unknown ensemblestats method rankhist"):
        get("rankhist", "ensemblestats")
    with pytest.raises(ValueError, match="Unknown diagnostics method mean"):
        get("mean", "diagnostics")
    with pytest.raises(ValueError, match="Unknown method type verification"):
        get("mean", "verification")
    with pytest.raises(TypeError, match="Only strings supported for for the method_type"):
        get("mean", None)
    with pytest.raises(TypeError, match="Only strings supported for the method's names"):
        get(1, "ensemblestats")


def test_blending_get_method_names():
    _check_names("blending", {"linear_blending": blend, "salient_blending": SALIENT})
    assert SALIENT.func is blend and SALIENT.keywords == {"saliency": True} and not SALIENT.args
    with pytest.raises(ValueError, match="Unknown blending method steps"):
        pysteps_b200.blending.get_method("steps")
    with pytest.raises(TypeError, match="Only strings supported"):
        pysteps_b200.blending.get_method(None)


def test_get_method_errors_match_the_reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    ref = _refimport.ref_module("pysteps.postprocessing.interface")
    for args in ((None, "ensemblestats"), ("mean", 3), ("x", "ensemblestats"), ("mean", "other"),
                 ("mean", "diagnostics")):
        with pytest.raises(Exception) as want:
            ref.get_method(*args)
        with pytest.raises(type(want.value)) as got:
            pysteps_b200.postprocessing.get_method(*args)
        # first line: the lists of available methods differ by this package's "_b200" names
        assert str(got.value).split("\n")[0] == str(want.value).split("\n")[0], args


def test_methods_lists_the_categories():
    got = pysteps_b200.interface.methods()
    assert list(got) == ["extrapolation", "motion", "noise", "nowcasts", "ensemblestats", "blending"]
    assert got["extrapolation"] == {"semilagrangian_b200": extrapolate}
    assert got["motion"] == {"lk_b200": dense_lucaskanade, "lucaskanade_b200": dense_lucaskanade, "vet_b200": vet,
                             "proesmans_b200": proesmans, "constant_b200": constant, "darts_b200": DARTS}
    assert got["noise"] == {"bps_b200": (initialize_bps, generate_bps)}
    assert got["blending"] == {"linear_blending_b200": blend, "salient_blending_b200": SALIENT}


def test_methods_lists_the_ensemblestats():
    assert pysteps_b200.interface.methods()["ensemblestats"] == {
        "mean_b200": es.mean, "excprob_b200": es.excprob, "banddepth_b200": es.banddepth}


def test_methods_lists_the_nowcasts():
    assert pysteps_b200.interface.methods()["nowcasts"] == {
        "lagrangian_probability_b200": probability, "probability_b200": probability,
        "extrapolation_b200": extrapolation_nowcast, "lagrangian_b200": extrapolation_nowcast}


@pytest.fixture
def stock():
    """the reference's six registries, as whatever ran earlier left them; restored afterwards"""
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    # the reference's Cython extensions are not built here; only the registries are needed
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    with registries.restored() as regs:
        yield regs


def _assert_stock_names_are_pysteps_own(stock):
    """Every stock name this package provides resolves to pysteps' own callable, whatever ran earlier in
    this process, so that the checks of what register() leaves alone mean something."""
    for category, provided in PROVIDED.items():
        for name in provided:
            assert all(callable(f) for f in _functions(stock[category][name])), (category, name)
            assert not _from_pysteps_b200(stock[category][name]), (category, name)


def test_register_into_reference_registries(stock):
    _assert_stock_names_are_pysteps_own(stock)
    before = {category: dict(registry) for category, registry in stock.items()}
    done = pysteps_b200.register()
    assert done == [category + ":" + name + "_b200" for category, provided in PROVIDED.items() for name in provided]
    for category, provided in PROVIDED.items():
        get = _theirs(category)
        for name, fn in provided.items():
            assert _same(get(name + "_b200"), fn) and _same(get(name.upper() + "_B200"), fn), (category, name)
        # nothing but the "_b200" names was added, and every stock entry is the same object
        assert set(stock[category]) == set(before[category]) | {name + "_b200" for name in provided}, category
        assert all(stock[category][k] is v for k, v in before[category].items()), category
    done = pysteps_b200.register(override=True)
    assert done == [category + ":" + name + suffix for category, provided in PROVIDED.items()
                    for name in provided for suffix in ("_b200", "")]


# stock entries of each pysteps registry that this package does not provide
NOT_PROVIDED = {"extrapolation": ("eulerian", None, "none"), "motion": ("farneback", None),
                "noise": ("parametric", "nonparametric", "ssft", "nested"),
                "nowcasts": ("anvil", "eulerian", "linda", "sprog", "sseps", "steps"),
                "ensemblestats": (), "blending": ("steps", "pca_enkf")}


def _check_override(stock, swapped):
    """register(override=True) binds each stock name of ``swapped`` (category -> {stock name: callable}) to
    this package's callable, and leaves alone what this package does not provide."""
    _assert_stock_names_are_pysteps_own(stock)
    before = {category: dict(stock[category]) for category in swapped}
    done = pysteps_b200.register(override=True)
    for category, names in swapped.items():
        get = _theirs(category)
        for name, fn in names.items():
            assert category + ":" + name in done and category + ":" + name + "_b200" in done, (category, name)
            for key in (name, name.upper(), name + "_b200"):
                assert _same(get(key), fn), (category, key)
        assert set(stock[category]) == set(before[category]) | {name + "_b200" for name in PROVIDED[category]}
        assert set(before[category]) == set(PROVIDED[category]) | set(NOT_PROVIDED[category]), category
        for name in NOT_PROVIDED[category]:
            old = before[category][name]
            assert stock[category][name] is old and not _from_pysteps_b200(old), (category, name)
        # only the registry changes: importing the stock function directly still gives pysteps' own
        for name in names:
            for f in _functions(before[category][name]):
                assert getattr(importlib.import_module(f.__module__), f.__name__) is f, (category, name)


def test_register_override_swaps_the_advection_methods(stock):
    _check_override(stock, {"extrapolation": {"semilagrangian": extrapolate},
                            "motion": {"lk": dense_lucaskanade, "lucaskanade": dense_lucaskanade, "vet": vet,
                                       "proesmans": proesmans},
                            "noise": {"bps": (initialize_bps, generate_bps)}})


def test_register_override_swaps_the_stock_constant(stock):
    _check_override(stock, {"motion": {"constant": constant}})


def test_register_override_swaps_the_stock_darts(stock):
    _check_override(stock, {"motion": {"darts": DARTS}})


def test_register_override_swaps_the_stock_probability(stock):
    _check_override(stock, {"nowcasts": {"probability": probability, "lagrangian_probability": probability}})


def test_register_override_swaps_the_stock_ensemblestats(stock):
    _check_override(stock, {"ensemblestats": {"mean": es.mean, "excprob": es.excprob, "banddepth": es.banddepth}})


def test_register_override_swaps_the_stock_names(stock):
    _check_override(stock, {"blending": {"linear_blending": blend, "salient_blending": SALIENT},
                            "nowcasts": {"extrapolation": extrapolation_nowcast,
                                         "lagrangian": extrapolation_nowcast}})
