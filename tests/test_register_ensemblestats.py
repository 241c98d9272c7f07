"""CPU: the ensemble statistics in this package's postprocessing registry and in the reference's (where it
exists).  The stock functions come from pysteps.postprocessing.ensemblestats, not from the registry,
which an earlier register(override=True) in this process may have changed."""
import importlib
import sys
from unittest.mock import MagicMock

import pytest


def test_get_method_names():
    from pysteps_b200.postprocessing import ensemblestats as es
    from pysteps_b200.postprocessing import get_method
    for name, fn in (("mean", es.mean), ("ExcProb", es.excprob), ("BANDDEPTH_B200", es.banddepth),
                     ("excprob_b200", es.excprob)):
        assert get_method(name, "ensemblestats") is fn
        assert get_method(name, "EnsembleStats") is fn
    with pytest.raises(ValueError, match="Unknown ensemblestats method rankhist"):
        get_method("rankhist", "ensemblestats")
    with pytest.raises(ValueError, match="Unknown diagnostics method mean"):
        get_method("mean", "diagnostics")
    with pytest.raises(ValueError, match="Unknown method type verification"):
        get_method("mean", "verification")
    with pytest.raises(TypeError, match="Only strings supported for for the method_type"):
        get_method("mean", None)
    with pytest.raises(TypeError, match="Only strings supported for the method's names"):
        get_method(1, "ensemblestats")


def test_get_method_errors_match_the_reference():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    ref = _refimport.ref_module("pysteps.postprocessing.interface")
    from pysteps_b200.postprocessing import get_method
    for args in ((None, "ensemblestats"), ("mean", 3), ("x", "ensemblestats"), ("mean", "other"),
                 ("mean", "diagnostics")):
        with pytest.raises(Exception) as want:
            ref.get_method(*args)
        with pytest.raises(type(want.value)) as got:
            get_method(*args)
        # first line: the lists of available methods differ by this package's "_b200" names
        assert str(got.value).split("\n")[0] == str(want.value).split("\n")[0], args


def test_methods_lists_the_ensemblestats():
    import pysteps_b200
    from pysteps_b200.postprocessing import ensemblestats as es
    assert pysteps_b200.interface.methods()["ensemblestats"] == {
        "mean_b200": es.mean, "excprob_b200": es.excprob, "banddepth_b200": es.banddepth}


def test_register_and_override():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    ppi = importlib.import_module("pysteps.postprocessing.interface")
    stock = importlib.import_module("pysteps.postprocessing.ensemblestats")
    import pysteps_b200
    from pysteps_b200.postprocessing import ensemblestats as es
    saved = dict(ppi._ensemblestats_methods)
    try:
        for name in ("mean", "excprob", "banddepth"):
            ppi._ensemblestats_methods[name] = getattr(stock, name)
        done = pysteps_b200.register()
        for name in ("mean", "excprob", "banddepth"):
            assert "ensemblestats:%s_b200" % name in done
            assert ppi.get_method(name + "_b200", "ensemblestats") is getattr(es, name)
            assert ppi.get_method(name, "ensemblestats") is getattr(stock, name)
        done = pysteps_b200.register(override=True)
        for name in ("mean", "excprob", "banddepth"):
            assert "ensemblestats:" + name in done
            assert ppi.get_method(name.upper(), "ensemblestats") is getattr(es, name)
            # direct imports are not patched
            assert getattr(stock, name) is not getattr(es, name)
    finally:
        ppi._ensemblestats_methods.clear()
        ppi._ensemblestats_methods.update(saved)
