"""CPU: the blending methods and the extrapolation nowcast in this package's registries and in the
reference's (where it exists), with and without override."""
import importlib
import sys
from unittest.mock import MagicMock

import pytest


def test_blending_get_method_names():
    from pysteps_b200.blending import get_method
    from pysteps_b200.blending.linear_blending import forecast
    assert get_method("linear_blending") is forecast and get_method("LINEAR_BLENDING_B200") is forecast
    sal = get_method("Salient_Blending")
    assert sal.func is forecast and sal.keywords == {"saliency": True}
    assert get_method("salient_blending_b200") is sal
    with pytest.raises(ValueError, match="Unknown blending method steps"):
        get_method("steps")
    with pytest.raises(TypeError, match="Only strings supported"):
        get_method(None)


def test_nowcast_names():
    from pysteps_b200.extrapolation.interface import eulerian_persistence
    from pysteps_b200.nowcasts import get_method
    from pysteps_b200.nowcasts.extrapolation import forecast
    for name in ("extrapolation", "Lagrangian", "extrapolation_b200", "lagrangian_b200"):
        assert get_method(name) is forecast
    assert get_method("eulerian") is eulerian_persistence


def test_register_override_swaps_the_stock_names():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    bi = importlib.import_module("pysteps.blending.interface")
    ni = importlib.import_module("pysteps.nowcasts.interface")
    import pysteps_b200
    from pysteps_b200.blending.linear_blending import forecast
    from pysteps_b200.nowcasts.extrapolation import forecast as extrapolation
    saved_b, saved_n = dict(bi._blending_methods), dict(ni._nowcast_methods)
    stock_lin = importlib.import_module("pysteps.blending.linear_blending").forecast
    stock_ext = importlib.import_module("pysteps.nowcasts.extrapolation").forecast
    try:
        bi._blending_methods["linear_blending"] = stock_lin
        ni._nowcast_methods["extrapolation"] = ni._nowcast_methods["lagrangian"] = stock_ext
        done = pysteps_b200.register()
        assert "blending:linear_blending_b200" in done and "nowcasts:extrapolation_b200" in done
        assert bi.get_method("linear_blending_b200") is forecast and bi.get_method("linear_blending") is stock_lin
        assert ni.get_method("lagrangian_b200") is extrapolation and ni.get_method("extrapolation") is stock_ext
        done = pysteps_b200.register(override=True)
        assert "blending:salient_blending" in done and "nowcasts:lagrangian" in done
        assert bi.get_method("linear_blending") is forecast
        assert bi.get_method("salient_blending").keywords == {"saliency": True}
        assert ni.get_method("extrapolation") is extrapolation and ni.get_method("lagrangian") is extrapolation
        assert bi.get_method("steps") is saved_b["steps"]
    finally:
        bi._blending_methods.clear()
        bi._blending_methods.update(saved_b)
        ni._nowcast_methods.clear()
        ni._nowcast_methods.update(saved_n)
