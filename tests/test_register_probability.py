"""CPU: the probability nowcast in this package's registry and in the reference's (where it exists)."""
import importlib
import sys
from unittest.mock import MagicMock

import pytest


def test_get_method_names():
    from pysteps_b200.nowcasts import get_method
    from pysteps_b200.nowcasts.lagrangian_probability import forecast
    for name in ("probability", "Lagrangian_Probability", "PROBABILITY_B200", "lagrangian_probability_b200"):
        assert get_method(name) is forecast
    with pytest.raises(ValueError, match="Unknown nowcasting method steps"):
        get_method("steps")
    with pytest.raises(TypeError, match="Only strings supported"):
        get_method(None)


def test_methods_lists_the_nowcasts():
    import pysteps_b200
    from pysteps_b200.nowcasts.lagrangian_probability import forecast
    assert pysteps_b200.interface.methods()["nowcasts"] == {"lagrangian_probability_b200": forecast,
                                                            "probability_b200": forecast}


def test_register_override_swaps_the_stock_probability():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    ni = importlib.import_module("pysteps.nowcasts.interface")
    import pysteps_b200
    from pysteps_b200.nowcasts.lagrangian_probability import forecast
    saved = dict(ni._nowcast_methods)
    stock = importlib.import_module("pysteps.nowcasts.lagrangian_probability").forecast
    try:
        # start from the stock entries (an earlier register(override=True) in this process may have replaced them)
        ni._nowcast_methods["probability"] = ni._nowcast_methods["lagrangian_probability"] = stock
        done = pysteps_b200.register()
        assert "nowcasts:probability_b200" in done and "nowcasts:lagrangian_probability_b200" in done
        assert ni.get_method("probability_b200") is forecast and ni.get_method("lagrangian_probability_b200") is forecast
        assert ni.get_method("probability") is stock and ni.get_method("lagrangian_probability") is stock
        done = pysteps_b200.register(override=True)
        assert "nowcasts:probability" in done and "nowcasts:lagrangian_probability" in done
        assert ni.get_method("probability") is forecast and ni.get_method("Lagrangian_Probability") is forecast
        assert ni.get_method("steps") is saved["steps"]
    finally:
        ni._nowcast_methods.clear()
        ni._nowcast_methods.update(saved)
