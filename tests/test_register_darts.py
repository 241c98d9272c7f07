"""CPU: the DARTS method in this package's registry and in the reference's (where it exists)."""
import importlib
import sys
from unittest.mock import MagicMock

import pytest


def test_get_method_names():
    from pysteps_b200.motion import get_method
    from pysteps_b200.motion.darts import DARTS
    assert get_method("darts") is DARTS
    assert get_method("DARTS_B200") is DARTS
    assert get_method("Darts") is DARTS


def test_register_override_swaps_the_stock_darts():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    mi = importlib.import_module("pysteps.motion.interface")
    import pysteps_b200
    from pysteps_b200.motion.darts import DARTS
    saved = dict(mi._methods)
    stock = mi.get_method("darts")
    try:
        assert "motion:darts_b200" in pysteps_b200.register()
        assert mi.get_method("darts_b200") is DARTS and mi.get_method("darts") is stock
        assert "motion:darts" in pysteps_b200.register(override=True)
        assert mi.get_method("darts") is DARTS
    finally:
        mi._methods.clear()
        mi._methods.update(saved)
    assert mi.get_method("darts") is stock
