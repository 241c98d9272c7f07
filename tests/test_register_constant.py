"""CPU: the constant method in this package's registry and in the reference's (where it exists)."""
import importlib
import sys
from unittest.mock import MagicMock

import pytest


def test_get_method_names():
    from pysteps_b200.motion import get_method
    from pysteps_b200.motion.constant import constant
    assert get_method("constant") is constant
    assert get_method("CONSTANT_B200") is constant
    assert get_method("Constant") is constant


def test_register_override_swaps_the_stock_constant():
    import _refimport
    if not _refimport.available():
        pytest.skip("the reference is not present")
    _refimport.import_reference()
    for ext in ("pysteps.motion._proesmans", "pysteps.motion._vet"):
        sys.modules.setdefault(ext, MagicMock())
    mi = importlib.import_module("pysteps.motion.interface")
    import pysteps_b200
    from pysteps_b200.motion.constant import constant
    saved = dict(mi._methods)
    stock = mi.get_method("constant")
    try:
        assert "motion:constant_b200" in pysteps_b200.register()
        assert mi.get_method("constant_b200") is constant and mi.get_method("constant") is stock
        assert "motion:constant" in pysteps_b200.register(override=True)
        assert mi.get_method("constant") is constant
    finally:
        mi._methods.clear()
        mi._methods.update(saved)
    assert mi.get_method("constant") is stock
