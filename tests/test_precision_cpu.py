"""SSP_PRECISION, read once by the engine's constructor: unset or "exact" selects the split-fp16 forward, "fast" the single-term
one, in any case; any other value is refused instead of silently selecting the default.  Darknet(cfg) builds its engine
without a device."""
import pytest

from singleshotpose_b200 import Darknet, _lib


@pytest.mark.parametrize("value, fast", [(None, False), ("exact", False), ("EXACT", False), ("fast", True), ("Fast", True)])
def test_accepted_values(cfg_path, monkeypatch, value, fast):
    if value is None:
        monkeypatch.delenv("SSP_PRECISION", raising=False)
    else:
        monkeypatch.setenv("SSP_PRECISION", value)
    assert Darknet(cfg_path)._engine.fast is fast


@pytest.mark.parametrize("value", ["fats", "parity", "", "fast "])
def test_other_values_raise_naming_the_accepted_ones(cfg_path, monkeypatch, value):
    monkeypatch.setenv("SSP_PRECISION", value)
    with pytest.raises(_lib.SspError) as e:
        Darknet(cfg_path)
    msg = str(e.value)
    assert "SSP_PRECISION" in msg and "'exact'" in msg and "'fast'" in msg and repr(value) in msg
