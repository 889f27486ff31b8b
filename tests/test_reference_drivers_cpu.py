"""The import switch of INTEGRATION.md section A (``SIAMMOT_ENGINE=b200`` + ``import siammot_b200.dropin``): without the
environment variable it must leave the reference's own ``siammot.modelling.rcnn`` alone."""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


def test_dropin_switch_is_inert_without_the_environment_variable(monkeypatch):
    from siammot_b200 import dropin
    monkeypatch.delenv("SIAMMOT_ENGINE", raising=False)
    dropin.uninstall()
    assert dropin.install() is False and not getattr(sys.modules.get("siammot.modelling.rcnn"), "__siammot_b200__", False)
