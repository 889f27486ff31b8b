"""The import switch of INTEGRATION.md section A, as code.

The reference's drivers obtain the model through one name -- ``from siammot.modelling.rcnn import build_siammot``
(demos/demo_inference.py:13, tools/test_net.py:13, used at demo_inference.py:85 / test_net.py:39).  ``install()`` registers a
module under that name whose ``build_siammot`` is the engine's, BEFORE the reference's own module is imported, so the
reference's ``DemoInference`` / ``DatasetInference`` / ``do_inference`` run on the engine without a single edited line:

    SIAMMOT_ENGINE=b200 python -c "import siammot_b200.dropin" demos/demo.py ...        # or: import siammot_b200.dropin at start-up

``install()`` does nothing unless ``SIAMMOT_ENGINE=b200`` (or ``force=True``), and refuses to run after the reference's
module has already been imported (the caller would then hold the reference's builder)."""
import os
import sys
import types


def install(force=False):
    if not (force or os.environ.get("SIAMMOT_ENGINE", "") == "b200"):
        return False
    name = "siammot.modelling.rcnn"
    have = sys.modules.get(name)
    if have is not None and not getattr(have, "__siammot_b200__", False):
        raise RuntimeError("%s was imported before siammot_b200.dropin.install(): import the drop-in first" % name)
    from .modelling import rcnn as ours
    mod = types.ModuleType(name)
    mod.__siammot_b200__ = True
    mod.__doc__ = "siammot_b200 engine behind the reference's builder name (siammot_b200/dropin.py)"
    mod.build_siammot = ours.build_siammot
    mod.SiamMOT = ours.SiamMOT
    sys.modules[name] = mod
    return True


def uninstall():
    mod = sys.modules.get("siammot.modelling.rcnn")
    if mod is not None and getattr(mod, "__siammot_b200__", False):
        del sys.modules["siammot.modelling.rcnn"]


install()
