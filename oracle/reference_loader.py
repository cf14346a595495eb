"""Imports the UNMODIFIED reference (frgfm/Holocron) as ``holocron.*`` modules from the checkout named by the
``HOLOCRON_REFERENCE`` environment variable.

Used by ``tests/golden/make_golden.py`` to generate the committed golden fixtures (the tests themselves only read those
fixtures and never need the reference).

``import holocron`` itself fails in this image (its __init__ pulls matplotlib/fastprogress and a generated
version.py), so a stub parent package whose __path__ points at the reference is pre-seeded and the needed
sub-packages are imported directly.
"""
import importlib
import os
import sys
import types
from pathlib import Path

REFERENCE_ROOT = Path(os.environ.get("HOLOCRON_REFERENCE", "holocron-reference"))


def available() -> bool:
    return (REFERENCE_ROOT / "holocron" / "nn" / "functional.py").exists()


def load():
    """Returns the stub ``holocron`` package with nn, ops, optim and models imported from the reference."""
    if not available():
        raise RuntimeError(f"reference tree not available at {REFERENCE_ROOT} (set HOLOCRON_REFERENCE)")
    existing = sys.modules.get("holocron")
    if existing is not None and getattr(existing, "__holocron_reference__", False):
        return existing
    pkg = types.ModuleType("holocron")
    pkg.__path__ = [str(REFERENCE_ROOT / "holocron")]
    pkg.__holocron_reference__ = True
    sys.modules["holocron"] = pkg
    for sub in ("nn", "ops", "optim", "models"):
        setattr(pkg, sub, importlib.import_module(f"holocron.{sub}"))
    return pkg
