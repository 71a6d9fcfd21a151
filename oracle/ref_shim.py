"""TEST INFRASTRUCTURE ONLY — import shim for the *unmodified* reference modules under /root/reference.

Only used where the reference tree exists, to generate the committed golden fixtures in `tests/golden/` that pin the CPU
oracle in `oracle/*.py` against the reference's own code (generator: tests/golden/make_golden.py).  Nothing in the
product or the test suite imports this.

The reference package cannot be imported normally (SURVEY.md §8c): `cambrian/__init__.py` eagerly imports
every encoder, which needs timm / open_clip / diffusers / ezcolorlog / torch_xla.  Recipe: stub those
third-party modules with MagicMock, pre-seed namespace packages whose __path__ points into the reference
tree (skipping the eager __init__s), then import the hot-path modules file by file.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.machinery
import sys
import types
from pathlib import Path
from unittest.mock import MagicMock

REF_ROOT = Path("/root/reference")
_STUBS = ("ezcolorlog", "open_clip", "timm", "diffusers", "shortuuid", "torch_xla", "gcsfs", "google")


def available() -> bool:
    return (REF_ROOT / "cambrian" / "model" / "vision_sampler.py").exists()


class _StubFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, name, path=None, target=None):
        if name.split(".")[0] in _STUBS:
            return importlib.machinery.ModuleSpec(name, self, is_package=True)
        return None

    def create_module(self, spec):
        m = MagicMock(name=spec.name)
        m.__path__ = []
        m.__spec__ = spec
        return m

    def exec_module(self, module):
        pass


_installed = False


def install() -> None:
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError("/root/reference is not present — the shim needs the reference tree")
    import transformers  # noqa: F401  (must be imported before the stubs shadow anything it probes)
    sys.meta_path.insert(0, _StubFinder())
    for pkg in ("cambrian", "cambrian.model", "cambrian.model.multimodal_encoder",
                "cambrian.model.multimodal_projector", "cambrian.model.language_model"):
        m = types.ModuleType(pkg)
        m.__path__ = [str(REF_ROOT / pkg.replace(".", "/"))]
        sys.modules[pkg] = m
    _installed = True


def ref_module(name: str):
    """e.g. ref_module('cambrian.model.vision_sampler')"""
    install()
    return importlib.import_module(name)
