"""The unmodified reference's Gated PixelCNN for tools/bench_prior.py -- TEST INFRASTRUCTURE ONLY.

Same recipe as ``oracle.build_ref`` for the VQ-VAE, kept in a file tuple of its own so ``ref_path()`` (and with it
bench.py) does not change: ``build_prior_ref()`` copies the reference's ``pixelcnn/__init__.py`` and
``pixelcnn/models.py`` verbatim into the git-ignored ``oracle/_ref/`` where a checkout of the reference exists (a
no-op elsewhere), and ``load_reference_prior()`` imports that copy under its own name without disturbing the
product's ``pixelcnn`` package.
"""
import os
import shutil
import sys

from .build import REF_SRC, _REF_OUT

_PRIOR_REF_FILES = ("pixelcnn/__init__.py", "pixelcnn/models.py")


def ref_prior_path() -> str:
    """oracle/_ref when the verbatim copy of the reference's pixelcnn package is present, else ''."""
    return _REF_OUT if all(os.path.exists(os.path.join(_REF_OUT, f)) for f in _PRIOR_REF_FILES) else ""


def build_prior_ref() -> str:
    """Copy the reference's pixelcnn package into oracle/_ref/ (where the reference checkout exists)."""
    if not os.path.isdir(REF_SRC):
        return ref_prior_path()
    for f in _PRIOR_REF_FILES:
        dst = os.path.join(_REF_OUT, f)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        shutil.copyfile(os.path.join(REF_SRC, f), dst)
    return _REF_OUT


def _drop(name):
    for k in [k for k in sys.modules if k == name or k.startswith(name + ".")]:
        del sys.modules[k]


def load_reference_prior():
    """The reference's GatedPixelCNN class from oracle/_ref, or None when the copy is absent.  The product's
    ``pixelcnn`` modules are set aside during the import and restored afterwards."""
    ref_dir = ref_prior_path()
    if not ref_dir:
        return None
    saved = {k: v for k, v in sys.modules.items() if k == "pixelcnn" or k.startswith("pixelcnn.")}
    _drop("pixelcnn")
    sys.path.insert(0, ref_dir)
    try:
        from pixelcnn.models import GatedPixelCNN
    finally:
        sys.path.remove(ref_dir)
        _drop("pixelcnn")
        sys.modules.update(saved)
    return GatedPixelCNN
