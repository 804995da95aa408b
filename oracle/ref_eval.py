"""The reference's second program, ``eval.py``, staged UNMODIFIED next to its ``train.py`` under ``oracle/_ref/`` and
imported for the host tests of the linear evaluation -- TEST INFRASTRUCTURE ONLY.

``stage()`` copies ``/root/reference/eval.py`` byte for byte to ``oracle/_ref/eval.py`` (git-ignored, like the rest
of ``oracle/_ref``) whenever the reference checkout is present.  ``__graft_entry__.build()`` calls it before
``oracle/stage_ref.stage()``, so the sha256 of ``eval.py`` lands in the same ``MANIFEST.json``; a copy staged before
this file existed gains ``eval.py`` on the next build.

``load()`` imports the staged file under the module name ``ref_eval`` (``eval`` is a builtin's name), after
``oracle/ref_runner._load_reference`` has applied its shims (identity ``.cuda()``, a ``termcolor`` stub, a one-rank
gloo process group).  ``eval.py``'s module-level ``logger`` exists only under ``__main__`` (eval.py:372), and
``load_checkpoint`` / ``save_checkpoint`` / ``load_pretrained`` log through it, so ``load()`` sets it.
"""
from __future__ import annotations

import importlib.util
import logging
import os
import shutil

from . import ref_runner, stage_ref

PATH = os.path.join(stage_ref.REF_DST, "eval.py")


def staged() -> bool:
    return os.path.isfile(PATH)


def stage() -> bool:
    """Copy the reference's eval.py to oracle/_ref/.  Returns True when a staged copy exists afterwards."""
    src = os.path.join(stage_ref.REF_SRC, "eval.py")
    if os.path.isfile(src):
        os.makedirs(stage_ref.REF_DST, exist_ok=True)
        shutil.copyfile(src, PATH)
    return staged()


_eval = None


def load():
    """The staged eval.py as module ``ref_eval``, with ref_runner's shims and its ``logger`` set (idempotent)."""
    global _eval
    if _eval is not None:
        return _eval
    if not staged():
        raise RuntimeError("oracle/_ref/eval.py is not staged: run __graft_entry__.build() where the reference "
                           "checkout exists")
    ref_runner._load_reference()
    spec = importlib.util.spec_from_file_location("ref_eval", PATH)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.logger = logging.getLogger("moco_ref_eval")
    mod.logger.setLevel(logging.WARNING)
    _eval = mod
    return mod
