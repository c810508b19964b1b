"""Stages the reference project for ``bench.py --impl reference``.

The reference (ronghanghu/vit_10b_fsdp_example: ``run_vit_training.py`` and ``utils.py``) is not part of this
repository.  ``stage()`` byte-compiles those two modules into ``oracle/_ref/`` (ignored by git), from where
``baseline/reference_arm.py`` imports them; nothing is read from outside the repository at benchmark time.  The
reference is looked for in ``$VIT_REFERENCE_DIR`` or in a ``reference`` directory next to the repository.

    python oracle/stage_reference.py [REFERENCE_DIR]
"""
import os
import py_compile
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
MODULES = ("run_vit_training", "utils")


def staged() -> bool:
    return all(os.path.exists(os.path.join(REF_DIR, m + ".pyc")) for m in MODULES)


def stage(src: str = "") -> bool:
    """Returns True when oracle/_ref holds both modules afterwards."""
    src = src or os.environ.get("VIT_REFERENCE_DIR", os.path.join(os.path.dirname(ROOT), "reference"))
    if not all(os.path.exists(os.path.join(src, m + ".py")) for m in MODULES):
        return staged()
    os.makedirs(REF_DIR, exist_ok=True)
    for m in MODULES:
        py_compile.compile(os.path.join(src, m + ".py"), cfile=os.path.join(REF_DIR, m + ".pyc"), dfile=m + ".py",
                           doraise=True)
    return True


if __name__ == "__main__":
    print("staged" if stage(sys.argv[1] if len(sys.argv) > 1 else "") else "reference not found")
