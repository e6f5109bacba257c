"""TEST / BASELINE INFRASTRUCTURE (never imported by `lhotse_b200/`): makes the *reference* (lhotse) importable where
`soundfile`, `intervaltree` and `cytoolz` are absent (SURVEY.md §8c).  The reference is an unmodified lhotse source tree named
by LHOTSE_REFERENCE_ROOT, or else the archive `oracle/_ref/lhotse_ref.zip` that `oracle/make_ref.py` (run by `build()`) packs
from such a tree (git-ignored; imported through zipimport).  Where neither exists, `reference_available()` is False and the
tests that need lhotse itself skip.
Users: `tests/refshim.py` (the parity tests) and `bench.py`'s CPU reference legs (`cpu_baseline`, `--impl reference`)."""
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE_ZIP = os.path.join(_HERE, "_ref", "lhotse_ref.zip")


def _resolve_root() -> str:
    env = os.environ.get("LHOTSE_REFERENCE_ROOT")
    if env:
        return env
    return REFERENCE_ZIP


REFERENCE_ROOT = _resolve_root()


class _Stub(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (), {})


def reference_available() -> bool:
    if REFERENCE_ROOT.endswith(".zip"):
        return os.path.isfile(REFERENCE_ROOT)
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "lhotse"))


def reference_kind() -> str:
    """"tree" (build container), "zip" (GPU box) or "none"."""
    if not reference_available():
        return "none"
    return "zip" if REFERENCE_ROOT.endswith(".zip") else "tree"


def import_reference():
    """Returns the imported `lhotse` package from the reference tree / archive (or raises ImportError)."""
    if not reference_available():
        raise ImportError("reference tree not present")
    for m in ("soundfile", "intervaltree", "cytoolz"):
        if m not in sys.modules:
            try:
                __import__(m)
            except Exception:
                import importlib.machinery

                stub = _Stub(m)
                stub.__spec__ = importlib.machinery.ModuleSpec(m, None)  # keeps importlib.util.find_spec(m) working
                sys.modules[m] = stub
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    sys.dont_write_bytecode = True
    import lhotse  # noqa

    return lhotse
