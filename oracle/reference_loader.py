"""Import the reference package -- TEST / BENCHMARK INFRASTRUCTURE ONLY.

A checkout of the reference is looked for at ``$TORCHCDE_REFERENCE_ROOT`` (default ``/root/reference``);
``oracle/_ref`` is an unmodified ``pip install --target`` of it (recipe in ``oracle/Makefile``, git-ignored).
This module is used by ``oracle/make_golden.py`` and ``oracle/make_reference_golden.py`` (to generate the
committed fixtures) and by ``bench.py``'s CPU arm (the reference's own ``cdeint`` timed on the host cores).

The reference's ``torchcde/__init__.py:7`` imports ``solver.py``, whose first lines import
``torchdiffeq`` and ``torchsde`` (solver.py:2-3).  Neither is installed.  We therefore put
two stand-in modules in ``sys.modules`` before importing:
  * ``torchdiffeq`` -> ``oracle.odeint_port`` (the restated fixed-grid solver), so that the
    reference's own ``cdeint`` / ``_check_compatability`` / ``_VectorField`` / output permute
    run unmodified around it;
  * ``torchsde``    -> an empty module (that backend is out of scope).
Nothing is copied from the reference tree; it is imported where it lies.
"""
import importlib
import os
import sys
import types

_HERE = os.path.dirname(os.path.abspath(__file__))
# the reference checkout, or the unmodified install of it under oracle/_ref (oracle/Makefile)
_CANDIDATES = [os.environ.get("TORCHCDE_REFERENCE_ROOT", "/root/reference"), os.path.join(_HERE, "_ref")]


def _root():
    for cand in _CANDIDATES:
        if os.path.isfile(os.path.join(cand, "torchcde", "__init__.py")):
            return cand
    return None


REFERENCE_ROOT = _root() or _CANDIDATES[0]


def reference_source():
    """The reference checkout (with its setup.py) that oracle/Makefile can install into oracle/_ref, or None."""
    src = _CANDIDATES[0]
    return src if os.path.isfile(os.path.join(src, "setup.py")) else None


def reference_available():
    return _root() is not None


def reference_kind():
    """'live' = the reference checkout itself, '_ref' = the pip-installed copy under oracle/_ref, None = neither."""
    root = _root()
    if root is None:
        return None
    return "_ref" if os.path.abspath(root) == os.path.join(_HERE, "_ref") else "live"


def load_reference():
    """Return the reference ``torchcde`` module, or raise ``ImportError`` if the tree is absent."""
    if not reference_available():
        raise ImportError("reference tree not present at any of {}".format(_CANDIDATES))
    if "torchcde" in sys.modules and getattr(sys.modules["torchcde"], "_b200_oracle_loaded", False):
        return sys.modules["torchcde"]
    from . import odeint_port

    diffeq = types.ModuleType("torchdiffeq")
    diffeq.odeint = odeint_port.odeint
    diffeq.odeint_adjoint = odeint_port.odeint_adjoint
    diffeq.__version__ = "port-of-0.2.x"
    sys.modules["torchdiffeq"] = diffeq
    sys.modules.setdefault("torchsde", types.ModuleType("torchsde"))
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    module = importlib.import_module("torchcde")
    module._b200_oracle_loaded = True
    return module
