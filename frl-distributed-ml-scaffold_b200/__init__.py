"""frl_b200 — H100-native data-parallel training step behind the FRL Distributed ML Scaffold
plugin API (``Problem`` / ``Task`` / criteria / ``Solver.solve``).

Import as ``frl_b200`` (see ``frl_b200.py`` at the repository root).  ``install_reference_alias``
additionally registers the package under the reference's import name ``frldistml.scaffold`` so
an existing ``Problem`` module runs unchanged.
"""
import sys as _sys
import types as _types

__version__ = "0.1.0"

_SUBMODULES = ("types", "criteria", "model", "lr_scheduler", "sampler", "transform", "task",
               "problem", "multitask_problem", "solver_worker", "solver", "local_solver",
               "storage_layers", "storage_layers.dataset", "indexed_dataset", "text_dataset")


def install_reference_alias(top: str = "frldistml", sub: str = "scaffold") -> None:
    """Make ``import frldistml.scaffold.<module>`` resolve to this package's modules."""
    import importlib
    if top not in _sys.modules:
        _sys.modules[top] = _types.ModuleType(top)
        _sys.modules[top].__path__ = []          # mark as package
    me = _sys.modules[__name__]
    _sys.modules[f"{top}.{sub}"] = me
    setattr(_sys.modules[top], sub, me)
    for name in _SUBMODULES:
        mod = importlib.import_module(f"{__name__}.{name}")
        _sys.modules[f"{top}.{sub}.{name}"] = mod
