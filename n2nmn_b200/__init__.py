"""n2nmn_b200 — H100-native (sm_90a) implementation of the N2NMN module-network hot path.

Public surface mirrors the reference: ``Assembler`` (models_*/nmn3_assembler.py), ``Modules``
(models_*/nmn3_modules.py) and the layout executor of ``NMN3Model`` (models_*/nmn3_model.py).
Importing the package does not need a GPU; constructing ``Modules`` / ``LayoutExecutor`` does, and
fails loudly if ``lib/libn2nmn_b200.so`` has not been built.
"""
from .assembler import Assembler, INVALID_EXPR  # noqa: F401

__all__ = ['Assembler', 'INVALID_EXPR', 'LayoutExecutor', 'ModulesCLEVR', 'ModulesSHAPES',
           'ModulesVQA']


def __getattr__(name):   # torch-dependent parts load lazily
    if name == 'LayoutExecutor':
        from .executor import LayoutExecutor
        return LayoutExecutor
    if name in ('ModulesCLEVR', 'ModulesSHAPES', 'ModulesVQA'):
        from . import modules
        return getattr(modules, name)
    raise AttributeError(name)
