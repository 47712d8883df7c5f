"""Resolution of clean-pvnet's package tree for the opt-in drop-ins (install_as_reference_module,
install_nn_as_reference_module): only leaf modules are ever replaced."""
import importlib
import importlib.util
import sys
import types


def reference_package(name):
    """Returns the package `name` (e.g. "lib.csrc.nn"), resolving it and each of its parents in turn: the REAL package
    whenever it can be imported (the normal case: the clean-pvnet checkout is on sys.path, so `lib.config`,
    `lib.networks`, ... keep importing), a namespace stand-in only for a parent that does not exist anywhere on sys.path
    (using the drop-ins outside a clean-pvnet checkout).  Every package is bound as an attribute of its parent."""
    parts = name.split(".")
    parent = None
    for i in range(1, len(parts) + 1):
        full = ".".join(parts[:i])
        mod = sys.modules.get(full)
        if mod is None:
            try:
                found = importlib.util.find_spec(full) is not None
            except (ImportError, ValueError, AttributeError):
                found = False
            if found:
                mod = importlib.import_module(full)        # the real package; errors inside it propagate
            else:
                mod = types.ModuleType(full)
                mod.__path__ = []                            # genuinely absent: namespace stand-in
                mod.__pvb_stand_in__ = True
                sys.modules[full] = mod
        if parent is not None and not hasattr(parent, parts[i - 1]):
            setattr(parent, parts[i - 1], mod)
        parent = mod
    return parent
