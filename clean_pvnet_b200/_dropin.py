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


def chain_wrapper_factory(task, wrapper, marker):
    """Patches lib.train.trainers.make_trainer._wrapper_factory to return wrapper(network) for cfg.task == task and to
    call the factory it replaces for every other task.  make_trainer loads the trainer file by path (make_trainer.py:6-10),
    so replacing a sys.modules entry would not reach it.  Each drop-in's factory carries its `marker` attribute and the
    markers of the factories it chains to, so installing a drop-in again is a no-op whatever was installed in between."""
    trainer = reference_package("lib.train.trainers.make_trainer")
    original = getattr(trainer, "_wrapper_factory", None)
    if getattr(original, marker, False):
        return
    if original is None:
        def original(cfg, network):
            raise RuntimeError(f"no trainer for task {cfg.task!r}: lib.train.trainers.make_trainer is not importable")

    def _wrapper_factory(cfg, network):
        if cfg.task == task:
            return wrapper(network)
        return original(cfg, network)

    for name, value in vars(original).items():
        if name.startswith("__pvb_"):
            setattr(_wrapper_factory, name, value)
    setattr(_wrapper_factory, marker, True)
    trainer._wrapper_factory = _wrapper_factory
