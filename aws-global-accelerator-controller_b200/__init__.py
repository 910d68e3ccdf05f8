"""garecon — H100-native batch reconcile-diff engine for the aws-global-accelerator-controller hot path.

The directory name carries the upstream project's hyphens, so import it with
`importlib.import_module("aws-global-accelerator-controller_b200")` (tests/conftest.py does this and
exposes it as `garecon`).
"""
from . import abi, tables  # noqa: F401
from .abi import Engine, GarError, ChangeSet  # noqa: F401
from .tables import pack, pack_bindings, Snapshot  # noqa: F401

__version__ = "0.1.0"
