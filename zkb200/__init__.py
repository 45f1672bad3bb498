"""zkb200 -- importable name of the `zkevm-circuits_b200/` package (a hyphen cannot appear in a Python module name).

The package body lives in `zkevm-circuits_b200/`; this shim only extends the module search path to it.
"""
import os as _os

__path__.append(_os.path.join(_os.path.dirname(_os.path.dirname(_os.path.abspath(__file__))), "zkevm-circuits_b200"))

from .lib import ZkbError, load_library, Context, default_context, init_comm_local  # noqa: E402,F401
