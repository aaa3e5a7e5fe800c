"""Drop-in shim: ``import cityflow`` resolves to the H100 engine (same class names as the
reference's pybind11 module, src/cityflow.cpp:10-48)."""
from cityflow_b200 import Archive, Engine, __version__  # noqa: F401
