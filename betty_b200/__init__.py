"""betty_b200 -- H100-native hypergradient engine behind ``betty.hypergradient.{neumann, cg, darts}``."""
from . import hypergradient  # noqa: F401
from .hypergradient import install  # noqa: F401

__version__ = "0.1.0"
