"""cosmo_b200: H100-native ADMM iteration engine behind COSMO.jl's solver API.

The directory is named ``cosmo.jl_b200`` (not importable as written); the
top-level shim ``cosmo_b200.py`` registers it under the name ``cosmo_b200``.
"""
from .engine import Engine, EngineError, default_settings, load_library, nccl_unique_id  # noqa: F401
from .model import (Box, ComplexPsdConeTriangle, Constraint, CustomCone, CustomConeType, DualExponentialCone,  # noqa: F401
                    DualPowerCone, ExponentialCone, Model, Nonnegatives, PowerCone, PsdCone, PsdConeTriangle, Result, ResultInfo, SecondOrderCone, Settings,
                    ZeroSet, assemble, optimize, ruiz_equilibrate)
from . import problems  # noqa: F401
from . import sharding  # noqa: F401,E402
from . import chordal  # noqa: F401,E402
