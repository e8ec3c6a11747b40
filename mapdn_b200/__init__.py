"""mapdn_b200 - batched, H100-native MAPDN voltage-control environment step."""
from .network import NetDesc, ProfileDesc  # noqa: F401

__version__ = "0.1.0"
