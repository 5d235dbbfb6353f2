"""H100-native (sm_90a) implementation of the 3DHumanGAN generator/discriminator hot path.

The directory name starts with a digit, so import it with
    pkg = importlib.import_module("3dhumangan_b200")
or put `3dhumangan_b200/dropin` on PYTHONPATH to get the reference's own import paths
(`lib.generators`, `lib.discriminators`, `lib.implicit_funcitions`, `configs`).
"""
from . import configs, rng, synthetic  # noqa: F401
