"""pilco_b200 -- H100-native engine for the PILCO moment-matching rollout path.

Public API mirrors nrontsis/PILCO: ``models.{MGPR,SMGPR,PILCO}``, ``controllers.{RbfController,
LinearController,squash_sin}``, ``rewards.{ExponentialReward,LinearReward,CombinedRewards}``.
The compute path is hand-written sm_90a CUDA behind the C ABI in ``include/pilco_b200.h``; importing
this package without the built shared library raises (no CPU fallback).
"""
from . import _lib            # noqa: F401  (fails loudly if the .so is missing)
from . import models, controllers, rewards   # noqa: F401
