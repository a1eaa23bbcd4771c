"""raisimlib_b200 -- H100-native batched rigid-body step behind the RaiSim World::integrate() surface.

The product is the CUDA library (csrc/ -> librsb.so, C-ABI in include/rsb.h) and the header-only
C++ facade in include/raisim/.  This Python package only binds the C-ABI for tests and bench.py.
"""
from .capi import Model, Batch, RsbError, KMAX, HOST, DEVICE, FORCE_AND_TORQUE, PD_PLUS_FEEDFORWARD_TORQUE  # noqa: F401
import os

RSC_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rsc")
