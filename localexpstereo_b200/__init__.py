"""localexpstereo_b200 -- H100-native unary-cost + guided-filter engine behind LocalExpStereo's
StereoEnergy interface.  The compute lives in liblexp_cuda.so (hand-written sm_90a kernels behind
the C-ABI of include/lexp_cuda.h); this package is the thin host-side mirror of the reference interface."""
from ._capi import LexpError, SO_PATH  # noqa: F401
from .energy import (COST_FOR_INVALID, PROP_EXPANSION, PROP_LIST, PROP_RANDOM, PROP_RANSAC, VOL_FILL, VOL_PLAIN, VOL_RIGHT_FROM_LEFT, CostVolumeEnergy, Layer, LayerManager, NaiveStereoEnergy, Parameters, Plan, Plane, host_register,  # noqa: F401
                     host_unregister, save_pfm_file)
