"""fiducials_b200 -- H100-native (sm_90a) implementation of the aruco_detect + fiducial_slam hot path.

The product is the C-ABI shared library ``libfiducials_b200.so`` (include/fiducials_b200.h) built from
``fiducials_b200/csrc``; this package is the thin python host mirror used by tests and bench.py.
"""
__version__ = "0.1.0"
