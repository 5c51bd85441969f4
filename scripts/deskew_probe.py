"""Host deskew timing per thread count (run it on a host with many physical cores)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from mad_icp_b200 import synth
from mad_icp_b200.pybind.pypeline import Pipeline, VectorEigen3d

pts = np.ascontiguousarray(synth.registration_case(K=1)["scans"][0])
Ta, Tb = synth.pose_xyyaw(0.0, 1.0, 0.0), synth.pose_xyyaw(0.8, 1.05, 0.03)
v = VectorEigen3d(pts)
os.environ["MADTREE_TIMING"] = "1"
for thr in (1, 1, 4, 4, 16, 16, 16, 32, 32):
    Pipeline._deskewOnly(v, Ta, Tb, 10.0, thr)
