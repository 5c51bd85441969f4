import hashlib

import numpy as np


def digest(a):
    """SHA-256 of an array's values and shape: equal digests <=> np.array_equal(a, b, equal_nan=True) for arrays of
    the same kind (floats compared as float64 with NaNs and the sign of zero made canonical, integers as int64)."""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        a = a.astype(np.float64) + 0.0  # -0.0 -> +0.0
        a = np.where(np.isnan(a), np.nan, a)
    elif a.dtype.kind in "iub":
        a = a.astype(np.int64)
    a = np.ascontiguousarray(a)
    return hashlib.sha256(f"{a.dtype.kind}{a.shape}".encode() + a.tobytes()).hexdigest()


def bits_equal(a, b):
    """Bit-for-bit equality of float64 arrays (NaN == NaN when the payload matches or both NaN)."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    return bool(((a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))).all())


def pose_error(Xa, Xb):
    """(rotation angle [rad], translation distance [m]) between two 3x4 / 4x4 poses."""
    Xa, Xb = np.asarray(Xa)[:3], np.asarray(Xb)[:3]
    dR = Xa[:, :3] @ Xb[:, :3].T
    # atan2 form: arccos((tr-1)/2) has a ~2e-8 rad noise floor near the identity
    s = 0.5 * np.linalg.norm([dR[2, 1] - dR[1, 2], dR[0, 2] - dR[2, 0], dR[1, 0] - dR[0, 1]])
    ang = float(np.arctan2(s, (np.trace(dR) - 1.0) / 2.0))
    return ang, float(np.linalg.norm(Xa[:, 3] - Xb[:, 3]))


# north_star tolerances
POSE_RAD, POSE_M = 1e-5, 1e-4
# H/b: relative to the largest |entry| (the CPU sums ~1e5 terms sequentially; SURVEY 8d asks 1e-12)
HB_REL = 1e-12
