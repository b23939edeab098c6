"""NumPy restatement of csrc/exposure.cu (sb_exposure_apply, sb_exposure_backward), the rule include/splatam_b200.h
states.  The apply and gx are float32, each operation rounded as the kernel rounds it, so they equal the kernel bit for
bit; the two sums of the backward are float64 (math.fsum, exact before the final rounding), which the kernel's fixed
block order matches to about 1e-15 relative."""
import math

import numpy as np


def gains(ab, inverse=False):
    """float32 [3]: float(exp(+-double(a_c)))."""
    a = np.asarray(ab, dtype=np.float32)[:3].astype(np.float64)
    return np.exp(-a if inverse else a).astype(np.float32)


def apply(x, ab, inverse=False):
    """x float32 [3,H,W], ab float32 [6] -> y float32 [3,H,W]."""
    x = np.asarray(x, dtype=np.float32)
    g = gains(ab, inverse)[:, None, None]
    b = np.asarray(ab, dtype=np.float32)[3:6, None, None]
    if inverse:
        return ((x - b).astype(np.float32) * g).astype(np.float32)
    return ((g * x).astype(np.float32) + b).astype(np.float32)


def backward(x, ab, gy):
    """-> (gx float32 [3,H,W], g_ab float64 [6] = (exp(a_c) sum_c gy x, sum_c gy))."""
    x, gy = np.asarray(x, dtype=np.float32), np.asarray(gy, dtype=np.float32)
    gx = (gains(ab)[:, None, None] * gy).astype(np.float32)
    a = np.asarray(ab, dtype=np.float32)[:3].astype(np.float64)
    x64, g64 = x.astype(np.float64).reshape(3, -1), gy.astype(np.float64).reshape(3, -1)
    s = np.array([math.fsum(x64[c] * g64[c]) for c in range(3)])
    g = np.array([math.fsum(g64[c]) for c in range(3)])
    return gx, np.concatenate([np.exp(a) * s, g])
