"""CFG-Zero* (Fan et al., 2025) restated in fp64 numpy, independent of scail_b200: the optimised scale, the guided
velocity and the zero-init rule, as the paper's code states them for one sample."""
import numpy as np


def optimized_scale(u, c):
    """s* = <c, u> / (|u|^2 + 1e-8) over all elements, in fp64."""
    u = np.asarray(u, dtype=np.float64).ravel()
    c = np.asarray(c, dtype=np.float64).ravel()
    return float(np.dot(c, u) / (np.dot(u, u) + 1e-8))


def guided_velocity(u, c, scale, s_star):
    """g = s* u + scale (c - s* u), in fp64."""
    u = np.asarray(u, dtype=np.float64)
    c = np.asarray(c, dtype=np.float64)
    su = s_star * u
    return su + scale * (c - su)


def zero_init(step, k):
    """Step `step` (0-based, counted since reset) uses a velocity of exactly zero iff it is one of the first k."""
    return step < k
