"""The generation of a framed follower's query (include/chd_gpu_facing.h) restated in numpy: every product, sum, square root and
quotient is one IEEE f64 operation rounded on its own, in the header's order, so the device's results compare bit for bit."""
import numpy as np


def has_facing(fx, fz):
    """A facing is one when both components are finite and not both zero."""
    fx, fz = np.asarray(fx, np.float64), np.asarray(fz, np.float64)
    return np.isfinite(fx) & np.isfinite(fz) & ((fx != 0) | (fz != 0))


def frame_query(x, z, fx, fz, off_fwd, off_right, rot_cos, rot_sin, cone_dx, cone_dz):
    """-> (fx, fz, cx, cz, dx, dz) of the query a framed follower gets from its entity at (x, z) with facing (fx, fz): the facing
    the query used (0, 0: none), its centre and its cone direction (none: the entity's position and the bound direction)."""
    a = [np.asarray(v, np.float64) for v in (x, z, fx, fz, off_fwd, off_right, rot_cos, rot_sin, cone_dx, cone_dz)]
    a = np.broadcast_arrays(*a)
    x, z, fx, fz, fwd, right, rc, rs, cdx, cdz = a
    has = has_facing(fx, fz)
    fx = np.where(has, fx, 0.0)
    fz = np.where(has, fz, 0.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        m = np.sqrt(fx * fx + fz * fz)
        ux, uz = fx / m, fz / m
        cx = np.where(has, (x + fwd * ux) - right * uz, x)
        cz = np.where(has, (z + fwd * uz) + right * ux, z)
        dx = np.where(has, fx * rc - fz * rs, cdx)
        dz = np.where(has, fx * rs + fz * rc, cdz)
    return fx, fz, cx, cz, dx, dz
