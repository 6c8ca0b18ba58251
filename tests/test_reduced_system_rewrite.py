"""K4 (reduced_system_kernel) writes every entry the rest of the LM step reads: the lower 64x64 tiles of the reduced
system M (diagonal tiles in full) and rhs, whatever M and rhs held before.

ctvio_debug_lm_step_poison fills M and rhs with NaN before K4 runs.  In deterministic mode the poisoned call must
return, bit for bit, what the plain call returns: M's lower tiles, rhs, the solution y of K5 and the step (dc, dl) of
K6, at C1 (one tile), C2 size (nb = 4) and dag15 (nb = 15, the largest tile-DAG grid).
"""
import ctypes as C

import numpy as np
import pytest

from helpers import pkg
from test_lm_step_regimes import regime_options, regime_window


def lm_step_outputs(est, radius, poison):
    f = est.lib.lib.ctvio_debug_lm_step_poison
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.POINTER(C.c_int64), C.c_int32]
    n = C.c_int64(0)
    assert f(est.h, radius, None, C.byref(n), 0) == 0
    buf = np.full(n.value, np.nan)
    assert f(est.h, radius, buf.ctypes.data, C.byref(n), 1 if poison else 0) == 0, est.lib._fn["last_error"]()
    np_, npad, nL = int(buf[0]), int(buf[1]), int(buf[2])
    pos = 16 + np_ * np_ + np_ + 2 * nL + nL * np_ + 2 * np_ + 2 * nL
    M = buf[pos:pos + npad * npad].reshape(npad, npad)
    pos += npad * npad
    rhs, y = buf[pos:pos + npad], buf[pos + npad:pos + 2 * npad]
    pos += 2 * npad
    dc, dl = buf[pos:pos + np_], buf[pos + np_:pos + np_ + nL]
    assert pos + np_ + nL == len(buf)
    return npad, M, rhs, y, dc, dl


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["c1", "c2", "dag15"])
def test_reduced_system_rewrites_lower_tiles_and_rhs(cuda_lib, name):
    est = pkg.setup_estimator(cuda_lib, regime_window(name), options=regime_options(name))
    est.SetDeterministic(True)
    for radius in (1e4, 1e-3):
        npad, M0, rhs0, y0, dc0, dl0 = lm_step_outputs(est, radius, poison=False)
        _, M1, rhs1, y1, dc1, dl1 = lm_step_outputs(est, radius, poison=True)
        t = np.arange(npad) // 64
        lower_tiles = t[:, None] >= t[None, :]
        bits0, bits1 = M0.view(np.int64), M1.view(np.int64)
        for a in (M1[lower_tiles], rhs1, y1, dc1, dl1):
            assert np.isfinite(a).all(), (name, radius)
        assert np.array_equal(bits1[lower_tiles], bits0[lower_tiles]), (name, radius)
        for a, b in ((rhs0, rhs1), (y0, y1), (dc0, dc1), (dl0, dl1)):
            assert np.array_equal(a.view(np.int64), b.view(np.int64)), (name, radius)
