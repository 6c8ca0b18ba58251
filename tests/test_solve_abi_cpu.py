"""CPU-only check that the LM driver's entry point (solve.cu) reports its errors through the library's one error slot:
ctvio_solve is called with a NULL handle right after an engine.cu call has left a different message, and
ctvio_last_error must then return ctvio_solve's own message (no device is touched on this path)."""
import ctypes as C

from helpers import pkg

P, I32 = C.c_void_p, C.c_int32


def test_solve_null_handle_error_reaches_last_error():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_set_knots.argtypes = [P, I32, P, P]
    lib.ctvio_solve.argtypes = [P, I32, P]
    lib.ctvio_solve.restype = C.c_int
    assert lib.ctvio_set_knots(None, 0, None, None) < 0
    assert lib.ctvio_last_error() == b"need >= 4 knots"
    assert lib.ctvio_solve(None, 15, None) < 0
    assert lib.ctvio_last_error() == b"null handle"
