"""CPU-only check that the resident-window entry points report their errors through the library's one error slot:
each is called with a NULL handle right after an engine-side call has left a different message, and
ctvio_last_error must then return the entry point's own message (no device is touched on this path)."""
import ctypes as C

import pytest

from helpers import pkg

P, I32, I64, F64 = C.c_void_p, C.c_int32, C.c_int64, C.c_double

# entry point -> (argument types after the handle, arguments after the handle, expected message)
CASES = {
    "triangulate": ([I32, P, P, P, P, I32, P, P, P, I32, F64, P], [0, None, None, None, None, 0, None, None, None, 10, 5.0, None],
                    "bad argument"),
    "extend_knots_to": ([I64, P], [0, None], "knots have not been set"),
    "slide_window": ([I32, I32, I32], [0, 0, 0], "knots have not been set"),
    "slide_window_second_new": ([], [], "null handle"),
    "remap_landmarks": ([I32, P, P], [0, None, None], "bad argument"),
    "triangulate_window": ([I32, P, P, P, F64, P, P], [0, None, None, None, 5.0, None, None], "null handle"),
    "triangulate_window_from_table": ([F64, P, P], [5.0, None, None], "null handle"),
    "check_keyframe": ([I32, P, F64, P, P, P, P], [1, None, 0.0, None, None, None, None], "null handle"),
    "feature_table_add": ([I32, P, P], [0, None, None], "null handle"),
    "feature_table_window": ([I32, P, I32, P], [1, None, 10, None], "null handle"),
    "add_image_features_from_table": ([I32, P], [0, None], "null handle"),
    "feature_table_slide": ([I32, P], [0, None], "null handle"),
    "feature_table_landmarks": ([I32, P, P, P], [0, None, None, None], "null handle"),
    "feature_table_map": ([I32, P, I32, I32, P, P, P, P, P, P], [1, None, 10, 0, None, None, None, None, None, None],
                          "null handle"),
    "ingest_feature_cloud": ([I32, I64, I32, P, P, P, P, P, P], [0, 0, 0, None, None, None, None, None, None],
                             "bad feature cloud"),
    "add_image_features_from_slots": ([I32, P, P, P, P, P, P], [0, None, None, None, None, None, None], "null argument"),
    "ingest_imu": ([I32, P, I32, I32, I32, I64], [0, None, 56, 8, 32, 0], "bad IMU record layout"),
    "add_imu_from_table": ([I64, I64, I32, P, I32, I64, P], [0, 0, 0, None, 0, 0, None], "bad argument"),
}


@pytest.fixture(scope="module")
def raw():
    lib = C.CDLL(pkg.load().path)
    lib.ctvio_last_error.restype = C.c_char_p
    lib.ctvio_set_knots.argtypes = [P, I32, P, P]
    return lib


@pytest.mark.parametrize("name", sorted(CASES))
def test_null_handle_error_reaches_last_error(raw, name):
    assert raw.ctvio_set_knots(None, 0, None, None) < 0
    assert raw.ctvio_last_error() == b"need >= 4 knots"
    argtypes, args, message = CASES[name]
    fn = getattr(raw, "ctvio_" + name)
    fn.argtypes = [P] + argtypes
    fn.restype = C.c_int
    assert fn(None, *args) < 0
    assert raw.ctvio_last_error().decode() == message
