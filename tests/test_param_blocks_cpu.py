"""The parameter-block rules of the prior and the marginalization (csrc/param_blocks.h), compiled with plain g++.

No GPU needed: tests/emu/param_blocks.cpp wraps the header's functions in a small shared library.  They are checked
against the camera-dim layout of include/ctvio.h (np = 6*n_knots + 6*n_bias + 1: rot, pos per knot, then bg, ba per
bias node, then the line delay), against a restatement of the reference's drop set of the old prior
(trajectory_manager.cpp:166-203), and for every message of the prior's column-tiling check.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROT, POS, BG, BA, LD, RHO = range(6)  # CTVIO_BLK_*
WINDOWS = [(4, 0), (4, 1), (7, 3), (12, 6)]  # (n_knots, n_bias)


@pytest.fixture(scope="module")
def pb(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("param_blocks") / "libparam_blocks.so")
    src = os.path.join(HERE, "emu", "param_blocks.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", src, "-o", so], check=True)
    lib = C.CDLL(so)
    lib.pb_prior_tiling_error.restype = C.c_char_p
    return lib


def window_blocks(nK, nB):
    """Every block of a window in the order the layout puts them, with its first camera dim and size."""
    out = []
    for k in range(nK):
        out += [(ROT, k, 6 * k, 3), (POS, k, 6 * k + 3, 3)]
    for b in range(nB):
        out += [(BG, b, 6 * nK + 6 * b, 3), (BA, b, 6 * nK + 6 * b + 3, 3)]
    return out + [(LD, 0, 6 * nK + 6 * nB, 1)]


def test_block_dim_and_kind(pb):
    assert [pb.pb_block_dim(t) for t in range(6)] == [3, 3, 3, 3, 1, 1]
    assert [pb.pb_block_is_knot(t) for t in range(-1, 7)] == [0, 1, 1, 0, 0, 0, 0, 0]
    assert [pb.pb_block_is_bias(t) for t in range(-1, 7)] == [0, 0, 0, 1, 1, 0, 0, 0]


@pytest.mark.parametrize("nK,nB", WINDOWS)
def test_block_base_follows_the_camera_dim_layout(pb, nK, nB):
    for t, i, base, _ in window_blocks(nK, nB):
        assert pb.pb_block_base(t, i, nK, nB) == base, (t, i)
    for t, n in ((ROT, nK), (POS, nK), (BG, nB), (BA, nB)):
        for i in (-1, n, n + 5):
            assert pb.pb_block_base(t, i, nK, nB) == -1, (t, i)
    for i in (-1, 0, 3):
        assert pb.pb_block_base(RHO, i, nK, nB) == -1
    for t in (-1, 6, 100):
        assert pb.pb_block_base(t, 0, nK, nB) == -1


@pytest.mark.parametrize("nK,nB", WINDOWS)
def test_block_order_is_camera_dim_order(pb, nK, nB):
    # the marginalization orders blocks by knots (rot, pos per knot), bias nodes (bg, ba per node), the line delay; keyed
    # by their first camera dim they must come out in that order and tile the np dims without a gap
    blocks = window_blocks(nK, nB)
    rng = np.random.default_rng(nK * 10 + nB)
    shuffled = [blocks[k] for k in rng.permutation(len(blocks))]
    by_base = sorted(shuffled, key=lambda b: pb.pb_block_base(b[0], b[1], nK, nB))
    assert [(t, i) for t, i, _, _ in by_base] == [(t, i) for t, i, _, _ in blocks]
    end = 0
    for t, i, _, _ in by_base:
        assert pb.pb_block_base(t, i, nK, nB) == end
        end += pb.pb_block_dim(t)
    assert end == 6 * nK + 6 * nB + 1


def reference_dropped(t, i, now, later):
    """trajectory_manager.cpp:166-203: the parameter blocks of knots now .. later-1 and of bias node 0."""
    drop = {(ROT, k) for k in range(now, later)} | {(POS, k) for k in range(now, later)} | {(BG, 0), (BA, 0)}
    return (t, i) in drop


def test_prior_block_dropped_matches_the_reference_rule(pb):
    for now in range(0, 5):
        for later in range(0, 8):
            for t in range(6):
                for i in range(-1, 9):
                    assert pb.pb_prior_block_dropped(t, i, now, later) == reference_dropped(t, i, now, later), \
                        (t, i, now, later)


def tiling(pb, n, blocks):
    t = np.array([b[0] for b in blocks], dtype=np.int32)
    c = np.array([b[1] for b in blocks], dtype=np.int32)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    msg = pb.pb_prior_tiling_error(n, len(blocks), ip(t), ip(c))
    return None if msg is None else msg.decode()


def test_prior_tiling_check(pb):
    # (type, col) pairs
    assert tiling(pb, 11, [(ROT, 0), (POS, 3), (BG, 6), (LD, 9), (RHO, 10)]) is None
    assert tiling(pb, 7, [(BA, 4), (LD, 3), (ROT, 0)]) is None
    assert tiling(pb, 3, [(6, 0)]) == "prior block type out of range"
    assert tiling(pb, 3, [(-1, 0)]) == "prior block type out of range"
    assert tiling(pb, 4, [(ROT, 0), (LD, 4)]) == "prior block column outside [0, n)"
    assert tiling(pb, 4, [(LD, -1), (ROT, 0)]) == "prior block column outside [0, n)"
    assert tiling(pb, 4, [(ROT, 2)]) == "prior block column outside [0, n)"
    assert tiling(pb, 6, [(ROT, 0), (POS, 2)]) == "prior blocks overlap"
    assert tiling(pb, 4, [(LD, 3), (RHO, 3)]) == "prior blocks overlap"
    assert tiling(pb, 7, [(ROT, 0), (POS, 4)]) == "prior blocks do not cover all n columns"
    assert tiling(pb, 4, [(ROT, 0)]) == "prior blocks do not cover all n columns"
    # the first failure in block order is the one reported
    assert tiling(pb, 6, [(ROT, 0), (ROT, 2), (7, 0)]) == "prior blocks overlap"
