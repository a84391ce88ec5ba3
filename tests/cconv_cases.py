"""Far-neighbour cases of continuous_conv, shared by tests/test_oracle_ops.py (the C oracle) and
tests/test_gpu_cconv_forward.py (the kernel): neighbours so far outside the filter that the filter coordinate u is
beyond the range of a 32-bit int, where converting floor(u) to int before clamping it picks the wrong border cell.

Test infrastructure, not product code: nothing under open3d-ml_b200/ imports it.
"""
from collections import namedtuple

import numpy as np

FAR = (1e3, 1e9, 1e12)

Case = namedtuple("Case", "filters out_pos inp_pos feat index splits want")


def far_neighbours(sizes, align, interp, mags=FAR):
    """One output per (axis, side, magnitude), all at the same point c, each with one neighbour at c + side * mag along
    that axis; extent 1 and offset 0, so p = 2 * side * mag on that axis and 0 on the other two.  Cin = Cout = 1, one
    feature of 1, and a filter whose value at each cell is its flat index (z * Sy + y) * Sx + x, sizes = (Sx, Sy, Sz).

    want is the closed-form output: nearest and linear take the border cell (0 on the - side, S - 1 on the + side) on
    the far axis and the filter coordinate of p = 0 on the other two (its nearest cell, or the coordinate itself under
    linear, since linear interpolation of the flat index is exact); linear_border weighs every corner 0, except on
    an axis of size 1 under align_corners, where every p lies on the one cell.  The
    identity and ball_to_cube_radial mappings agree here: p lies on an axis, where |p|_2 = |p|_inf."""
    S = np.array(sizes, np.int64)
    filters = np.arange(S.prod(), dtype=np.float32).reshape(S[2], S[1], S[0], 1, 1)
    centre = np.float32([0.5, 0.25, 0.75])
    u0 = (S - 1) / 2.0 if align else S / 2.0 - 0.5                      # the filter coordinate of p = 0
    mid = np.floor(u0 + 0.5) if interp == 0 else u0
    inp, want = [], []
    for a in range(3):
        for side in (-1, 1):
            for mag in mags:
                p = centre.astype(np.float64)
                p[a] += side * mag
                inp.append(p)
                cell = mid.copy()
                cell[a] = 0 if side < 0 else S[a] - 1
                outside = not (align and S[a] == 1)        # align_corners maps every p to u = 0 on an axis of size 1
                want.append(0.0 if interp == 2 and outside else (cell[2] * S[1] + cell[1]) * S[0] + cell[0])
    m = len(inp)
    return Case(filters, np.tile(centre, (m, 1)), np.array(inp, np.float32), np.ones((m, 1), np.float32),
                np.arange(m, dtype=np.int64), np.arange(m + 1, dtype=np.int64),
                np.array(want, np.float32).reshape(m, 1))
