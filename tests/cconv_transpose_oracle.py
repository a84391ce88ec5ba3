"""Float64 oracle of continuous_conv_transpose and invert_neighbors_list, written from their contract (DESIGN.md
section 2, the header of csrc/cconv.cu) and not through the forward op's oracle, so that the adjoint identity of
tests/test_oracle_cconv_transpose.py compares two independent statements.  Test infrastructure: numpy only, no GPU."""
import numpy as np


def _axis_taps(u, size, interp):
    """Filter indices [E, T] along one axis and their weights [E, T] (T = 1 for nearest, 2 for the linear kinds).
    Indices are clamped to the filter; linear_border (interp 2) gives a weight of 0 to an index outside it."""
    if interp == 0:
        return np.clip(np.floor(u + 0.5), 0, size - 1).astype(np.int64)[:, None], np.ones((len(u), 1))
    fl = np.floor(u)
    c = fl[:, None] + np.array([0.0, 1.0])
    w = np.stack([1.0 - (u - fl), u - fl], 1)
    if interp == 2:
        w = np.where((c < 0) | (c >= size), 0.0, w)
    return np.clip(c, 0, size - 1).astype(np.int64), w


def continuous_conv_transpose(filters, out_pos, out_imp, extents, offset, inp_pos, feat, inp_imp_sum, inp_splits,
                              nbr, nbr_imp, splits, align_corners, mapping, normalize, interp):
    """out [num_out, Cout] float32: for output j and entry e of its list, i = nbr[e],
        q = (out_pos[j] - inp_pos[i]) * 2 / extent_i + offset     (extent_i = extents[i] for [num_inp] extents)
        out[j] = oimp_j * sum_e nimp_e * s_i * W(u(q))^T feat[i]
    s_i = 1 / inp_imp_sum[i], or 1 / the length of row i of inp_splits, under normalize; 1 for a zero divisor and
    without normalize.  mapping 0 identity / 1 ball_to_cube_radial; interp 0 nearest / 1 linear / 2 linear_border.
    A corner is skipped on its interpolation weight alone, so a non-finite feature of zero importance propagates.
    None for an importance, inp_imp_sum or inp_splits means "not given"."""
    filters = np.asarray(filters, np.float64)
    sz, sy, sx, cin, cout = filters.shape
    S = np.array([sx, sy, sz])
    out_pos = np.asarray(out_pos, np.float64).reshape(-1, 3)
    inp_pos = np.asarray(inp_pos, np.float64).reshape(-1, 3)
    feat = np.asarray(feat, np.float64).reshape(-1, cin)
    ext = np.asarray(extents, np.float64).reshape(-1)
    nbr, splits = np.asarray(nbr, np.int64), np.asarray(splits, np.int64)
    num_out = len(out_pos)
    if normalize and inp_imp_sum is None and inp_splits is None:
        raise ValueError("normalize needs inp_imp_sum or inp_splits")
    out = np.zeros((num_out, cout))
    e_count = int(splits[-1]) if len(splits) else 0
    if e_count:
        with np.errstate(invalid="ignore", over="ignore"):      # non-finite features propagate, as in the kernel
            j = np.repeat(np.arange(num_out), np.diff(splits))
            i = nbr[:e_count]
            ext_i = ext[i] if len(ext) > 1 else np.full(e_count, ext[0])
            inv = np.where(ext_i > 0, 2.0 / np.where(ext_i > 0, ext_i, 1.0), 0.0)
            q = (out_pos[j] - inp_pos[i]) * inv[:, None] + np.asarray(offset, np.float64).reshape(1, 3)
            if mapping == 1:
                length = np.sqrt((q * q).sum(1))
                mx = np.abs(q).max(1)
                q = np.where(mx[:, None] > 0, q * (length / np.where(mx > 0, mx, 1.0))[:, None], 0.0)
            u = (q + 1) * 0.5 * (S - 1) if align_corners else (q + 1) * 0.5 * S - 0.5
            s = np.ones(e_count)
            if normalize:
                d = (np.asarray(inp_imp_sum, np.float64)[i] if inp_imp_sum is not None
                     else np.diff(np.asarray(inp_splits, np.int64))[i].astype(np.float64))
                s = np.where(d != 0, 1.0 / np.where(d != 0, d, 1.0), 1.0)
            scale = s * (1.0 if nbr_imp is None else np.asarray(nbr_imp, np.float64)[:e_count])
            x = feat[i] * scale[:, None]                                                      # [E, Cin]
            taps = [_axis_taps(u[:, a], S[a], interp) for a in range(3)]
            flat = filters.reshape(-1, cin, cout)
            for ax in range(taps[0][0].shape[1]):
                for ay in range(taps[1][0].shape[1]):
                    for az in range(taps[2][0].shape[1]):
                        w = taps[0][1][:, ax] * taps[1][1][:, ay] * taps[2][1][:, az]
                        cell = (taps[2][0][:, az] * S[1] + taps[1][0][:, ay]) * S[0] + taps[0][0][:, ax]
                        contrib = np.einsum("ec,eco->eo", x * w[:, None], flat[cell])
                        np.add.at(out, j, np.where(w[:, None] == 0, 0.0, contrib))
    if out_imp is not None:
        out *= np.asarray(out_imp, np.float64)[:, None]
    return out.astype(np.float32)


def invert_neighbors_list(num_points, idx, splits):
    """Counting sort of the entries by id: row j lists, in input order, the input rows of the entries whose id is j;
    ids outside [0, num_points) go to a last bucket after row num_points - 1, also in input order.
    -> (neighbors_index int64 [E], neighbors_row_splits int64 [num_points + 1], permutation int64 [E])."""
    idx, splits = np.asarray(idx, np.int64), np.asarray(splits, np.int64)
    keys = [int(v) if 0 <= v < num_points else num_points for v in idx[:splits[-1]]]
    count = [0] * (num_points + 2)
    for k in keys:
        count[k + 1] += 1
    for k in range(num_points + 1):
        count[k + 1] += count[k]
    row_splits = np.array(count[:num_points + 1], np.int64)      # entries of a smaller key
    fill = list(count)
    out_idx, perm = np.zeros(len(keys), np.int64), np.zeros(len(keys), np.int64)
    for row in range(len(splits) - 1):
        for e in range(splits[row], splits[row + 1]):
            t = fill[keys[e]]
            fill[keys[e]] += 1
            out_idx[t], perm[t] = row, e
    return out_idx, row_splits, perm
