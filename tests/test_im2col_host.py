"""The A tile of the wgmma convolution as TMA im2col fills it, restated on the host (defer_b200/csrc/conv_umma.cu).

M tile t of a conv is the 128 consecutive output pixels [128 t, 128 t + 128) in (n, ho, wo) order.  For tap (kh, kw) the
producer issues one im2col load per 64-channel block: the walk starts at the input corner (ow * sw - pad_l,
oh * sh - pad_t, n) of the tile's first output pixel, steps by the stride along a row of the bounding box, goes on at the
box's lower corner of the next row after its last column, and at the first row of the next image after its last row.
Each visited corner is read at the tap offset (kw, kh); pixels outside the input, and rows past the batch, are zeros.
The bounding box (`im2col_corners`) runs from (-pad_l, -pad_t) to the corner of the last output pixel, the upper corner
given as an offset from input pixel (w - 1, h - 1), and a rank-4 tensor map holds corners in [-128, 127].

Row r of tile t must then hold what direct convolution indexing reads for output pixel 128 t + r at that tap.  Checked
on every conv the applications run through im2col (tests/app_convs.py) at batch 1 and 32, and on the edge geometries
tests/test_gpu_conv_im2col.py runs on the GPU."""
import numpy as np
import pytest

import app_convs as C

BM = 128

# geometries (n, h, w, cin, cout, kh, kw, sh, sw, pad t, l, b, r) that the applications do not run; also bit for bit on the
# GPU (tests/test_gpu_conv_im2col.py)
IM2COL_EDGES = {
    "ragged_across_images": (3, 10, 10, 64, 128, 3, 3, 1, 1, 1, 1, 1, 1),   # M = 300: tiles straddle images, last of 44 rows
    "map7_three_images": (5, 7, 7, 128, 128, 3, 3, 1, 1, 1, 1, 1, 1),      # tile 0 holds pixels of images 0, 1 and 2
    "stride2_odd": (2, 17, 17, 128, 64, 3, 3, 2, 2, 1, 1, 1, 1),           # 9 x 9 outputs of an odd input
    "stride2_1x1_odd": (2, 13, 13, 64, 128, 1, 1, 2, 2, 0, 0, 0, 0),
    "zeropad_asym": (2, 14, 14, 64, 64, 3, 3, 2, 2, 0, 0, 1, 1),           # ZeroPadding2D(((0, 1), (0, 1))) + valid 3x3/2
    "pad_1x1_asym": (2, 9, 9, 64, 64, 1, 1, 1, 1, 0, 0, 1, 1),             # 1x1/1 with ho != h: im2col, not the flat view
    "wide_stride2": (1, 5, 301, 64, 64, 3, 3, 2, 2, 1, 1, 1, 1),           # 151 outputs per row, 301 input columns
    "rect_asym": (2, 9, 20, 64, 128, 3, 5, 1, 2, 2, 0, 0, 1),              # W and H corners differ
}


def out_size(geom):
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    return (h + pt + pb - kh) // sh + 1, (w + pl + pr - kw) // sw + 1


def uses_im2col(geom):
    """umma_conv_prepare: every conv but a 1x1 / stride-1 one whose output grid is its input grid."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    return (kh, kw, sh, sw, pt, pl) != (1, 1, 1, 1, 0, 0) or out_size(geom) != (h, w)


def im2col_corners(h, w, ho, wo, sh, sw, pt, pl):
    """(lower, upper) corners of the bounding box in (W, H) order, as the tensor map takes them."""
    return (-pl, -pt), ((wo - 1) * sw - pl - (w - 1), (ho - 1) * sh - pt - (h - 1))


def tile_start(t, ho, wo, sh, sw, pt, pl):
    """The producer's coordinates of the walk of tile t: input corner (x, y) and image of output pixel 128 t."""
    m0 = t * BM
    ow, oh, n0 = m0 % wo, (m0 // wo) % ho, m0 // (wo * ho)
    return ow * sw - pl, oh * sh - pt, n0


def walk(geom, t):
    """The 128 corners (n, y, x) TMA visits for tile t, one pixel after another."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    ho, wo = out_size(geom)
    lo, up = im2col_corners(h, w, ho, wo, sh, sw, pt, pl)
    x_end, y_end = w - 1 + up[0], h - 1 + up[1]
    x, y, nn = tile_start(t, ho, wo, sh, sw, pt, pl)
    out = np.empty((BM, 3), np.int64)
    for r in range(BM):
        out[r] = nn, y, x
        x += sw
        if x > x_end:
            x, y = lo[0], y + sh
            if y > y_end:
                y, nn = lo[1], nn + 1
    return out


def tile_rows(geom, t, tap):
    """Linear input pixel (n, iy, ix) that row r of tile t holds for tap (a, b), or -1 where TMA fills zeros."""
    n, h, w = geom[:3]
    c = walk(geom, t)
    nn, iy, ix = c[:, 0], c[:, 1] + tap[0], c[:, 2] + tap[1]
    inside = (nn < n) & (iy >= 0) & (iy < h) & (ix >= 0) & (ix < w)
    return np.where(inside, (nn * h + iy) * w + ix, -1)


def direct_rows(geom, t, tap):
    """Linear input pixel direct convolution reads for output pixels 128 t + r (-1: padding; rows past the output: -1)."""
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    ho, wo = out_size(geom)
    m = t * BM + np.arange(BM)
    nn, rem = np.divmod(m, ho * wo)
    oh, ow = np.divmod(rem, wo)
    iy, ix = oh * sh - pt + tap[0], ow * sw - pl + tap[1]
    inside = (m < n * ho * wo) & (iy >= 0) & (iy < h) & (ix >= 0) & (ix < w)
    return np.where(inside, (nn * h + iy) * w + ix, -1)


def check_geometry(geom):
    n, h, w, cin, cout, kh, kw, sh, sw, pt, pl, pb, pr = geom
    ho, wo = out_size(geom)
    lo, up = im2col_corners(h, w, ho, wo, sh, sw, pt, pl)
    assert all(-128 <= v <= 127 for v in lo + up), (geom, lo, up)        # encodable in a rank-4 tensor map
    assert ((w - 1 + up[0]) - lo[0]) // sw + 1 == wo and ((h - 1 + up[1]) - lo[1]) // sh + 1 == ho   # a box row = an output row
    m_total = n * ho * wo
    m_tiles = -(-m_total // BM)
    for t in range(m_tiles):
        c = walk(geom, t)
        m = t * BM + np.arange(BM)
        valid = m < m_total
        nn, rem = np.divmod(m[valid], ho * wo)
        oh, ow = np.divmod(rem, wo)
        # the walk visits exactly the corners of the tile's output pixels, and only images past the batch after them
        np.testing.assert_array_equal(c[valid], np.stack([nn, oh * sh - pt, ow * sw - pl], 1), err_msg=f"{geom} tile {t}")
        assert (c[~valid, 0] >= n).all(), (geom, t)
        for tap in ((0, 0), (kh - 1, kw - 1), (kh // 2, 0), (0, kw - 1)):
            np.testing.assert_array_equal(tile_rows(geom, t, tap), direct_rows(geom, t, tap), err_msg=f"{geom} tile {t} {tap}")
    return m_tiles


APP_IM2COL = {f"{name}@{b}": (b, *g) for name, (g, _, batches) in C.APP_CONVS.items() for b in batches
              if uses_im2col((b, *g))}


def test_resnet50_im2col_convs_are_listed():
    """The 22 im2col launches of ResNet50 at bench.py's batch: its 16 3x3 convs (4 geometries) and 6 strided 1x1s."""
    names = {k.split("@")[0] for k in APP_IM2COL if k.startswith("ResNet50:") and k.endswith(f"@{C.BENCH_BATCH}")}
    assert names == {"ResNet50:res2a_branch2b", "ResNet50:res3a_branch2b", "ResNet50:res4a_branch2b", "ResNet50:res5a_branch2b",
                     "ResNet50:res3a_branch2a", "ResNet50:res3a_branch1", "ResNet50:res4a_branch2a", "ResNet50:res4a_branch1",
                     "ResNet50:res5a_branch2a", "ResNet50:res5a_branch1"}


@pytest.mark.parametrize("name", list(APP_IM2COL))
def test_app_conv_tiles(name):
    check_geometry(APP_IM2COL[name])


@pytest.mark.parametrize("name", list(IM2COL_EDGES))
def test_edge_tiles(name):
    check_geometry(IM2COL_EDGES[name])


def test_tile_counts():
    """Flat tiles: ceil(N * Ho * Wo / 128), e.g. 49 instead of 64 at 14 x 14 and 13 instead of 16 at 7 x 7 (batch 32)."""
    assert check_geometry(APP_IM2COL["ResNet50:res4a_branch2b@32"]) == 49
    assert check_geometry(APP_IM2COL["ResNet50:res5a_branch2b@32"]) == 13
    assert check_geometry(APP_IM2COL["ResNet50:res4a_branch1@32"]) == 49


def test_edges_reach_what_they_name():
    g = IM2COL_EDGES
    ho, wo = out_size(g["ragged_across_images"])
    assert (g["ragged_across_images"][0] * ho * wo) % BM and (BM % (ho * wo))                # ragged, tiles straddle images
    assert len({int(v) for v in walk(g["map7_three_images"], 0)[:, 0]}) == 3
    assert g["stride2_odd"][1] % 2 == 1 and g["stride2_odd"][7] == 2
    assert out_size(g["zeropad_asym"]) != g["zeropad_asym"][1:3] and out_size(g["pad_1x1_asym"]) != g["pad_1x1_asym"][1:3]
    assert out_size(g["wide_stride2"])[1] * 2 > 256
    lo, up = im2col_corners(*g["rect_asym"][1:3], *out_size(g["rect_asym"]), *g["rect_asym"][7:9], *g["rect_asym"][9:11])
    assert lo[0] != lo[1] and up[0] != up[1]                                                   # W and H corners differ
