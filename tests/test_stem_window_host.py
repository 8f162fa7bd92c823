"""Host restatement (no GPU) of the fused RGB stem's image window (conv_umma.cu, stem_body): the 2-D tile geometry, the
window fill by the 128 producer threads in all three input modes (fp32 image, uint8 with Keras caffe or tf preprocessing,
zeros outside the image after preprocessing), and the builder's k -> window index.  Built tile by tile, the patch rows must
be exactly the im2col patch matrix of the preprocessed image, at the shapes the GPU tests run and at the edges of the
geometry: ragged tiles, asymmetric padding, 1 and 4 input channels, K = 256, a 600-pixel-wide image."""
import numpy as np
import pytest

BM, BK, PROD = 128, 64, 128
TILE_W = 16
WIN_VALS = 24 * 1024 // 4
FILL = WIN_VALS // PROD
CAFFE_SHIFT = np.array([-103.939, -116.779, -123.68], dtype=np.float32)


def stem_tile(ho, wo, kh, kw, sh, sw, cin):
    tile_w = min(wo, TILE_W)
    tile_h = min(BM // tile_w, ho)
    return tile_h, tile_w, (tile_h - 1) * sh + kh, ((tile_w - 1) * sw + kw) * cin


def preprocess(img, mode):
    """The conv input the stem reads: the fp32 image, or the uint8 image through Keras caffe / tf preprocess_input."""
    if mode == "f32":
        return img
    x = img.astype(np.float32)
    if mode == "caffe":
        return x[..., ::-1] + CAFFE_SHIFT
    return x / np.float32(127.5) - np.float32(1)


def fill(img, mode, geo, n0, h0, w0):
    """stem_fill_load + stem_fill_store: thread p holds window values p + 128 j; raw values, then the conversion."""
    H, W, cin, sh, sw, pad_t, pad_l, win_rows, win_cols = geo
    rowlen, nwin = W * cin, win_rows * win_cols
    flat = img[n0].reshape(H, rowlen)
    ih0, col0 = h0 * sh - pad_t, (w0 * sw - pad_l) * cin
    dq, dm = PROD // win_cols, PROD % win_cols
    win = np.full(WIN_VALS, np.nan, dtype=np.float32)
    for p in range(PROD):
        wr, wc = divmod(p, win_cols)
        c = wc % 3
        raw = []
        for j in range(FILL):
            ih, col = ih0 + wr, col0 + wc
            inside = p + PROD * j < nwin and 0 <= ih < H and 0 <= col < rowlen
            if mode == "f32":
                raw.append(flat[ih, col] if inside else np.float32(0))
            else:
                raw.append(int(flat[ih, col + (2 - 2 * c if mode == "caffe" else 0)]) if inside else 0x100)
            wr, wc = wr + dq, wc + dm
            if wc >= win_cols:
                wc, wr = wc - win_cols, wr + 1
            c = 2 if c == 0 else c - 1
        c = (p % win_cols) % 3
        for j in range(FILL):
            e = p + PROD * j
            if e < nwin:
                if mode == "f32":
                    v = raw[j]
                elif raw[j] > 255:
                    v = np.float32(0)
                elif mode == "caffe":
                    v = np.float32(raw[j]) + CAFFE_SHIFT[c]
                else:
                    v = np.float32(raw[j]) / np.float32(127.5) - np.float32(1)
                win[e] = v
            c = 2 if c == 0 else c - 1
    return win


def build_index(tile_h, tile_w, kh, kw, sh, sw, cin, win_cols, k_pad):
    """stem_build: window index of (patch row r, k) for k < K (the incremental walk of the kernel), -1 beyond."""
    run, K = kw * cin, kh * kw * cin
    idx = np.full((BM, k_pad), -1, dtype=np.int64)
    for r in range(BM):
        th, tw = divmod(r, tile_w)
        if th >= tile_h:
            th = tw = 0
        row_base = th * sh * win_cols + tw * sw * cin
        for kb in range(k_pad // BK):
            k = kb * BK
            a, jj = divmod(k, run)
            src = row_base + a * win_cols + jj
            for _ in range(BK):
                if k < K:
                    idx[r, k] = src
                k, src, jj = k + 1, src + 1, jj + 1
                if jj == run:
                    jj, src = 0, src + win_cols - run
    return idx


def im2col(x, kh, kw, sh, sw, pad_t, pad_l, ho, wo, k_pad):
    n, H, W, cin = x.shape
    xp = np.zeros((n, H + kh + ho * sh, W + kw + wo * sw, cin), dtype=np.float32)
    xp[:, pad_t:pad_t + H, pad_l:pad_l + W] = x
    cols = np.zeros((n, ho, wo, k_pad), dtype=np.float32)
    K = kh * kw * cin
    for a in range(kh):
        for b in range(kw):
            patch = xp[:, a:a + (ho - 1) * sh + 1:sh, b:b + (wo - 1) * sw + 1:sw]
            k0 = (a * kw + b) * cin
            cols[..., k0:k0 + cin] = patch
    assert k0 + cin == K
    return cols


# batch, h, w, cin, k, s, (pad t, b), (pad l, r)
SHAPES = {
    "resnet": (2, 224, 224, 3, 7, 2, (3, 3), (3, 3)),
    "vgg": (1, 224, 224, 3, 3, 1, (1, 1), (1, 1)),
    "straddle": (3, 61, 47, 3, 7, 2, (3, 2), (1, 4)),
    "cin1_5x5": (2, 40, 36, 1, 5, 1, (2, 2), (2, 2)),
    "cin4_k256": (2, 64, 64, 4, 8, 2, (3, 3), (3, 3)),
    "wide": (1, 16, 600, 3, 7, 2, (3, 3), (3, 3)),
    "narrow": (2, 9, 11, 3, 3, 1, (0, 2), (1, 0)),    # output narrower than a tile: 12 x 10 pixels, 8 rows unused
}


def _image(shape, mode, seed):
    b, h, w, cin = shape
    rng = np.random.default_rng(seed)
    if mode == "f32":
        return rng.standard_normal((b, h, w, cin)).astype(np.float32)
    return rng.integers(0, 256, size=(b, h, w, cin), dtype=np.uint8)


def _patch_rows(img, mode, b, h, w, cin, k, s, pads, padl, shift=(0, 0)):
    ho = (h + sum(pads) - k) // s + 1
    wo = (w + sum(padl) - k) // s + 1
    K = k * k * cin
    k_pad = (K + 63) // 64 * 64
    tile_h, tile_w, win_rows, win_cols = stem_tile(ho, wo, k, k, s, s, cin)
    assert win_rows * win_cols <= WIN_VALS
    geo = (h, w, cin, s, s, pads[0], padl[0], win_rows, win_cols)
    idx = build_index(tile_h, tile_w, k, k, s, s, cin, win_cols, k_pad)
    out = np.full((b, ho, wo, k_pad), np.nan, dtype=np.float32)
    tiles_h, tiles_w = -(-ho // tile_h), -(-wo // tile_w)
    for n0 in range(b):
        for ti in range(tiles_h):
            for tj in range(tiles_w):
                h0, w0 = ti * tile_h, tj * tile_w
                win = fill(img, mode, geo, n0, h0 + shift[0], w0 + shift[1])
                rows = np.where(idx >= 0, win[np.maximum(idx, 0)], np.float32(0))
                for r in range(tile_h * tile_w):
                    oh, ow = h0 + r // tile_w, w0 + r % tile_w
                    if oh < ho and ow < wo:       # the epilogue stores no other row
                        out[n0, oh, ow] = rows[r]
    return out, (ho, wo, k_pad)


@pytest.mark.parametrize("mode", ["f32", "caffe", "tf"])
@pytest.mark.parametrize("name", list(SHAPES))
def test_window_rows_are_the_patch_matrix(name, mode):
    b, h, w, cin, k, s, pads, padl = SHAPES[name]
    if mode != "f32" and cin != 3:
        pytest.skip("uint8 ingress is 3-channel RGB")
    if name in ("resnet", "vgg", "wide") and mode != "f32":
        b = 1
    img = _image((b, h, w, cin), mode, seed=len(name))
    out, (ho, wo, k_pad) = _patch_rows(img, mode, b, h, w, cin, k, s, pads, padl)
    ref = im2col(preprocess(img, mode), k, k, s, s, pads[0], padl[0], ho, wo, k_pad)
    assert np.array_equal(out.view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("shift", [(0, 1), (1, 0)])
def test_a_shifted_window_origin_is_caught(shift):
    b, h, w, cin, k, s, pads, padl = SHAPES["straddle"]
    img = _image((1, h, w, cin), "caffe", seed=1)
    out, (ho, wo, k_pad) = _patch_rows(img, "caffe", 1, h, w, cin, k, s, pads, padl, shift=shift)
    ref = im2col(preprocess(img, "caffe"), k, k, s, s, pads[0], padl[0], ho, wo, k_pad)
    assert not np.array_equal(out, ref)


def test_geometry():
    # ResNet 7x7/2 at 224: 8 x 16 tiles, 14 x 7 per image, a 21 x 111 window (9.3 KB)
    assert stem_tile(112, 112, 7, 7, 2, 2, 3) == (8, 16, 21, 111)
    # VGG 3x3/1 at 224: 10 x 54 (2.2 KB)
    assert stem_tile(224, 224, 3, 3, 1, 1, 3) == (8, 16, 10, 54)
    # 32 channels, 2x2/2: 16 x 1024 values, over the 24 KB buffer: stays on the im2col path
    _, _, r, c = stem_tile(112, 112, 2, 2, 2, 2, 32)
    assert r * c > WIN_VALS
