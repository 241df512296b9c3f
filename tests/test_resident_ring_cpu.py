"""Resident tiles of the fused TV-L1 kernel (tvl1_fused.cu, run_chunk / process_tile): when a level has no more tiles than a
lane has CTAs, every CTA keeps its tile on chip across chunks, reads back only the ring (tile pixels outside its interior)
and writes back only the band (interior pixels within 2h of a tile edge that has a neighbouring tile).  That is exact only
if every in-image ring pixel of every tile lies in the band of the tile whose interior owns it, and the interiors partition
the image.  The predicates below restate the kernel's, at lane granularity (4 pixels), on the tile geometry of
fused_tiles_along."""
import numpy as np
import pytest

import geometry_cases as gc

TW, TH = 128, 64


def tiles_along(n, T, h):
    return 1 if n <= T else (n - 2 * h + (T - 2 * h) - 1) // (T - 2 * h)


def tile_masks(W, H, k, tx, ty, ntx, nty):
    """(interior, band, in-image) of tile (tx, ty) over its 128 x 64 cells, as process_tile computes them"""
    hy, hx = k, (k + 3) & ~3
    rx0, ry0 = tx * (TW - 2 * hx), ty * (TH - 2 * hy)
    lx4 = (np.arange(TW) // 4 * 4)[None, :]  # a lane's four pixels share its predicates
    ry = np.arange(TH)[:, None]
    gx0, gy = rx0 + lx4, ry0 + ry
    lane_in = ((tx == 0) | (lx4 >= hx)) & (lx4 < TW - hx + (hx if rx0 + TW >= W else 0)) & (gx0 < W)
    ry_lo = 0 if ty == 0 else hy
    ry_hi = TH - hy + (hy if ry0 + TH >= H else 0)
    interior = lane_in & (ry >= ry_lo) & (ry < ry_hi) & (gy < H)
    lane_band = ((tx > 0) & (lx4 < 2 * hx)) | ((tx < ntx - 1) & (lx4 >= TW - 2 * hx))
    band = interior & (lane_band | ((ty > 0) & (ry < 2 * hy)) | ((ty < nty - 1) & (ry >= TH - 2 * hy)))
    image = ((rx0 + np.arange(TW))[None, :] < W) & (gy < H)
    return interior, band, image, rx0, ry0


def check_geometry(W, H, k):
    hy, hx = k, (k + 3) & ~3
    ntx, nty = tiles_along(W, TW, hx), tiles_along(H, TH, hy)
    owners = np.zeros((H, W), np.int32)
    in_band = np.zeros((H, W), bool)
    tiles = []
    for ty in range(nty):
        for tx in range(ntx):
            interior, band, image, rx0, ry0 = tile_masks(W, H, k, tx, ty, ntx, nty)
            w, h = min(TW, W - rx0), min(TH, H - ry0)
            owners[ry0:ry0 + h, rx0:rx0 + w] += interior[:h, :w] & image[:h, :w]
            in_band[ry0:ry0 + h, rx0:rx0 + w] |= band[:h, :w] & image[:h, :w]
            assert not (band & ~interior).any(), "%dx%d k %d tile (%d, %d): band outside the interior" % (W, H, k, tx, ty)
            tiles.append((interior, image, rx0, ry0, w, h))
    assert (owners == 1).all(), "%dx%d k %d: interiors do not partition the image (%d pixels)" % (W, H, k, (owners != 1).sum())
    for interior, image, rx0, ry0, w, h in tiles:
        ring = (image & ~interior)[:h, :w]
        missed = ring & ~in_band[ry0:ry0 + h, rx0:rx0 + w]
        assert not missed.any(), "%dx%d k %d tile at (%d, %d): %d ring pixels are in no band, first at %s" % (
            W, H, k, rx0, ry0, missed.sum(), tuple(np.argwhere(missed)[0]))


def pyramid(w, h):
    out = [(w, h)]
    for _ in range(1, gc.TV_SCALES):
        w, h = round(w * gc.TV_SCALE), round(h * gc.TV_SCALE)
        if w < gc.TV_MIN or h < gc.TV_MIN:
            break
        out.append((w, h))
    return out


SHAPES = sorted(set(gc.TINY + gc.SQUARES + gc.STRIPS + gc.LARGE + gc.TVL1_CUTS + gc.STAGE_SMALL + gc.STAGE_STRIPS
                    + [s for f in ((1920, 1080), (340, 256), (256, 256), (455, 256)) for s in pyramid(*f)]))


@pytest.mark.parametrize("k", range(1, 9))
def test_every_ring_pixel_is_in_its_owners_band(k):
    for w, h in SHAPES:
        check_geometry(w, h, k)


def test_a_band_without_its_corner_misses_ring_pixels():
    """the check above sees a band that leaves out the corner a diagonal neighbour's ring reaches"""
    W, H, k = 400, 200, 8
    hy, hx = k, (k + 3) & ~3
    ntx, nty = tiles_along(W, TW, hx), tiles_along(H, TH, hy)
    interior, band, image, rx0, ry0 = tile_masks(W, H, k, 1, 1, ntx, nty)
    band[:2 * hy, :2 * hx] = False  # top-left corner of the band of an interior tile
    # the diagonal neighbour (0, 0) has cells at (rx0 + hx .. rx0 + 2hx) x (ry0 + hy .. ry0 + 2hy) in its ring
    n_int, _, n_img, nrx0, nry0 = tile_masks(W, H, k, 0, 0, ntx, nty)
    ring = n_img & ~n_int
    ys, xs = np.nonzero(ring)
    gx, gy = xs + nrx0 - rx0, ys + nry0 - ry0
    inside = (gx >= 0) & (gx < TW) & (gy >= 0) & (gy < TH)
    assert inside.any()
    owned = interior[gy[inside], gx[inside]]
    assert (owned & ~band[gy[inside], gx[inside]]).any()
