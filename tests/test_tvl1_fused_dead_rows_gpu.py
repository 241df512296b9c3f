"""The chunk loop of the fused TV-L1 kernel at the visit lengths kk = 4, 6 and 7, which the stage pins of
test_tvl1_fused_stages_gpu.py do not run.

A warp of a tile visit skips the arithmetic of iteration `it` when its whole 4-row block lies outside the rows that can still
reach a kept pixel ([it+1, TH-it) for the primal step, counted from a region edge that is halo): warp 0 from iteration 3,
warp 1 from 7, warp 15 from 4.  kk = 8 meets those iterations in the middle of a visit; kk = 4, 6 and 7 also end visits on
them, so the last iteration of a visit (the error-summing one of a checking chunk) finds a dead warp at the top after 0, 2
and 3 earlier dead iterations (kk = 4, 6, 7) and at the bottom after 1 and 2 (kk = 6, 7), in interior, edge and
single-tile-row tiles.  The checks are the stage pins' own: the strict build equals the oracle bit for bit, the default build equals the stand-alone kernels bit for
bit, under every launch configuration (with and without TMA, neighbour-warp flags or CTA barriers)."""
import itertools

import pytest

from test_tvl1_fused_stages_gpu import CONFIGS, SINGLE_TILE, VARIANTS, edge_heights, edge_widths, level_shapes, run_chunks

pytestmark = pytest.mark.gpu
KS = [4, 6, 7]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kk", KS)
def test_chunks_every_level_at_more_visit_lengths(oracle, variant, kk):
    """two chunks at every level of the frame shapes (several tile rows: interior tiles with halo on both sides)"""
    for j, (w, h) in enumerate(level_shapes()):
        run_chunks(oracle, variant, w, h, kk, 2, CONFIGS[(5 * j + kk) % len(CONFIGS)], 300 * kk + j)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("kk", KS)
def test_chunks_tile_edges_at_more_visit_lengths(oracle, variant, kk):
    """every jlast and rbot, one to three tiles per row and column"""
    ws, hs = edge_widths(kk), edge_heights(kk)
    shapes = list(zip(ws, itertools.cycle(hs))) + list(zip(itertools.cycle(ws[::5]), hs))
    for j, (w, h) in enumerate(shapes):
        run_chunks(oracle, variant, w, h, kk, 1 + j % 3, CONFIGS[(7 * j + kk) % len(CONFIGS)], 1000 * kk + j)


@pytest.mark.parametrize("variant", VARIANTS)
def test_chunks_single_tile_at_more_visit_lengths(oracle, variant):
    for j, (w, h) in enumerate(SINGLE_TILE):
        for kk in KS:
            if 2 * kk < h:
                run_chunks(oracle, variant, w, h, kk, 2, CONFIGS[(3 * j + kk) % len(CONFIGS)], 50 * j + kk)
