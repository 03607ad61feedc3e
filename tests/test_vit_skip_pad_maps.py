"""CPU check of the index arithmetic behind the padding-window skip (csrc/vit_pipeline.cu): the three device
map kernels are mirrored here formula by formula and checked for the properties the pipeline relies on (partition of the token
grid, windows closed under the live set, constant tokens = tokens whose whole window is zero padding)."""
import math

import pytest


def cdiv(a, b):
    return (a + b - 1) // b


def geometry(Hr, Wr, P=16, G=64, ws=14):
    nW = cdiv(G, ws)
    lwy, lwx = min(nW, cdiv(cdiv(Hr, P), ws)), min(nW, cdiv(cdiv(Wr, P), ws))
    rows_live, cols_live = min(G, lwy * ws), min(G, lwx * ws)
    return nW, lwy, lwx, rows_live, cols_live


def live_window_map(B, G, ws, lwy, lwx):                      # live_window_map_kernel
    L, out = ws * ws, []
    for r in range(B * lwy * lwx * L):
        t, wb = r % L, r // L
        w, b = wb % (lwy * lwx), wb // (lwy * lwx)
        y, x = (w // lwx) * ws + t // ws, (w % lwx) * ws + t % ws
        out.append(b * G * G + y * G + x if (y < G and x < G) else -1)
    return out


def live_token_map(B, G, rows_live, cols_live):               # live_token_map_kernel
    per = rows_live * cols_live
    return [(r // per) * G * G + ((r % per) // cols_live) * G + (r % per) % cols_live for r in range(B * per)]


def const_token_map(G, rows_live, cols_live):                 # const_token_map_kernel
    n_const = G * G - rows_live * cols_live
    out = [None] * n_const
    per_live_row = G - cols_live
    for tok in range(G * G):
        y, x = tok // G, tok % G
        if y < rows_live and x < cols_live:
            continue
        idx = y * per_live_row + (x - cols_live) if y < rows_live else rows_live * per_live_row + (y - rows_live) * G + x
        assert out[idx] is None
        out[idx] = tok
    return out


@pytest.mark.parametrize("Hr,Wr", [(576, 1024), (1024, 576), (768, 1024), (1024, 1024), (160, 1024), (1024, 225)])
def test_maps_partition_the_grid_and_respect_windows(Hr, Wr):
    P, G, ws, B = 16, 64, 14, 2
    nW, lwy, lwx, rows_live, cols_live = geometry(Hr, Wr)
    GG = G * G
    ry, rx = cdiv(Hr, P), cdiv(Wr, P)                        # token rows / columns that contain image pixels
    tmap = live_token_map(B, G, rows_live, cols_live)
    cmap = const_token_map(G, rows_live, cols_live)
    wmap = live_window_map(B, G, ws, lwy, lwx)
    # 1. live + constant tokens partition every frame's grid
    for b in range(B):
        live_b = {t - b * GG for t in tmap if b * GG <= t < (b + 1) * GG}
        assert len(live_b) == rows_live * cols_live
        assert live_b | set(cmap) == set(range(GG)) and not (live_b & set(cmap))
    assert None not in cmap and len(set(cmap)) == len(cmap)
    # 2. the live windows cover exactly the live tokens, each once
    covered = [t for t in wmap if t >= 0]
    assert sorted(covered) == sorted(tmap)
    # 3. a constant token never shares a window with an image token, and every image token is live
    for tok in cmap:
        y, x = tok // G, tok % G
        wy, wx = y // ws, x // ws
        assert wy * ws >= ry or wx * ws >= rx                 # its whole window starts beyond the image
    for y in range(min(ry, G)):
        for x in range(min(rx, G)):
            assert y < rows_live and x < cols_live
    # 4. sizes used for the compacted GEMMs
    assert len(wmap) == B * lwy * lwx * ws * ws and len(tmap) == B * rows_live * cols_live
    if (Hr, Wr) == (576, 1024):                               # the C2 frame: 10 of 25 windows and 1408 of 4096 tokens are constant
        assert (lwy, lwx) == (3, 5) and len(cmap) == 1408


def test_square_input_has_nothing_to_skip():
    nW, lwy, lwx, rows_live, cols_live = geometry(1024, 1024)
    assert (lwy, lwx) == (nW, nW) and rows_live * cols_live == 64 * 64
