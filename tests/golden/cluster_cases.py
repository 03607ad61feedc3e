"""Masks of the cluster-selection golden cases (tests/golden/interactive_cluster_cases.json), rebuilt from their parameters."""
import numpy as np

CASES = [
    {"name": "one_pixel", "hw": (96, 128), "seed": 1},
    {"name": "two_pixels_no_cluster", "hw": (96, 128), "seed": 2},
    {"name": "three_pixels", "hw": (96, 128), "seed": 3},
    {"name": "sparse_no_core_point", "hw": (96, 128), "seed": 4},
    {"name": "largest_below_180", "hw": (480, 854), "seed": 5},
    {"name": "tied_largest", "hw": (480, 854), "seed": 6},
    {"name": "blobs_480x854", "hw": (480, 854), "seed": 7},
    {"name": "large_mask_480x854", "hw": (480, 854), "seed": 8},
]


def _ellipse(h, w, cy, cx, ry, rx):
    yy, xx = np.mgrid[:h, :w]
    return ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0


def make_mask(case) -> np.ndarray:
    h, w = case["hw"]
    m = np.zeros((h, w), bool)
    name = case["name"]
    if name == "one_pixel":
        m[40, 50] = True
    elif name == "two_pixels_no_cluster":
        m[10, 10] = m[60, 100] = True
    elif name == "three_pixels":
        m[10, 10] = m[11, 10] = m[60, 100] = True
    elif name == "sparse_no_core_point":
        m[::9, ::9] = True
    elif name == "largest_below_180":      # one cluster (every pixel is core at the 480x854 eps) of < 180 pixels
        m |= _ellipse(h, w, 200, 300, 6, 6)
    elif name == "tied_largest":           # two congruent clusters, < 18 000 pixels in all: both kept whole, equal counts
        m |= _ellipse(h, w, 120, 200, 30, 30)
        m |= np.roll(m, (200, 400), axis=(0, 1))
    elif name == "blobs_480x854":
        m |= _ellipse(h, w, 100, 150, 40, 60) | _ellipse(h, w, 300, 600, 80, 120) | _ellipse(h, w, 420, 100, 10, 10)
    elif name == "large_mask_480x854":
        m |= _ellipse(h, w, 240, 427, 200, 400)
        m[::7, ::5] = False
    return m
