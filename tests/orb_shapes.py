"""Frame shapes, extractor parameters and contents for the ORB sweep (test_orb_shapes_cpu.py, test_orb_shapes_gpu.py), and a
restatement of the extractor's per-level geometry (ORBextractor.cc:776-789 cells, :542 nIni) with the bound on how many keypoints
DistributeOctTree keeps on a level.

The bound: DistributeOctTree splits every one of its nIni root nodes once before it looks at the level's budget N, so after that
first pass the level may hold up to 4 * nIni nodes.  A later pass only runs while the level holds fewer than N nodes: a whole pass
runs only when it cannot overshoot N, and the careful pass (ORBextractor.cc:673-735) stops at the first division that reaches N,
which adds at most 3.  So a level keeps at most max(N + 2, 4 * nIni) keypoints, and none where it has no 30-px cell."""
import math
import os
from collections import namedtuple

import numpy as np

EDGE = 19                        # EDGE_THRESHOLD, ORBextractor.cc:74
MINB = EDGE - 3                  # minBorderX / minBorderY, :775

Case = namedtuple("Case", "id W H kind nf sf nl ini mn")

# the frames the first sweep found past the device's per-level capacities (wide strips, or small budgets)
STRIPS = [
    Case("4000x200-noise", 4000, 200, "noise", 1000, 1.2, 8, 20, 7),
    Case("4095x120-noise", 4095, 120, "noise", 1000, 1.2, 8, 20, 7),
    Case("4000x300-noise-500", 4000, 300, "noise", 500, 1.2, 8, 20, 7),
    Case("1920x240-noise-300", 1920, 240, "noise", 300, 1.2, 8, 20, 7),
    Case("1921x240-noise-300", 1921, 240, "noise", 300, 1.2, 8, 20, 7),
    Case("4095x160-noise-sf1.1", 4095, 160, "noise", 1000, 1.1, 8, 20, 7),
    Case("4095x200-synth-300", 4095, 200, "synth", 300, 1.2, 8, 20, 7),
    Case("4095x480-noise-100", 4095, 480, "noise", 100, 1.2, 8, 20, 7),
    Case("1280x62-noise-8x1", 1280, 62, "noise", 8, 1.2, 1, 20, 7),
    Case("1280x62-pairs-8x1", 1280, 62, "pairs", 8, 1.2, 1, 20, 7),
    # level 0: N = 2 and nIni = 42, so the first split alone needs 42 roots + up to 168 children in the node pool
    Case("1280x62-noise-8x8", 1280, 62, "noise", 8, 1.2, 8, 20, 7),
    Case("1280x62-pairs-8x8", 1280, 62, "pairs", 8, 1.2, 8, 20, 7),
]

# nIni = round(dx / dy) is 0 on every level: no keypoints at all (the reference indexes an empty vector there)
PORTRAIT = [
    Case("300x700-noise", 300, 700, "noise", 1000, 1.2, 8, 20, 7),
    Case("200x4000-noise", 200, 4000, "noise", 1000, 1.2, 8, 20, 7),
]

# 38 px: no cell; 62 px: one cell; 61/62/63, 95/96/97 and 127/128/129 straddle the 30-px cells and the 64x32 blur tiles
# at 2 levels every level stays wider than 32 px and the reference is defined; at 8 the top levels shrink to a few pixels
SMALL = [Case("38x38-noise", 38, 38, "noise", 1000, 1.2, 1, 20, 7),
         Case("38x38-noise-8l", 38, 38, "noise", 1000, 1.2, 8, 20, 7),
         Case("62x62-noise", 62, 62, "noise", 1000, 1.2, 2, 20, 7),
         Case("62x62-noise-8l", 62, 62, "noise", 1000, 1.2, 8, 20, 7)] + [
    Case(f"{w}x{h}-{kind}-{nl}l", w, h, kind, 500, 1.2, nl, 20, 7)
    for nl in (2, 8)
    for (w, h), kind in zip([(61, 127), (62, 128), (63, 129), (95, 97), (96, 96), (97, 95), (127, 61), (128, 62), (129, 63)],
                            ["noise", "binary", "synth"] * 3)]

PARAMS = [
    Case("640x480-nf1", 640, 480, "noise", 1, 1.2, 8, 20, 7),
    Case("640x480-nf8", 640, 480, "synth", 8, 1.2, 8, 20, 7),
    Case("640x480-nf50", 640, 480, "icl", 50, 1.2, 8, 20, 7),
    Case("640x480-1level", 640, 480, "icl", 1000, 1.2, 1, 20, 7),
    Case("640x480-16levels-sf1.1", 640, 480, "synth", 1000, 1.1, 16, 20, 7),
    Case("1280x960-16levels", 1280, 960, "noise", 2000, 1.2, 16, 20, 7),
    Case("640x480-sf1.05", 640, 480, "icl", 1000, 1.05, 8, 20, 7),
    Case("1280x960-sf1.5", 1280, 960, "synth", 1000, 1.5, 8, 20, 7),
    Case("1280x960-sf2.0", 1280, 960, "icl", 1000, 2.0, 5, 20, 7),
    # FAST thresholds (iniThFAST, minThFAST): the saturating byte compares of k_fast's phases A and B1 at their ends
    Case("640x480-th20-20", 640, 480, "noise", 1000, 1.2, 8, 20, 20),
    Case("640x480-th1-1", 640, 480, "low0", 1000, 1.2, 8, 1, 1),
    Case("640x480-th1-1-high", 640, 480, "high255", 1000, 1.2, 8, 1, 1),
    Case("640x480-th254-7", 640, 480, "binary", 1000, 1.2, 8, 254, 7),
    Case("640x480-th254-254", 640, 480, "binary", 1000, 1.2, 8, 254, 254),
]

CONTENT = [
    Case("640x480-binary", 640, 480, "binary", 1000, 1.2, 8, 20, 7),
    Case("640x480-low0", 640, 480, "low0", 1000, 1.2, 8, 20, 7),
    Case("640x480-high255", 640, 480, "high255", 1000, 1.2, 8, 20, 7),
    Case("1500x600-icl-tiled", 1500, 600, "icl", 1000, 1.2, 8, 20, 7),
    # close corner pairs: nodes split into a single child for many passes (the node pool's hardest case)
    Case("640x480-pairs-4000x1", 640, 480, "pairs", 4000, 1.2, 1, 20, 7),
    Case("640x480-pairs-300", 640, 480, "pairs", 300, 1.2, 8, 20, 7),
    Case("4095x240-pairs-1000", 4095, 240, "pairs", 1000, 1.2, 8, 20, 7),
]

GRID = STRIPS + PORTRAIT + SMALL + PARAMS + CONTENT


def _icl():
    import cv2
    img = cv2.imread(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "icl_office_gray.png"), cv2.IMREAD_GRAYSCALE)
    assert img is not None
    return img


def corner_pairs(W, H, seed):
    """Isolated bright pixels on a dark ground, in pairs 2 or 3 px apart (along x, y or a diagonal): every pixel is a FAST corner
    that survives NMS, and the octree needs many halvings of a node to part the two."""
    rng = np.random.default_rng(seed)
    img = np.full((H, W), 40, np.uint8)
    step = 11
    for y in range(MINB + 5, H - MINB - 8, step):
        for x in range(MINB + 5, W - MINB - 8, step):
            jx, jy = (int(v) for v in rng.integers(0, 4, 2))
            d = [(2, 0), (3, 0), (0, 2), (0, 3), (2, 2), (3, 3)][int(rng.integers(0, 6))]
            img[y + jy, x + jx] = 230
            img[y + jy + d[1], x + jx + d[0]] = int(rng.integers(200, 256))
    return img


def frame(kind, W, H, seed=0):
    rng = np.random.default_rng(1000 + 7 * seed + W * 31 + H)
    if kind == "noise":
        return rng.integers(0, 256, (H, W), dtype=np.uint8)
    if kind == "binary":
        return (rng.integers(0, 2, (H, W)) * 255).astype(np.uint8)
    if kind == "low0":                                   # low contrast at the bottom of the range: v - th saturates at 0
        return rng.integers(0, 12, (H, W), dtype=np.uint8)
    if kind == "high255":                                # and at the top: v + th saturates at 255
        return (255 - rng.integers(0, 12, (H, W))).astype(np.uint8)
    if kind == "icl":
        icl = _icl()
        return np.ascontiguousarray(np.tile(icl, (-(-H // icl.shape[0]), -(-W // icl.shape[1])))[:H, :W])
    if kind == "synth":
        import synth
        return synth.frame(W, H, seed)
    if kind == "pairs":
        return corner_pairs(W, H, seed)
    raise ValueError(kind)


def _round_half_away(q):
    return int(math.floor(float(q) + 0.5))              # roundf of a positive float: |q| < 2^12, so q + 0.5 is exact in double


def levels(tables, W, H):
    """Per-level geometry of a W x H frame from the extractor's tables (invscale, nfeat): size, cells, nIni and the keypoint bound."""
    out = []
    for l, (inv, N) in enumerate(zip(tables["invscale"], tables["nfeat"])):
        w = int(np.rint(np.float32(W) * np.float32(inv))); h = int(np.rint(np.float32(H) * np.float32(inv)))   # cvRound, :1111-1112
        dx, dy = w - 2 * MINB, h - 2 * MINB          # maxBorderX - minBorderX, :777-787
        cells = int(np.float32(dx) / np.float32(30)) > 0 and int(np.float32(dy) / np.float32(30)) > 0 and dx > 0 and dy > 0
        nIni = _round_half_away(np.float32(dx) / np.float32(dy)) if cells else 0
        out.append(dict(l=l, w=w, h=h, dx=dx, dy=dy, cells=cells, nIni=nIni, N=int(N),
                        bound=max(int(N) + 2, 4 * nIni) if cells else 0))
    return out


def reference_defined(lv):
    """Where the reference's ORBextractor has a defined result (confirmed by running it on the shapes on either side):
    - every level must be wider and taller than 2 * minBorder = 32 px: at dy <= 0 or dx < 0, nIni = round(dx / dy) is not a
      usable size and vpIniNodes.resize(nIni) throws std::length_error (640x480 at 16 levels, 1280x64 at 8 levels);
    - every level with cells needs nIni >= 1: at dx / dy < 0.5 it indexes the empty vpIniNodes (300x700, 200x4000)."""
    return all(v["w"] > 2 * MINB and v["h"] > 2 * MINB for v in lv) and all(v["nIni"] >= 1 for v in lv if v["cells"])
