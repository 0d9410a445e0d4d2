"""LSD region by region: every candidate region the device's walker hands to the NFA kernels, against the oracle's sequential lsd.cpp.

With SSLPL_LINE_TRACE=1 the handle records one row per NFA job (seed, min(n0, 65535), 0, log_nfa, x1, y1, x2, y2, width, p); the oracle
records one per region that reached region2rect.  The oracle runs with cr_trig=True: region2rect then takes cos / sin(theta) from the
host build of the device's correctly-rounded ddtrig.h (test_lsd_numerics_cpu.py proves it against mpmath) instead of glibc, so both
sides build the rectangle with the same rounding and it is compared bit for bit, accepted or rejected.  Unlike the segment-level tests,
this sees regions that end up rejected: their rectangles, rect_improve's choices and their NFA.

The content is chosen to reach what the line tests' frames do not: regions above 65,535 pixels (diagonal ramps at 1920x1080), flat
rectangles (lines within 2 degrees of horizontal: l_rect_count's lane-per-pixel branch), rectangles cut by the frame border, dense noise
(many rejected jobs, p halved again in rect_improve's last phase), the smallest frame sizes, and the solo one-warp walker, which the handle
picks only for batches of at least twice the SM count.  The coverage assertions keep later content changes from hollowing this out."""
import math
import os
from concurrent.futures import ThreadPoolExecutor
import numpy as np
import cv2
import pytest

from test_line_gpu import WALKERS
from test_lsd_numerics_gpu import DV_ABS, DV_REL

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

NL = 40
_POOL = ThreadPoolExecutor(max(4, min(32, os.cpu_count() or 4)))   # the oracle's ctypes calls release the GIL


def _ramp(W, H, deg, slope):
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    a = math.radians(deg)
    return np.clip(np.round(127.5 + slope * ((xx - W / 2) * math.cos(a) + (yy - H / 2) * math.sin(a))), 0, 255).astype(np.uint8)


def _radial(W, H, slope):
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    return (np.floor(slope * np.hypot(xx - 0.3 * W, yy - 0.6 * H)) % 256).astype(np.uint8)


def _lines(W, H, deg, seed):
    """Step edges and 1-3 px lines a fraction of a degree to two degrees from horizontal (or vertical)."""
    rng = np.random.default_rng(seed)
    img = np.full((H, W), 90, np.uint8)
    a = math.radians(deg)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    d = -xx * math.sin(a) + yy * math.cos(a)
    lo, hi = d.min(), d.max()
    img[d > lo + 0.7 * (hi - lo)] = 170
    for c in rng.uniform(lo + 0.05 * (hi - lo), lo + 0.65 * (hi - lo), 12):
        img[np.abs(d - c) < rng.uniform(0.5, 1.5)] = int(rng.integers(0, 256))
    return img


def _border_rects(W, H, seed):
    """Rotated filled rectangles that cross the frame border."""
    rng = np.random.default_rng(seed)
    img = np.full((H, W), 40, np.uint8)
    for _ in range(12):
        c = (float(rng.choice([rng.uniform(-40, 40), rng.uniform(W - 40, W + 40)])), float(rng.uniform(-40, H + 40)))
        box = cv2.boxPoints((c, (float(rng.uniform(60, 400)), float(rng.uniform(8, 120))), float(rng.uniform(0, 180))))
        cv2.fillPoly(img, [np.round(box).astype(np.int32)], int(rng.integers(100, 256)))
    return img


def contents(synth, icl):
    """(tag, image) of every frame compared through single-frame calls."""
    rng = np.random.default_rng(11)
    out = [("icl", icl)] + [(f"syn640/{f}", synth.frame(640, 480, f)) for f in range(32)]
    out += [("noise", rng.integers(0, 256, (480, 640)).astype(np.uint8)),
            ("low-contrast noise", rng.integers(120, 137, (480, 640)).astype(np.uint8)),
            ("low-contrast noise 2", (128 + np.round(rng.normal(0, 3.5, (480, 640)))).clip(0, 255).astype(np.uint8))]
    out += [(f"ramp {d} deg", _ramp(1920, 1080, d, 5.0)) for d in (0, 30, 45, 90, 179, 60.6, 119.4)]
    out += [("radial", _radial(1920, 1080, 5.0))]
    out += [(f"lines {d} deg", _lines(640, 480, d, i)) for i, d in enumerate((0.1, 0.5, 1.0, 2.0, 90.3, 91.5))]
    out += [(f"border rects {s}", _border_rects(640, 480, s)) for s in range(3)]
    out += [(f"syn{w}x{h}", synth.frame(w, h, 5)) for (w, h) in ((16, 16), (17, 23), (333, 251), (1280, 960), (1920, 1080))]
    return out


def oracle_trace(oracle, img):
    lo = oracle.LineOracle(NL, cr_trig=True)
    lo.extract(img)
    return lo.trace()


def flat(rows):
    """Rows whose rectangle spans fewer than 16 scan lines (l_rect_count then spreads each row's pixels over the lanes)."""
    x1, y1, x2, y2, w = rows[:, 4], rows[:, 5], rows[:, 6], rows[:, 7], rows[:, 8]
    L = np.maximum(np.hypot(x2 - x1, y2 - y1), 1e-12)
    ext = np.abs(y2 - y1) + w * np.abs(x2 - x1) / L
    return ext < 15


def compare(tag, dev, orc):
    """Device trace rows against the oracle's, minus its refine-failure rows (the device emits rows only for jobs).  Returns the
    compared oracle rows."""
    orc = orc[orc[:, 3] != -1e9]
    assert len(dev) == len(orc), f"{tag}: {len(dev)} jobs on the device, {len(orc)} regions in the oracle"
    bad = []
    for i in range(len(dev)):
        d, o = dev[i], orc[i]
        why = []
        if d[0] != o[0] or d[1] != min(o[1], 65535.0):
            why.append("seed / n0")
        # column 2 (the size after refine) is always 0 on the device: not compared
        if (d[3] > 0) != (o[3] > 0):
            why.append("accept / reject")
        if d[4:].tobytes() != o[4:].tobytes():
            why.append("rectangle / p")
        if not abs(d[3] - o[3]) <= DV_ABS + DV_REL * abs(o[3]):
            why.append("log_nfa")
        if why:
            bad.append(f"  row {i} seed {int(o[0])} ({', '.join(why)})\n    device {d.tolist()}\n    oracle {o.tolist()}")
    assert not bad, f"{tag}: {len(bad)} of {len(dev)} rows differ\n" + "\n".join(bad[:10])
    return orc


class Coverage:
    def __init__(self):
        self.big = self.flat = self.rejected = self.halved6 = self.rows = 0

    def add(self, rows):
        self.rows += len(rows)
        self.big += int((rows[:, 1] >= 65535).sum())
        self.flat += int(flat(rows).sum())
        self.rejected += int((rows[:, 3] <= 0).sum())
        self.halved6 += int((rows[:, 9] <= 0.125 / 64).sum())


def _trace_env(monkeypatch, env=None):
    monkeypatch.delenv("SSLPL_WALKER_WARPS", raising=False)
    monkeypatch.setenv("SSLPL_LINE_TRACE", "1")
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)


def test_single_frames_region_by_region(pkg, oracle, synth, icl_gray, monkeypatch):
    _trace_env(monkeypatch)
    frames = contents(synth, icl_gray)
    oracle_trace(oracle, frames[0][1])                    # first call in this thread (the oracle's LBD tables initialise once)
    futs = [_POOL.submit(oracle_trace, oracle, img) for _, img in frames]
    ls = pkg.LineSegment(NL, max_width=1920, max_height=1080)
    cov = Coverage()
    for (tag, img), fut in zip(frames, futs):
        ls.ExtractLineSegment(img)
        rows = compare(tag, ls.debug_trace(), fut.result())
        cov.add(rows)
    print(f"\n{len(frames)} frames, {cov.rows} regions: {cov.big} of >= 65535 pixels, {cov.flat} flat, {cov.rejected} rejected, "
          f"{cov.halved6} with p halved 6+ times")
    assert cov.big >= 1 and cov.flat >= 1 and cov.rejected >= 100 and cov.halved6 >= 1, vars(cov)


@pytest.mark.parametrize("name,env", WALKERS, ids=[w[0] for w in WALKERS])
def test_every_walker_region_by_region(pkg, oracle, synth, icl_gray, monkeypatch, name, env):
    """Each region-walker form and warp count, forced, on a subset: the multi-warp walker is timing dependent, so two runs each."""
    _trace_env(monkeypatch, env)
    rng = np.random.default_rng(5)
    frames = [("icl", icl_gray), ("syn640/3", synth.frame(640, 480, 3)), ("lines 0.5 deg", _lines(640, 480, 0.5, 1)),
              ("low-contrast noise", rng.integers(120, 137, (480, 640)).astype(np.uint8)), ("border rects", _border_rects(640, 480, 7))]
    futs = [_POOL.submit(oracle_trace, oracle, img) for _, img in frames]
    ls = pkg.LineSegment(NL, max_width=640, max_height=480)
    for (tag, img), fut in zip(frames, futs):
        want = fut.result()
        for rep in range(1 if name.startswith("one warp") else 2):
            ls.ExtractLineSegment(img)
            compare(f"{name}/{tag}/run {rep}", ls.debug_trace(), want)


def test_solo_walker_batch_region_by_region(pkg, oracle, synth, icl_gray, monkeypatch):
    """2 * SM count + 1 frames of 320x240 in one call: the handle picks the one-warp walker by itself.  Device-resident frames, then
    the same frames from host memory through extract_batch."""
    _trace_env(monkeypatch)
    B = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    W, H = 320, 240
    rng = np.random.default_rng(9)
    imgs = [cv2.resize(icl_gray, (W, H), interpolation=cv2.INTER_AREA)] + [synth.frame(W, H, s) for s in range(B - 3)]
    imgs += [rng.integers(0, 256, (H, W)).astype(np.uint8), _lines(W, H, 1.0, 2)]
    futs = [_POOL.submit(oracle_trace, oracle, img) for img in imgs]
    frames = np.stack(imgs)
    ls = pkg.LineSegment(NL, max_width=W, max_height=H, max_batch=B)
    d = torch.from_numpy(frames).cuda()
    ls.extract_batch_device(d.data_ptr(), B, W, H, W, W * H)
    ls.sync()
    dev = [ls.debug_trace(f) for f in range(B)]
    ls.extract_batch(frames)
    host = [ls.debug_trace(f) for f in range(B)]
    for f in range(B):
        want = futs[f].result()
        compare(f"device batch frame {f}", dev[f], want)
        compare(f"host batch frame {f}", host[f], want)
