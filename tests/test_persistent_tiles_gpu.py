"""The line pre-pass (k_lsd_prep in csrc/line.cu) is a persistent tile loop: the grid holds as many CTAs as fit on the device, every CTA
takes tiles from a counter in the handle's workspace, and the next tile's input box is loaded while the current one is computed.  These
tests cover what the plane-by-plane tests of test_line_prep_gpu.py do not: batches whose tiles outnumber the grid many times over, a
grid larger than the work, the counter of one handle used by calls back to back, and two handles (two counters) running at once on
their own streams.  Every frame's pre-pass planes, seed order and lines must equal a fresh handle's single-frame results bit for bit."""
import numpy as np
import pytest

from test_line_prep_gpu import assert_prep

torch = pytest.importorskip("torch")

NL = 40


def _contents(synth, icl, W, H, k):
    """k distinct frames of size W x H: the ICL office frame (tiled / cropped) and synthetic scenes."""
    icl_wh = np.ascontiguousarray(np.tile(icl, (-(-H // 480), -(-W // 640)))[:H, :W])
    return [icl_wh] + [synth.frame(W, H, s) for s in range(k - 1)]


def _single(pkg, img):
    """A fresh handle's single-frame pre-pass planes and lines."""
    H, W = img.shape
    ls = pkg.LineSegment(NL, max_width=W, max_height=H)
    kl, ld, eq = ls.ExtractLineSegment(img)
    out = dict(prep=ls.prep_planes(), kl=kl.tobytes(), ld=ld, eq=eq)
    ls.close()
    return out


def _pinned(shape, dtype):
    """A zeroed numpy array in page-locked host memory, so that the copies of an asynchronous call do not wait for the host."""
    dtype = np.dtype(dtype)
    buf = torch.zeros(int(np.prod(shape)) * dtype.itemsize, dtype=torch.uint8, pin_memory=True)
    return buf.numpy().view(dtype).reshape(shape)


def _batch_out(pkg, B):
    return (_pinned((B, NL), pkg.KEYLINE_DTYPE), _pinned((B, NL, 32), np.uint8), _pinned((B, NL, 3), np.float64), _pinned((B,), np.int32))


def _stack(imgs, order):
    fr = _pinned((len(order),) + imgs[0].shape, np.uint8)
    for i, c in enumerate(order):
        fr[i] = imgs[c]
    return fr


def _assert_batch(tag, ls, out, order, refs):
    """Frame i of the last call of `ls` against refs[order[i]]."""
    kl, ld, eq, n = out
    for i, c in enumerate(order):
        want = refs[c]
        assert_prep(f"{tag} frame {i}", ls.prep_planes(i), want["prep"])
        m = int(n[i])
        assert kl[i, :m].tobytes() == want["kl"], f"{tag} frame {i}: KeyLines differ"
        assert np.array_equal(ld[i, :m], want["ld"]) and np.array_equal(eq[i, :m], want["eq"]), f"{tag} frame {i}: LBD / line equations differ"


@pytest.mark.gpu
def test_tiles_outnumber_the_grid(pkg, synth, icl_gray):
    """513 frames of 640x480: 24624 tiles, about 27 for each of the 924 CTAs of the grid on an H100."""
    W, H, B = 640, 480, 513
    imgs = _contents(synth, icl_gray, W, H, 8)
    refs = [_single(pkg, im) for im in imgs]
    order = [(i * 5) % len(imgs) for i in range(B)]
    frames = _stack(imgs, order)
    ls = pkg.LineSegment(NL, max_width=W, max_height=H, max_batch=B)
    out = ls.extract_batch(frames, _batch_out(pkg, B))
    _assert_batch("513x640x480", ls, out, order, refs)


@pytest.mark.gpu
@pytest.mark.parametrize("W,H,B", [(16, 16, 1), (161, 41, 3)], ids=["16x16x1", "161x41x3"])
def test_grid_exceeds_the_tiles(pkg, synth, icl_gray, W, H, B):
    """One tile (16x16) and 3 x 4 tiles (161x41): most of the grid finds no work and exits."""
    imgs = _contents(synth, icl_gray, W, H, B)
    refs = [_single(pkg, im) for im in imgs]
    ls = pkg.LineSegment(NL, max_width=W, max_height=H, max_batch=B)
    out = ls.extract_batch(_stack(imgs, range(B)), _batch_out(pkg, B))
    _assert_batch(f"{W}x{H}x{B}", ls, out, list(range(B)), refs)


@pytest.mark.gpu
def test_counter_is_reset_between_calls(pkg, synth, icl_gray):
    """Three calls of one handle enqueued back to back with no wait between them; each batch differs from the one before, so a call that
    found the counter used up would leave the previous call's planes in place."""
    W, H = 640, 480
    imgs = _contents(synth, icl_gray, W, H, 6)
    refs = [_single(pkg, im) for im in imgs]
    ls = pkg.LineSegment(NL, max_width=W, max_height=H, max_batch=32)
    orders = [[i % 3 for i in range(32)], [3 + i % 3 for i in range(20)], [(i + 1) % 6 for i in range(7)]]
    batches = [_stack(imgs, o) for o in orders]
    outs = [_batch_out(pkg, len(o)) for o in orders]
    for fr, out in zip(batches, outs):
        ls.extract_batch_begin(fr, out)
    ls.sync()
    _assert_batch("third call", ls, outs[2], orders[2], refs)
    for k in (0, 1):       # the lines of the earlier calls were copied out before the next call overwrote the workspace
        kl, ld, eq, n = outs[k]
        for i, c in enumerate(orders[k]):
            m = int(n[i])
            assert kl[i, :m].tobytes() == refs[c]["kl"] and np.array_equal(ld[i, :m], refs[c]["ld"]), f"call {k} frame {i}: lines differ"
    ls.extract_batch(batches[1], outs[1])
    _assert_batch("second batch again", ls, outs[1], orders[1], refs)


@pytest.mark.gpu
def test_two_handles_on_two_streams(pkg, synth, icl_gray):
    """Two handles, each on its own stream with its own counter, enqueued together so that their pre-passes share the device."""
    W, H, B = 640, 480, 64
    imgs = _contents(synth, icl_gray, W, H, 6)
    refs = [_single(pkg, im) for im in imgs]
    orders = [[i % 3 for i in range(B)], [3 + (i * 2) % 3 for i in range(B)]]
    handles = [pkg.LineSegment(NL, max_width=W, max_height=H, max_batch=B) for _ in orders]
    frames = [_stack(imgs, o) for o in orders]
    outs = [_batch_out(pkg, B) for _ in orders]
    for ls, fr, out in zip(handles, frames, outs):
        ls.extract_batch_begin(fr, out)
    for ls in handles:
        ls.sync()
    for k, (ls, out, o) in enumerate(zip(handles, outs, orders)):
        _assert_batch(f"handle {k}", ls, out, o, refs)
