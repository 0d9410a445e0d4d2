"""ORB extraction from frames already in device memory, through every staging path of the tile kernels: byte loads (base or pitch
not word aligned), TMA boxes (16-byte aligned pitch) and the word-load fallback that reads rows up to the pitch (SSLPL_NO_TMA=1),
with junk in the padding and between frames.  Keypoints, descriptors, pyramid levels and blurred levels must equal the host path's,
and the host path's keypoints and descriptors the oracle's.  Also a handle whose staging buffer holds an earlier, wider frame."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

W, H, B = 640, 480, 3
ORB_ARGS = (1000, 1.2, 8, 20, 7)


class _DevArray:
    """A raw device pointer as a __cuda_array_interface__ object, for torch.as_tensor."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = dict(shape=(nbytes,), typestr="|u1", data=(ptr, False), version=3, strides=None)


def _download(ptr, nbytes, dtype):
    return torch.as_tensor(_DevArray(ptr, nbytes), device="cuda").cpu().numpy().view(dtype)


def _place(frames, offset, pitch, stride, seed):
    """Host image of the device buffer: frame f at offset + f * stride with rows `pitch` bytes apart, random bytes everywhere else."""
    n = offset + stride * (len(frames) - 1) + pitch * (H - 1) + W + 64
    buf = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    for f, img in enumerate(frames):
        np.lib.stride_tricks.as_strided(buf[offset + f * stride:], shape=(H, W), strides=(pitch, 1))[...] = img
    return buf


def _planes(ext, f):
    return [ext.level(l, f) for l in range(ext.nlevels)] + [ext.blurred(l, f) for l in range(ext.nlevels)]


def _make(pkg, monkeypatch, no_tma):
    if no_tma:
        monkeypatch.setenv("SSLPL_NO_TMA", "1")
    ext = pkg.ORBextractor(*ORB_ARGS, max_width=W, max_height=H, max_batch=B)
    monkeypatch.delenv("SSLPL_NO_TMA", raising=False)
    return ext


@pytest.fixture(scope="module")
def host_results(pkg, oracle, synth, icl_gray):
    frames = np.stack([icl_gray, synth.frame(W, H, 3), synth.frame(W, H, 9)])
    ext = pkg.ORBextractor(*ORB_ARGS, max_width=W, max_height=H, max_batch=B)
    kps, desc, n = ext.extract_batch(frames)
    out = []
    for f in range(B):
        okps, odesc = oracle.OrbOracle(*ORB_ARGS).extract(frames[f])
        assert n[f] == len(okps) and kps[f, :n[f]].tobytes() == okps.tobytes() and np.array_equal(desc[f, :n[f]], odesc), f"host frame {f}"
        out.append((kps[f, :n[f]].tobytes(), desc[f, :n[f]].copy(), _planes(ext, f)))
    return frames, out


VIEWS = [  # (name, base offset, pitch, frame stride, SSLPL_NO_TMA)
    ("base +1 (byte loads)", 1, W, W * H, False),
    ("odd pitch (byte loads)", 0, W + 3, (W + 3) * H, False),
    ("pitch 16-aligned, junk padding (TMA)", 0, W + 16, (W + 16) * H, False),
    ("pitch 16-aligned, junk padding, SSLPL_NO_TMA (word loads up to the pitch)", 0, W + 16, (W + 16) * H, True),
    ("pitch 4-aligned, junk padding (word loads up to the pitch)", 0, W + 12, (W + 12) * H, False),
    ("odd frame stride, junk between frames", 0, W + 16, (W + 16) * H + 5, False),
]


@pytest.mark.parametrize("name,offset,pitch,stride,no_tma", VIEWS, ids=[v[0] for v in VIEWS])
def test_device_views_equal_the_host_path(pkg, host_results, monkeypatch, name, offset, pitch, stride, no_tma):
    frames, want = host_results
    ext = _make(pkg, monkeypatch, no_tma)
    buf = torch.from_numpy(_place(frames, offset, pitch, stride, seed=len(name))).cuda()
    ext.extract_batch_device(buf.data_ptr() + offset, B, W, H, pitch, stride)
    ext.sync()
    d_kps, d_desc, d_n, cap = ext.device_results()
    n = _download(d_n, 4 * B, np.int32)
    kps = _download(d_kps, B * cap * pkg.KEYPOINT_DTYPE.itemsize, pkg.KEYPOINT_DTYPE).reshape(B, cap)
    desc = _download(d_desc, B * cap * 32, np.uint8).reshape(B, cap, 32)
    for f in range(B):
        k0, d0, p0 = want[f]
        assert kps[f, :n[f]].tobytes() == k0, f"{name}, frame {f}: keypoints differ ({n[f]} vs {len(d0)})"
        assert np.array_equal(desc[f, :n[f]], d0), f"{name}, frame {f}: descriptors differ"
        for i, (g, w) in enumerate(zip(_planes(ext, f), p0)):
            kind, l = ("level", i) if i < ext.nlevels else ("blurred level", i - ext.nlevels)
            assert np.array_equal(g, w), f"{name}, frame {f}: {kind} {l} differs at {int((g != w).sum())} pixels"
    del buf


def test_staging_buffer_of_a_wider_frame_does_not_leak(pkg, oracle, synth, monkeypatch):
    """Host frames are staged with a 16-byte aligned pitch: 624 for a 613-wide frame, whose columns 613-623 still hold bytes of the
    640-wide frame before it.  The word-load fallback reads rows up to the pitch; the result must still be a fresh handle's."""
    big = synth.frame(W, H, 4)
    crop = np.ascontiguousarray(synth.frame(W, H, 12)[:, :613])
    used = _make(pkg, monkeypatch, True)
    used(big)
    k1, d1 = used(crop)
    fresh = _make(pkg, monkeypatch, True)
    k2, d2 = fresh(crop)
    assert k1.tobytes() == k2.tobytes() and np.array_equal(d1, d2)
    for l in range(used.nlevels):
        assert np.array_equal(used.level(l), fresh.level(l)), l
    ok, od = oracle.OrbOracle(*ORB_ARGS).extract(crop)
    assert k1.tobytes() == ok.tobytes() and np.array_equal(d1, od)
