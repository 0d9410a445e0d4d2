"""The reference's answers to the calls of tests/test_ref_parity_cpu.py, frozen into tests/golden/ref_parity.npz so that the
comparison with the reference runs where the reference cannot be built (its sources are not part of this repository).

`Recorder` wraps oracle/ref.py (the reference compiled by oracle/ref_build.sh) and keeps every answer; `Replay` serves the
same answers from the file.  A call is identified by the function's name and a digest of its arguments, so a changed input
is a missing answer, never a wrong one.  Arrays larger than BIG bytes (keypoints and descriptors of whole frames, pyramid levels)
are kept as a `Digest` — dtype, shape and SHA-1 — which the tests compare with `same`.  tools/make_ref_golden.py records the file
by running the test module."""
import hashlib
import os
import pickle
import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_parity.npz")
BIG = 24 * 1024


class Digest:
    """A large array of a frozen answer: its dtype, shape and the SHA-1 of its bytes."""

    def __init__(self, a):
        a = np.ascontiguousarray(a)
        self.dtype, self.shape, self.sha1 = a.dtype.str, a.shape, hashlib.sha1(a.tobytes()).hexdigest()

    def __len__(self):
        return self.shape[0]

    def matches(self, b):
        b = np.ascontiguousarray(b)
        return b.dtype.str == self.dtype and b.shape == self.shape and hashlib.sha1(b.tobytes()).hexdigest() == self.sha1


def same(a, b):
    """a (an answer of the reference, live or frozen) holds exactly the elements of b."""
    if isinstance(a, Digest):
        return a.matches(b)
    return len(a) == len(b) and a.dtype == b.dtype and a.tobytes() == np.ascontiguousarray(b).tobytes()


def _freeze(v):
    if isinstance(v, np.ndarray) and v.nbytes > BIG:
        return Digest(v)
    if isinstance(v, tuple):
        return tuple(_freeze(x) for x in v)
    if isinstance(v, dict):
        return {k: _freeze(x) for k, x in v.items()}
    return v


def _feed(h, a):
    if isinstance(a, np.ndarray):
        a = np.ascontiguousarray(a)
        h.update(f"nd{a.dtype.str}{a.shape}".encode()); h.update(a.tobytes())
    elif isinstance(a, dict):
        h.update(b"dict")
        for k in sorted(a):
            h.update(str(k).encode()); _feed(h, a[k])
    elif isinstance(a, (list, tuple)):
        h.update(f"seq{len(a)}".encode())
        for x in a:
            _feed(h, x)
    elif isinstance(a, (bool, np.bool_)):
        h.update(b"T" if a else b"F")
    elif isinstance(a, (int, np.integer)):
        h.update(f"i{int(a)}".encode())
    elif isinstance(a, (float, np.floating)):
        h.update(f"f{float(a)!r}".encode())
    elif a is None or isinstance(a, str):
        h.update(repr(a).encode())
    else:
        raise TypeError(f"cannot digest {type(a)}")


def key(name, args, kwargs):
    h = hashlib.sha1(name.encode())
    _feed(h, list(args)); _feed(h, kwargs)
    return f"{name}:{h.hexdigest()[:20]}"


def _vocab_id(path):
    return hashlib.sha1(open(path, "rb").read()).hexdigest()[:20]


class _Calls:
    CAM640 = np.array([500, 500, 320, 240, 0, 640, 0, 480], np.float32)

    @staticmethod
    def cam(fx, fy, cx, cy, minx, maxx, miny, maxy):
        return np.array([fx, fy, cx, cy, minx, maxx, miny, maxy], np.float32)

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)
        return lambda *a, **kw: self._answer(name, a, kw)

    def Vocabulary(self, path):
        calls = self

        class Voc:
            vid = _vocab_id(path)

            def __len__(self):
                return calls._answer("Vocabulary.__len__", (self.vid,), {}, lambda: len(self.live))

            def transform(self, desc, levelsup=4):
                return calls._answer("Vocabulary.transform", (self.vid, desc, levelsup), {}, lambda: self.live.transform(desc, levelsup))

            def words(self, desc):
                return calls._answer("Vocabulary.words", (self.vid, desc), {}, lambda: self.live.words(desc))
        v = Voc()
        if isinstance(self, Recorder):
            v.live = self.R.Vocabulary(path)
        return v


class Recorder(_Calls):
    def __init__(self, R):
        self.R = R; self.answers = {}

    def _answer(self, name, a, kw, live=None):
        k = key(name, a, kw)                            # before the call: the key is what a replay sees
        out = live() if live else getattr(self.R, name)(*a, **kw)
        self.answers[k] = out
        return out

    def save(self, path=PATH):
        blob = pickle.dumps({k: _freeze(v) for k, v in self.answers.items()}, protocol=4)
        np.savez_compressed(path, answers=np.frombuffer(blob, np.uint8))


class Replay(_Calls):
    def __init__(self, path=PATH):
        self.answers = pickle.loads(np.load(path)["answers"].tobytes())

    def _answer(self, name, a, kw, live=None):
        k = key(name, a, kw)
        assert k in self.answers, f"no frozen reference answer for {name} with these arguments (tools/make_ref_golden.py records them)"
        return self.answers[k]
