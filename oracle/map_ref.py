"""ctypes front end of oracle/_ref/libmap_ref.so: the REFERENCE's own fiducial_slam Map (map.cpp + transform_with_variance.cpp compiled
unmodified from the reference checkout against the stand-in headers of oracle/ref_shim; built by oracle/Makefile where that
checkout exists).

TEST INFRASTRUCTURE ONLY -- never imported by the product (fiducials_b200/).  It pins oracle/slam_oracle.py (tests/test_map_ref.py)
and checks the CUDA map update (tests/test_gpu_slam.py) against the reference code itself rather than against a restatement.

Where the library cannot be built, the same calls are answered from a tape (use_tape): what the compiled reference returned,
call by call, recorded under tests/golden/map_ref/ by running the tests with FID_RECORD_MAP_REF=1 where the library exists.
Each recorded call keeps a digest of its inputs, so a tape that no longer matches the test's inputs fails instead of
answering for other inputs."""
import contextlib
import ctypes as C
import os
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libmap_ref.so")
_lib = None
_tape = None


def available() -> bool:
    return os.path.exists(LIB_PATH)


def _flat(x, out):
    if x is None:
        out.append(-1.0)
    elif isinstance(x, dict):
        for k in sorted(x):
            _flat(k, out)
            _flat(x[k], out)
    elif isinstance(x, (str, bytes)):
        b = x.encode() if isinstance(x, str) else x
        out.append(float(sum((i + 1) * c for i, c in enumerate(b))))
    elif isinstance(x, (list, tuple)):
        for v in x:
            _flat(v, out)
    else:
        out.extend(np.asarray(x, np.float64).ravel().tolist())
    return out


def _digest(*args) -> np.ndarray:
    """Checksums of the inputs: three differently weighted sums of the SIGNED values (a flipped sign or swapped entries
    change them), the sum of magnitudes (the scale of the tolerance) and the count."""
    v = np.array(_flat(args, []), np.float64)
    i = np.arange(len(v))
    w = [1.0 + (i % 97) / 97.0, 1.0 + ((7 * i) % 89) / 89.0, np.where(i % 2 == 0, 1.0, -1.0) * (1.0 + (i % 13) / 13.0)]
    return np.array([np.sum(v * wk) for wk in w] + [np.sum(np.abs(v)), len(v)], np.float64)


def _same_inputs(a, b) -> bool:
    """Digests agree up to last-bit differences of the inputs (relative to their magnitude), count exactly."""
    scale = 2.0 * max(1.0, a[3], b[3])
    return a[4] == b[4] and bool(np.all(np.abs(a[:4] - b[:4]) <= 1e-10 * scale))


class _Tape:
    def __init__(self, path, record):
        self.path, self.record, self.pos = path, record, 0
        self.codes, self.digests, self.chunks = [], [], []
        if not record:
            z = np.load(path)
            self.codes, self.digests = z["codes"].tolist(), list(z["digests"])
            offs, data = z["offsets"], z["data"]
            self.chunks = [data[offs[i]:offs[i + 1]] for i in range(len(offs) - 1)]

    def call(self, code, digest, live):
        if self.record:
            v = np.asarray(live(), np.float64).ravel()
            self.codes.append(code)
            self.digests.append(digest)
            self.chunks.append(v)
            return v
        i = self.pos
        self.pos += 1
        assert i < len(self.codes) and self.codes[i] == code, "recorded reference calls out of step at call %d (%s): %s" % (i, code, self.path)
        assert _same_inputs(self.digests[i], digest), "inputs of call %d (%s) differ from the recording %s" % (i, code, self.path)
        return self.chunks[i]

    def save(self):
        os.makedirs(os.path.dirname(self.path), exist_ok=True)
        offs = np.cumsum([0] + [len(c) for c in self.chunks]).astype(np.int64)
        data = np.concatenate(self.chunks) if self.chunks else np.zeros(0)
        np.savez_compressed(self.path, codes=np.array(self.codes, dtype=str), digests=np.array(self.digests, np.float64).reshape(-1, 5), offsets=offs, data=data)


@contextlib.contextmanager
def use_tape(path):
    """Within the block: live calls where libmap_ref.so exists (and recorded to `path` when FID_RECORD_MAP_REF=1), otherwise the
    answers recorded at `path`."""
    global _tape
    if available():
        _tape = _Tape(path, record=True) if os.environ.get("FID_RECORD_MAP_REF") == "1" else None
    else:
        if not os.path.exists(path):
            raise FileNotFoundError("%s: neither oracle/_ref/libmap_ref.so nor recorded answers of it" % path)
        _tape = _Tape(path, record=False)
    try:
        yield
        if _tape is not None and _tape.record:
            _tape.save()
        if _tape is not None and not _tape.record:
            assert _tape.pos == len(_tape.codes), "%d recorded reference calls were not made: %s" % (len(_tape.codes) - _tape.pos, path)
    finally:
        _tape = None


def _call(code, args, live):
    """One call of the compiled reference, as a float64 vector: live, recorded or replayed."""
    if _tape is None:
        return np.asarray(live(), np.float64).ravel()
    return _tape.call(code, _digest(code, *args), live)


def _replaying() -> bool:
    return _tape is not None and not _tape.record


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(LIB_PATH)
        lib.mapref_create.restype = C.c_void_p
        lib.mapref_create.argtypes = [C.c_double, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_char_p, C.c_char_p, C.c_char_p]
        lib.mapref_destroy.argtypes = [C.c_void_p]
        lib.mapref_set_tf.argtypes = [C.c_char_p, C.c_char_p, C.c_void_p]
        lib.mapref_update.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_double, C.c_char_p, C.c_void_p]
        lib.mapref_entries.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        lib.mapref_links.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
        lib.mapref_pose_tf.argtypes = [C.c_void_p, C.c_void_p]
        lib.mapref_add_fiducial.argtypes = [C.c_void_p, C.c_int]
        lib.mapref_clear.argtypes = [C.c_void_p]
        lib.mapref_load_map.argtypes = [C.c_void_p, C.c_char_p]
        lib.mapref_save_map.argtypes = [C.c_void_p, C.c_char_p]
        lib.mapref_state.argtypes = [C.c_void_p, C.c_void_p]
        lib.twvref_apply.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        lib.mapref_replay.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_char_p]
        _lib = lib
    return _lib


def twv_apply(op, a, b=None):
    """The reference's TransformWithVariance, directly.  a, b: x y z qx qy qz qw variance.  op: 'update', 'average', 'mul', 'inverse'."""
    a = np.asarray(a, np.float64)
    b = np.asarray(b if b is not None else a, np.float64)

    def live():
        out = np.zeros(8, np.float64)
        _load().twvref_apply({"update": 0, "average": 1, "mul": 2, "inverse": 3}[op], a.ctypes.data_as(C.c_void_p), b.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        return out

    return _call("twv_" + op, (a, b), live).copy()


CAMERA, BASE, MAP, ODOM = b"camera", b"base_link", b"map", b"odom"


class RefMap:
    """One Map instance of the reference.  tf look-ups are process-global in the stand-in buffer: set_tf before every update."""

    def __init__(self, weighting_scale=1e9, use_area=False, read_only=False, publish_6dof_pose=False, covariance_diagonal=None, odom=False, initial_map_text=None):
        self.h = None
        self.stamp = 100.0
        cov = np.asarray(covariance_diagonal, np.float64) if covariance_diagonal is not None else None
        _call("create", (weighting_scale, use_area, read_only, publish_6dof_pose, cov, odom, initial_map_text), lambda: [])
        if _replaying():
            return
        lib = _load()
        self._dir = tempfile.TemporaryDirectory()
        self.map_file = os.path.join(self._dir.name, "map.txt")
        if initial_map_text is not None:
            with open(self.map_file, "w") as f:
                f.write(initial_map_text)
        lib.mapref_clear_tf()
        self.h = C.c_void_p(lib.mapref_create(float(weighting_scale), int(use_area), int(read_only), int(publish_6dof_pose), cov.ctypes.data_as(C.c_void_p) if cov is not None else None,
                                              self.map_file.encode(), ODOM if odom else b"", BASE))

    def close(self):
        if self.h:
            _load().mapref_destroy(self.h)
            self.h = None
            self._dir.cleanup()

    @staticmethod
    def set_tf(target: bytes, source: bytes, t7):
        """t7 = x y z qx qy qz qw, the answer of lookupTransform(target, source); None removes nothing (clear_tf() resets all)."""
        a = np.asarray(t7, np.float64)
        _load().mapref_set_tf(target, source, a.ctypes.data_as(C.c_void_p))

    @staticmethod
    def clear_tf():
        _load().mapref_clear_tf()

    def update(self, transforms, T_baseCam=None, T_camBase=None, T_mapBase=None, T_odomBase=None):
        """transforms: dicts with fiducial_id, translation, rotation (xyzw), object_error, fiducial_area.  T_*: 7-vectors or None
        (= that tf look-up fails).  Returns (published, t3, q4, covariance diagonal)."""
        self.stamp += 0.05
        out = _call("update", (transforms, T_baseCam, T_camBase, T_mapBase, T_odomBase), lambda: self._update(transforms, T_baseCam, T_camBase, T_mapBase, T_odomBase))
        return bool(out[0]), out[1:4].copy(), out[4:8].copy(), out[8:14].copy()

    def _update(self, transforms, T_baseCam, T_camBase, T_mapBase, T_odomBase):
        self.clear_tf()
        if T_baseCam is not None:
            self.set_tf(BASE, CAMERA, T_baseCam)
        if T_camBase is not None:
            self.set_tf(CAMERA, BASE, T_camBase)
        if T_mapBase is not None:
            self.set_tf(MAP, BASE, T_mapBase)
        if T_odomBase is not None:
            self.set_tf(ODOM, BASE, T_odomBase)
        obs = np.zeros((len(transforms), 10), np.float64)
        for i, t in enumerate(transforms):
            obs[i] = [t["fiducial_id"], *t["translation"], *t["rotation"], t["object_error"], t["fiducial_area"]]
        out = np.zeros(14, np.float64)
        _load().mapref_update(self.h, len(transforms), obs.ctypes.data_as(C.c_void_p), self.stamp, CAMERA, out.ctypes.data_as(C.c_void_p))
        return out

    def replay(self, messages, T_baseCam=None, T_camBase=None):
        """The whole message sequence inside the compiled reference (one call; used for timing).  Returns the number of fiducials."""
        return int(_call("replay", (messages, T_baseCam, T_camBase), lambda: [self._replay(messages, T_baseCam, T_camBase)])[0])

    def _replay(self, messages, T_baseCam, T_camBase):
        self.clear_tf()
        if T_baseCam is not None:
            self.set_tf(BASE, CAMERA, T_baseCam)
        if T_camBase is not None:
            self.set_tf(CAMERA, BASE, T_camBase)
        flat = np.array([[t["fiducial_id"], *t["translation"], *t["rotation"], t["object_error"], t["fiducial_area"]] for msg in messages for t in msg], np.float64).reshape(-1, 10)
        off = np.zeros(len(messages) + 1, np.int32)
        off[1:] = np.cumsum([len(m) for m in messages])
        self._replay_args = (flat, off)
        return _load().mapref_replay(self.h, len(messages), off.ctypes.data_as(C.c_void_p), flat.ctypes.data_as(C.c_void_p), self.stamp, CAMERA)

    def entries(self):
        """rows: id, x, y, z, rx, ry, rz, variance, numObs, n_links (ids ascending)"""
        def live():
            out = np.zeros((4096, 10), np.float64)
            n = _load().mapref_entries(self.h, 4096, out.ctypes.data_as(C.c_void_p))
            return out[:n]

        return _call("entries", (), live).reshape(-1, 10).copy()

    def links(self):
        def live():
            buf = np.zeros((65536, 2), np.int32)
            n = _load().mapref_links(self.h, 65536, buf.ctypes.data_as(C.c_void_p))
            return buf[:n]

        d = {}
        for a, b in _call("links", (), live).reshape(-1, 2):
            d.setdefault(int(a), set()).add(int(b))
        return d

    def pose_tf(self):
        def live():
            out = np.zeros(9, np.float64)
            _load().mapref_pose_tf(self.h, out.ctypes.data_as(C.c_void_p))
            return out

        out = _call("pose_tf", (), live)
        return bool(out[0]), out[1:4].copy(), out[4:8].copy(), bool(out[8])

    def add_fiducial(self, fid):
        _call("add_fiducial", (fid,), lambda: [_load().mapref_add_fiducial(self.h, int(fid))][:0])

    def clear(self):
        _call("clear", (), lambda: [_load().mapref_clear(self.h)][:0])

    def save_map(self, path):
        """Writes the reference's map file to `path` (replayed: the recorded file)."""
        def live():
            ok = bool(_load().mapref_save_map(self.h, path.encode()))
            text = open(path, "rb").read() if ok else b""
            return [float(ok)] + list(text)

        out = _call("save_map", (), live)
        if _replaying() and out[0]:
            with open(path, "wb") as f:
                f.write(bytes(out[1:].astype(np.uint8)))
        return bool(out[0])

    def load_map(self, path):
        return bool(_call("load_map", (open(path).read() if os.path.exists(path) else None,), lambda: [_load().mapref_load_map(self.h, path.encode())])[0])

    def state(self):
        def live():
            s = np.zeros(4, np.int32)
            _load().mapref_state(self.h, s.ctypes.data_as(C.c_void_p))
            return s

        s = _call("state", (), live).astype(np.int64)
        return dict(frameNum=int(s[0]), isInitializingMap=bool(s[1]), originFid=int(s[2]), fiducialToAdd=int(s[3]))
