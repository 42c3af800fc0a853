"""Localization against the map (fid_map_localize): the host build of map_localize.cuh (tests/hostsim/map_localize_hostsim.cpp,
compiled with g++ into a temporary directory once per session), the cv2 / numpy oracle of every step map_localize.cuh states, and
scene helpers over tests/map_ba_cases.make_scene shared by the tests and tools/bench_map_localize.py."""
import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import map_ba_cases as mc
from fiducials_b200 import _lib

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None
_vp = C.c_void_p
LOC_DTYPE = np.dtype(_lib.fid_localization)


def _p(a):
    return a.ctypes.data_as(_vp)


def harness():
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_map_localize_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_map_localize_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "map_localize_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_map_localize.argtypes = [C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, C.c_double, C.c_int, _vp, _vp, C.c_double] + [_vp] * 4
    return _harness


def entry_variances(sc):
    """The variances of the scene's map entries: 0 for the fixed ones, as mc.file_entries writes them otherwise."""
    return np.array([0.0 if sc["fixed"][k] else 0.01 * (1 + k % 3) for k in range(len(sc["ids"]))])


def on_map(sc, which):
    """sc localized against `which` map: "true" (the markers' real poses) or "fold" (the perturbed start map)."""
    out = dict(sc)
    if which == "true":
        out["start_R"], out["start_t"] = sc["R"].copy(), sc["t"].copy()
    out["var"] = entry_variances(sc)
    return out


def hs_localize(sc, max_entry_variance=-1.0, cam_base=None):
    """The host build over the scene's map (start_R, start_t, var): (records [F], p0 [F][6], used [F][m])."""
    n = len(sc["ids"])
    poses = np.ascontiguousarray(np.concatenate([np.asarray(sc["start_R"]).reshape(n, 9), np.asarray(sc["start_t"]).reshape(n, 3)], 1), np.float64)
    var = np.ascontiguousarray(sc.get("var", entry_variances(sc)), np.float64)
    ids = np.ascontiguousarray(sc["ids"], np.int32)
    counts = np.ascontiguousarray(sc["counts"], np.int32)
    fids = np.ascontiguousarray(sc["fids"], np.int32)
    cr = np.ascontiguousarray(sc["corners"], np.float32)
    K, D = np.ascontiguousarray(sc["K"], np.float64), np.ascontiguousarray(sc["D"], np.float64)
    ovi, ovl = np.ascontiguousarray(sc["ov_ids"], np.int32), np.ascontiguousarray(sc["ov_lens"], np.float64)
    F, mm = fids.shape
    out = np.zeros(F, LOC_DTYPE)
    p0 = np.zeros((F, 6))
    used = np.zeros((F, mm), np.int32)
    cb = None if cam_base is None else np.ascontiguousarray(cam_base, np.float64)
    harness().hs_map_localize(n, _p(ids), _p(var), _p(poses), F, _p(counts), _p(fids), _p(cr), mm, _p(K), _p(D), float(sc["fiducial_len"]), len(ovi), _p(ovi), _p(ovl),
                              float(max_entry_variance), _p(cb) if cb is not None else None, _p(out), _p(p0), _p(used))
    return out, p0, used


# ---- the oracle ----------------------------------------------------------------------------------------------------------------
def counted(sc, f, max_entry_variance=-1.0):
    """Detection indices of frame f that count: id in the map, once in the frame, variance within the bound."""
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    var = sc.get("var", entry_variances(sc))
    ids = [int(v) for v in sc["fids"][f, :sc["counts"][f]]]
    return [j for j, i in enumerate(ids) if i in pos and ids.count(i) == 1 and (max_entry_variance < 0 or var[pos[i]] <= max_entry_variance)]


def board_points(sc, f, used):
    """The frame's board: object points (float32, map frame) and image points of the counted detections, in detection order."""
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    O = mc.object_points(sc)
    obj, img = [], []
    for j in used:
        k = pos[int(sc["fids"][f, j])]
        obj.append((O[k] @ np.asarray(sc["start_R"][k]).T + sc["start_t"][k]).astype(np.float32))
        img.append(sc["corners"][f, j].astype(np.float32))
    return np.concatenate(obj), np.concatenate(img)


def _reproj(obj, img, R, t, K, D):
    """Sum of squared reprojection errors, or -1 with a point behind the camera (the depth test of ba_reproj)."""
    import cv2

    o = obj.astype(np.float64)
    if np.any((o @ R.T + t)[:, 2] <= 0):
        return -1.0
    uv = cv2.projectPoints(o, cv2.Rodrigues(R)[0], t, K, D)[0].reshape(-1, 2)
    return float(np.sum((uv - img.astype(np.float64)) ** 2))


def cv2_start(sc, f, used):
    """The start rule with cv2: the board's cv2.solvePnP(ITERATIVE), unless one marker's own cv2.solvePnP composed with its map pose
    reprojects every corner better; candidates with a corner behind the camera never count.  (start, R, t) with start 0 = board,
    1 + k = the k-th counted marker, -1 = none."""
    import cv2

    obj, img = board_points(sc, f, used)
    K, D = sc["K"], sc["D"]
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    eb = -1.0
    try:  # cv2 raises for a non-planar board with fewer than 6 points
        ok, rv, tv = cv2.solvePnP(obj, img, K, D, flags=cv2.SOLVEPNP_ITERATIVE)
    except cv2.error:
        ok = False
    if ok:
        Rb, tb = cv2.Rodrigues(rv)[0], tv.ravel()
        eb = _reproj(obj, img, Rb, tb, K, D)
    ec, jc, Rc, tc = -1.0, -1, None, None
    for k, j in enumerate(used):
        e = pos[int(sc["fids"][f, j])]
        h = float(np.float32(sc["lens"][e]) / np.float32(2))
        o = np.array([[-h, h, 0], [h, h, 0], [h, -h, 0], [-h, -h, 0]], np.float32)
        ok, rv, tv = cv2.solvePnP(o, sc["corners"][f, j].astype(np.float32), K, D, flags=cv2.SOLVEPNP_ITERATIVE)
        Rcm = cv2.Rodrigues(rv)[0]
        Rm, tm = np.asarray(sc["start_R"][e]), np.asarray(sc["start_t"][e])
        R = Rcm @ Rm.T
        t = tv.ravel() - R @ tm
        err = _reproj(obj, img, R, t, K, D)
        if err >= 0 and (ec < 0 or err < ec):
            ec, jc, Rc, tc = err, k, R, t
    if eb >= 0 and not (ec >= 0 and ec < eb):
        return 0, Rb, tb
    if ec >= 0:
        return 1 + jc, Rc, tc
    return -1, None, None


def cv2_refine(sc, f, used, p0):
    """cv2.solvePnP(obj, img, K, D, rvec0, tvec0, useExtrinsicGuess=True, SOLVEPNP_ITERATIVE): (rvec, tvec)."""
    import cv2

    obj, img = board_points(sc, f, used)
    rv, tv = np.array(p0[:3], np.float64).reshape(3, 1), np.array(p0[3:], np.float64).reshape(3, 1)
    ok, rv, tv = cv2.solvePnP(obj, img, sc["K"], sc["D"], rv, tv, useExtrinsicGuess=True, flags=cv2.SOLVEPNP_ITERATIVE)
    return rv.ravel(), tv.ravel()


def image_error(sc, f, used, rvec, tvec):
    """Mean squared reprojection error with the projections rounded to float32."""
    import cv2

    obj, img = board_points(sc, f, used)
    uv = cv2.projectPoints(obj.astype(np.float64), np.asarray(rvec, np.float64), np.asarray(tvec, np.float64), sc["K"], sc["D"])[0].reshape(-1, 2)
    d = uv.astype(np.float32).astype(np.float64) - img.astype(np.float64)
    return float(np.mean(np.sum(d * d, 1)))


def q_to_R(q):
    x, y, z, w = [float(v) for v in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]]) / (x * x + y * y + z * z + w * w)


def map_pose(rvec, tvec, cam_base=None):
    """T_mapCam from the camera-from-map rvec / tvec, composed with T_camBase when given: (R, t)."""
    import cv2

    Rcm = cv2.Rodrigues(np.asarray(rvec, np.float64))[0]
    R, t = Rcm.T, -Rcm.T @ np.asarray(tvec, np.float64)
    if cam_base is not None:
        Rb = q_to_R(cam_base[3:])
        R, t = R @ Rb, R @ np.asarray(cam_base[:3], np.float64) + t
    return R, t


def covariance(sc, f, used, rvec, tvec, cam_base=None, h=1e-6):
    """sigma^2 (J^T J)^-1 of the output pose under (Exp([dtheta]x) R, t + dt), J by central differences through cv2.projectPoints;
    sigma^2 = sum |e|^2 / (2 n - 6).  Order x y z, rotation about map X Y Z."""
    import cv2

    obj, img = board_points(sc, f, used)
    o, c = obj.astype(np.float64), img.astype(np.float64)
    K, D = sc["K"], sc["D"]
    Rcm = cv2.Rodrigues(np.asarray(rvec, np.float64))[0]
    tcm = np.asarray(tvec, np.float64)
    Rx, tx = map_pose(rvec, tvec, cam_base)
    Rcx, tcx = Rcm @ Rx, Rcm @ tx + tcm  # fixed: camera from the output frame

    def resid(d):
        R = cv2.Rodrigues(d[3:])[0] @ Rx
        t = tx + d[:3]
        Rc = Rcx @ R.T
        tc = tcx - Rc @ t
        return (cv2.projectPoints(o, cv2.Rodrigues(Rc)[0], tc, K, D)[0].reshape(-1, 2) - c).ravel()

    J = np.zeros((2 * len(o), 6))
    for k in range(6):
        e = np.zeros(6)
        e[k] = h
        J[:, k] = (resid(e) - resid(-e)) / (2 * h)
    r0 = resid(np.zeros(6))
    s2 = float(np.sum(r0 ** 2)) / (2 * len(o) - 6)
    return s2 * np.linalg.inv(J.T @ J), s2


def object_error(sc, f, used, rvec, tvec, img_err):
    import cv2

    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    Rcm = cv2.Rodrigues(np.asarray(rvec, np.float64))[0]
    diag, depth = [], []
    for j in used:
        c = sc["corners"][f, j].astype(np.float64)
        diag.append(np.linalg.norm(c[0] - c[2]))
        depth.append(np.linalg.norm(Rcm @ np.asarray(sc["start_t"][pos[int(sc["fids"][f, j])]]) + np.asarray(tvec)))
    return (img_err / np.mean(diag)) * (np.mean(depth) / sc["fiducial_len"])


def with_edits(sc):
    """sc plus edited frames appended at its end: a duplicated id, an unmapped id (999), a high-variance entry's id and a frame
    with only unmapped ids.  Returns (scene, the appended frames' indices)."""
    out = dict(sc)
    F = len(sc["counts"])
    src = [f for f in range(F) if sc["counts"][f] >= 4][:3]
    fids, cr, counts = [sc["fids"]], [sc["corners"]], [sc["counts"]]
    for k, f in enumerate(src):
        a, c, n = sc["fids"][f].copy(), sc["corners"][f].copy(), int(sc["counts"][f])
        if k == 0:  # duplicated id: both of its detections drop
            a[n], c[n] = a[1], c[1] + 2.0
            n += 1
        elif k == 1:  # an unmapped id in the middle
            a[n], c[n] = a[2], c[2]
            a[2], c[2] = 999, c[0] + 3.0
            n += 1
        fids.append(a[None])
        cr.append(c[None])
        counts.append(np.array([n], np.int32))
    a = np.full_like(sc["fids"][0], -1)
    a[:2] = [997, 998]
    c = np.zeros_like(sc["corners"][0])
    c[:2] = sc["corners"][src[0], :2]
    fids.append(a[None])
    cr.append(c[None])
    counts.append(np.array([2], np.int32))
    out["fids"], out["corners"], out["counts"] = np.concatenate(fids), np.concatenate(cr), np.concatenate(counts).astype(np.int32)
    out["cams"] = list(sc["cams"]) + [sc["cams"][f] for f in src] + [sc["cams"][src[0]]]
    return out, list(range(F, F + len(src) + 1))
