"""Seeded bundle-adjustment scenes for fid_map_bundle_adjust, shared by the tests and tools/bench_map_ba.py; the scipy oracle of the
problem map_ba.cuh states; and the host build of map_ba.cuh (tests/hostsim/map_ba_hostsim.cpp, compiled with g++ into a temporary
directory once per session).

A scene is a map (ids, true poses, which entries are fixed), the map as the fold leaves it (the free entries' poses perturbed in
position and orientation, so that the ceiling is no longer planar), and a recorded sequence in fid_detect_pose_batch's dense layout: the corners of every visible marker projected with synth.project_points
plus Gaussian noise.  The markers sit on synth.make_c5_sequence's ceiling grid (1 m pitch, z = 2.5 m, rpy (180, 0, 180)) and,
optionally, on a wall at x = -1 facing +x; the camera follows make_c5_sequence's lawn-mower path below, looking up, tilted when
`oblique`."""
import atexit
import ctypes as C
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np

from fiducials_b200 import synth

_HERE = os.path.dirname(os.path.abspath(__file__))
_harness = None
_vp = C.c_void_p
REF_D = np.array([-0.28, 0.07, 1e-4, -2e-4, 0.0])  # the reference distortion of the sweep
MAX_MARKERS = 64


def _p(a):
    return a.ctypes.data_as(_vp)


def harness():
    global _harness
    if _harness is None:
        tmp = tempfile.mkdtemp(prefix="fid_map_ba_hostsim_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libfid_map_ba_hostsim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", so, os.path.join(_HERE, "hostsim", "map_ba_hostsim.cpp")])
        _harness = C.CDLL(so)
        _harness.hs_map_ba.argtypes = [C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, _vp, C.c_int, _vp, _vp, C.c_double, C.c_int, _vp, _vp, C.c_int, C.c_double] + [_vp] * 5
        _harness.hs_ba_corner.argtypes = [_vp] * 7
    return _harness


def rot(rvec):
    return synth._rodrigues(np.asarray(rvec, np.float64))


def rpy_R(r, p, y):
    return synth._q_to_R(synth._q_from_rpy(r, p, y))


def make_scene(seed, n_markers=16, n_frames=40, walls=0, noise=0.5, dist=False, oblique=False, overrides=False, n_fixed=1, visible=8, perturb=(0.03, 1.0),
               size=(1280, 800), f=700.0, fiducial_len=0.14, flat_start=False):
    """A seeded scene (see the module docstring).  n_markers on the ceiling grid (columns of ceil(sqrt(n)) at 1 m pitch) plus
    `walls` wall markers; entries 0 .. n_fixed - 1 are fixed (variance 0).  perturb = (metres, degrees) of the start map's error:
    in every direction, heights and tilts included, as a fold leaves a map (no longer planar); with flat_start only within each
    marker's plane (a planar ceiling stays planar)."""
    rng = np.random.default_rng(seed)
    cols = max(2, int(math.ceil(math.sqrt(n_markers))))
    ids = np.arange(n_markers + walls, dtype=np.int32) * 3 + 1  # not 0 .. n - 1: ids are looked up, not indexed
    R_ceil = rpy_R(math.pi, 0.0, math.pi)
    Rs, ts = [], []
    for i in range(n_markers):
        Rs.append(R_ceil @ rot([0.0, 0.0, rng.normal(0, math.radians(5))]))
        ts.append(np.array([float(i % cols), float(i // cols), 2.5]) + np.r_[rng.normal(0, 0.02, 2), 0.0])
    rows = int(math.ceil(n_markers / cols))
    for k in range(walls):
        Rs.append(rpy_R(math.pi / 2, 0.0, -math.pi / 2) @ rot(rng.normal(0, math.radians(2), 3)))  # z axis along +x
        ts.append(np.array([-1.0, (k + 0.5) * max(rows - 1, 1) / max(walls, 1), 1.6 + 0.6 * (k % 2)]))
    Rs, ts = np.array(Rs), np.array(ts)
    lens = np.full(len(ids), fiducial_len)
    ov_ids, ov_lens = np.zeros(0, np.int32), np.zeros(0)
    if overrides:
        sel = ids[1::3]
        ov_ids, ov_lens = sel.astype(np.int32), np.round(rng.uniform(0.1, 0.25, len(sel)), 3)
        for i, l in zip(ov_ids, ov_lens):
            lens[ids == i] = l
    fixed = np.zeros(len(ids), bool)
    fixed[:n_fixed] = True
    W, H = size
    K = np.array([[f, 0, (W - 1) / 2], [0, f, (H - 1) / 2], [0, 0, 1.0]])
    D = REF_D.copy() if dist else np.zeros(5)
    counts = np.zeros(n_frames, np.int32)
    fids = np.full((n_frames, MAX_MARKERS), -1, np.int32)
    corners = np.zeros((n_frames, MAX_MARKERS, 4, 2), np.float32)
    cams = []
    for k in range(n_frames):
        s = k / max(1, n_frames - 1) * rows
        row = min(int(s), rows - 1)
        fx = s - row
        c = np.array([fx * (cols - 1) if row % 2 == 0 else (1 - fx) * (cols - 1), float(row), 0.2 * math.sin(0.3 * k)])
        R_wc = rpy_R(0.0, 0.0, 0.3 * math.sin(0.05 * k) + 0.1 * k)
        if oblique or walls:
            R_wc = R_wc @ rot(np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.6, 0.1) - (0.4 if walls else 0.0), 0.0]))
        Rf, tf = R_wc.T, -R_wc.T @ c
        cams.append((Rf, tf))
        cand = []
        # markers farther than 8 m fail the facing test below anyway (the ceiling is 2.3 m above the path): skip them early
        for i in np.nonzero(np.linalg.norm(ts[:, :2] - c[:2], axis=1) < 8.0)[0]:
            h = float(np.float32(lens[i]) / np.float32(2))
            o = np.array([[-h, h, 0], [h, h, 0], [h, -h, 0], [-h, -h, 0]])
            Xc = (o @ Rs[i].T + ts[i]) @ Rf.T + tf
            if Xc[:, 2].min() < 0.3:
                continue
            n_c = Rf @ Rs[i][:, 2]
            if np.dot(n_c, Xc.mean(0)) / np.linalg.norm(Xc.mean(0)) > -0.35:  # facing the camera, at most ~70 degrees off
                continue
            uv = synth.project_points(o @ Rs[i].T + ts[i], Rf, tf, K, D)
            if uv.min() < 5 or uv[:, 0].max() > W - 6 or uv[:, 1].max() > H - 6:
                continue
            cand.append((np.linalg.norm(Xc.mean(0)), i, uv))
        cand.sort(key=lambda x: x[0])
        cand = cand[:visible]
        order = rng.permutation(len(cand))
        for j, q in enumerate(order):
            _, i, uv = cand[q]
            fids[k, j] = ids[i]
            corners[k, j] = (uv + rng.normal(0, noise, uv.shape)).astype(np.float32)
        counts[k] = len(cand)
    start_R, start_t = Rs.copy(), ts.copy()
    for i in range(len(ids)):
        if not fixed[i]:
            if flat_start:
                start_R[i] = Rs[i] @ rot([0.0, 0.0, rng.normal(0, math.radians(perturb[1]))])
                start_t[i] = ts[i] + Rs[i] @ np.r_[rng.normal(0, perturb[0], 2), 0.0]
            else:
                start_R[i] = Rs[i] @ rot(rng.normal(0, math.radians(perturb[1]), 3))
                start_t[i] = ts[i] + rng.normal(0, perturb[0], 3)
    return dict(ids=ids, R=Rs, t=ts, fixed=fixed, start_R=start_R, start_t=start_t, counts=counts, fids=fids, corners=corners, K=K, D=D, lens=lens,
                fiducial_len=fiducial_len, ov_ids=ov_ids, ov_lens=ov_lens, cams=cams, size=size)


def criteria_of(criteria):
    if criteria is None:
        return 100, 1e-12
    t, n, e = criteria
    return (min(max(int(n), 1), 1000) if t & 1 else 100), (float(e) if t & 2 else 1e-12)


def hs_bundle_adjust(sc, criteria=None, fixed=None, start=None):
    """The host build: dict with R, t of every entry (after), std [n][6] (0 for fixed / unreached), rvecs, tvecs, status per
    frame, rc and the stats.  criteria "init": only the initial frame poses (rvecs, tvecs)."""
    n = len(sc["ids"])
    fx = np.ascontiguousarray(sc["fixed"] if fixed is None else fixed, np.uint8)
    R0, t0 = (sc["start_R"], sc["start_t"]) if start is None else start
    poses = np.ascontiguousarray(np.concatenate([np.asarray(R0).reshape(n, 9), np.asarray(t0).reshape(n, 3)], 1), np.float64)
    nf = len(sc["counts"])
    rv, tv, st, sd, stats = np.zeros((nf, 3)), np.zeros((nf, 3)), np.zeros(nf, np.int32), np.zeros((n, 6)), np.zeros(16)
    max_iter, eps = (0, 0.0) if criteria == "init" else criteria_of(criteria)
    ids = np.ascontiguousarray(sc["ids"], np.int32)
    counts = np.ascontiguousarray(sc["counts"], np.int32)
    fids = np.ascontiguousarray(sc["fids"], np.int32)
    cr = np.ascontiguousarray(sc["corners"], np.float32)
    K = np.ascontiguousarray(sc["K"], np.float64)
    D = np.ascontiguousarray(sc["D"], np.float64)
    ovi, ovl = np.ascontiguousarray(sc["ov_ids"], np.int32), np.ascontiguousarray(sc["ov_lens"], np.float64)
    rc = harness().hs_map_ba(n, _p(ids), _p(fx), _p(poses), nf, _p(counts), _p(fids), _p(cr), fids.shape[1], _p(K), _p(D), float(sc["fiducial_len"]), len(ovi), _p(ovi),
                             _p(ovl), max_iter, eps, _p(rv), _p(tv), _p(st), _p(sd), _p(stats))
    return dict(rc=rc, R=poses[:, :9].reshape(n, 3, 3), t=poses[:, 9:].copy(), std=sd, rvecs=rv, tvecs=tv, status=st, initial_rms=stats[0], final_rms=stats[1],
                iterations=int(stats[2]), steps=int(stats[3]), frames_used=int(stats[4]), markers_used=int(stats[5]), observations=int(stats[6]),
                dropped_unmapped=int(stats[7]), dropped_duplicate=int(stats[8]), frames_unreached=int(stats[9]), markers_unreached=int(stats[10]),
                init_failed=int(stats[11]), converged=int(stats[12]))


def hs_corner(o, c, K, D, pf, pm):
    out = np.zeros(26)
    a = [np.ascontiguousarray(v, np.float64) for v in (o, K, D, pf, pm)]
    cc = np.ascontiguousarray(c, np.float32)
    harness().hs_ba_corner(_p(a[0]), _p(cc), _p(a[1]), _p(a[2]), _p(a[3]), _p(a[4]), _p(out))
    return out[:2], out[2:14].reshape(2, 6), out[14:].reshape(2, 6)


# ---- the oracle: scipy.optimize.least_squares on the same residuals ------------------------------------------------------------
def observations(sc):
    """The observations that count (map_ba.cuh's rules, restated): (frame, entry index, corners [4][2]) per observation, frames in
    order, detections in order; ids not in the map ignored, an id seen twice in a frame dropped there."""
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    out = []
    for f in range(len(sc["counts"])):
        ids = [int(v) for v in sc["fids"][f, :sc["counts"][f]]]
        for j, i in enumerate(ids):
            if i in pos and ids.count(i) == 1:
                out.append((f, pos[i], sc["corners"][f, j].astype(np.float64)))
    return out


def object_points(sc):
    out = []
    for i, l in zip(sc["ids"], sc["lens"]):
        h = float(np.float32(l) / np.float32(2))
        out.append(np.array([[-h, h, 0], [h, h, 0], [h, -h, 0], [-h, -h, 0]]))
    return np.array(out)


def scipy_bundle_adjust(sc, frame_R, frame_t, fixed=None):
    """least_squares (trf, x_scale='jac', xtol = ftol = gtol = 1e-15) over the used frames (frame_R / frame_t: dicts frame -> start
    pose) and the free entries, each rotation as R0 Rodrigues(delta).  Central differences by column groups (a residual depends on
    one frame and one marker).  Returns R, t of every entry, frame poses, cost = sum e^2, and the standard deviations of every free
    entry's (delta, t) from numpy's (J^T J)^-1 at the optimum times sum e^2 / (residuals - parameters)."""
    from scipy.optimize import least_squares

    fixed = sc["fixed"] if fixed is None else fixed
    obs = [o for o in observations(sc) if o[0] in frame_R]
    frames = sorted(frame_R)
    fidx = {f: k for k, f in enumerate(frames)}
    free = [i for i in range(len(sc["ids"])) if not fixed[i] and any(o[1] == i for o in obs)]
    midx = {i: k for k, i in enumerate(free)}
    O = object_points(sc)
    K, D = sc["K"], sc["D"]
    F, M = len(frames), len(free)
    oi_f = np.array([fidx[o[0]] for o in obs])
    oi_m = np.array([o[1] for o in obs])
    C4 = np.array([o[2] for o in obs])
    R0f = np.array([frame_R[f] for f in frames])
    R0m = np.array(sc["start_R"], np.float64)

    def rods(d):
        th = np.linalg.norm(d, axis=1)[:, None, None]
        th_s = np.where(th < 1e-300, 1.0, th)
        k = d / th_s[:, :, 0]
        Kx = np.zeros((len(d), 3, 3))
        Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 0], Kx[:, 1, 2], Kx[:, 2, 0], Kx[:, 2, 1] = -k[:, 2], k[:, 1], k[:, 2], -k[:, 0], -k[:, 1], k[:, 0]
        return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * (Kx @ Kx)

    def unpack(x):
        xf = x[:6 * F].reshape(F, 6)
        xm = x[6 * F:].reshape(M, 6)
        Rf = R0f @ rods(xf[:, :3])
        Rm = R0m.copy()
        tm = np.array(sc["start_t"], np.float64).copy()
        if M:
            Rm[free] = R0m[free] @ rods(xm[:, :3])
            tm[free] = xm[:, 3:]
        return Rf, xf[:, 3:], Rm, tm

    def resid(x):
        Rf, tf, Rm, tm = unpack(x)
        X = np.einsum("nij,nkj->nki", Rm[oi_m], O[oi_m]) + tm[oi_m][:, None, :]
        Xc = np.einsum("nij,nkj->nki", Rf[oi_f], X) + tf[oi_f][:, None, :]
        x_, y_ = Xc[..., 0] / Xc[..., 2], Xc[..., 1] / Xc[..., 2]
        k1, k2, p1, p2, k3 = D
        r2 = x_ * x_ + y_ * y_
        cd = 1 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2
        xd = x_ * cd + 2 * p1 * x_ * y_ + p2 * (r2 + 2 * x_ * x_)
        yd = y_ * cd + p1 * (r2 + 2 * y_ * y_) + 2 * p2 * x_ * y_
        u = np.stack([xd * K[0, 0] + K[0, 2], yd * K[1, 1] + K[1, 2]], -1)
        return (u - C4).reshape(-1)

    rows_f = np.repeat(oi_f, 8)
    rows_m = np.repeat(np.array([midx.get(i, -1) for i in oi_m]), 8)

    def jac(x):
        J = np.zeros((8 * len(obs), 6 * (F + M)))
        h = 1e-6
        for k in range(6):
            for block, n, rows in ((0, F, rows_f), (6 * F, M, rows_m)):
                if n == 0:
                    continue
                e = np.zeros_like(x)
                e[block + k:block + 6 * n:6] = h
                d = (resid(x + e) - resid(x - e)) / (2 * h)
                ok = rows >= 0
                J[np.nonzero(ok)[0], block + 6 * rows[ok] + k] = d[ok]
        return J

    x0 = np.concatenate([np.concatenate([np.zeros((F, 3)), np.array([frame_t[f] for f in frames])], 1).reshape(-1),
                         np.concatenate([np.zeros((M, 3)), np.array(sc["start_t"], np.float64)[free]], 1).reshape(-1) if M else np.zeros(0)])
    r = least_squares(resid, x0, jac=jac, method="trf", x_scale="jac", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    Rf, tf, Rm, tm = unpack(r.x)
    # the standard deviations in the tangent space at the optimum (R* Exp(delta), as the solver reports them): re-linearise at delta 0
    R0f[:] = Rf
    R0m[free] = Rm[free]
    x1 = r.x.copy()
    x1[:6 * F].reshape(F, 6)[:, :3] = 0
    if M:
        x1[6 * F:].reshape(M, 6)[:, :3] = 0
    J = jac(x1)
    cost = float(np.sum(r.fun ** 2))
    cov = np.linalg.inv(J.T @ J) * cost / (len(r.fun) - len(r.x))
    sd = np.zeros((len(sc["ids"]), 6))
    for i in free:
        sd[i] = np.sqrt(np.diag(cov)[6 * F + 6 * midx[i]:6 * F + 6 * midx[i] + 6])
    return dict(R=Rm, t=tm, frame_R=dict(zip(frames, Rf)), frame_t=dict(zip(frames, tf)), cost=cost, std=sd, free=free, nfev=r.nfev)


def rot_delta(Ra, Rb):
    """The rotation vector of Ra^T Rb (the R Exp(delta) convention of the solver)."""
    import cv2

    return cv2.Rodrigues(np.ascontiguousarray(Ra.T @ Rb))[0].ravel()


def assert_matches_scipy(got, ref, what="", std_tol=1e-4, cost_tol=1e-9):
    """Final cost within cost_tol relative, every free entry's (delta, t) within 1e-4 of its standard deviation, and the standard
    deviations within std_tol relative of scipy's."""
    n_c = 4 * got["observations"]
    cost = got["final_rms"] ** 2 * n_c
    assert abs(cost / ref["cost"] - 1) <= cost_tol, (what, cost, ref["cost"])
    for i in ref["free"]:
        sd = ref["std"][i]
        d = np.r_[rot_delta(ref["R"][i], got["R"][i]), got["t"][i] - ref["t"][i]]
        assert np.all(np.abs(d) <= 1e-4 * sd), (what, i, np.abs(d) / sd)
        assert np.all(np.abs(got["std"][i] / sd - 1) <= std_tol), (what, i, got["std"][i] / sd - 1)


def join_disconnected(sc, other):
    """sc plus `other`'s markers (ids moved past sc's, none fixed) and frames: `other`'s frames see only its own markers, so its
    group is not connected to sc's fixed entries."""
    off = int(sc["ids"].max()) + 1000
    out = dict(sc)
    for k in ("R", "t", "start_R", "start_t", "lens"):
        out[k] = np.concatenate([sc[k], other[k]])
    out["ids"] = np.concatenate([sc["ids"], other["ids"] + off]).astype(np.int32)
    out["fixed"] = np.concatenate([sc["fixed"], np.zeros(len(other["ids"]), bool)])
    of = np.where(other["fids"] >= 0, other["fids"] + off, -1)
    out["fids"] = np.concatenate([sc["fids"], of]).astype(np.int32)
    out["counts"] = np.concatenate([sc["counts"], other["counts"]]).astype(np.int32)
    out["corners"] = np.concatenate([sc["corners"], other["corners"]])
    out["cams"] = list(sc["cams"]) + list(other["cams"])
    return out


def board_init_cv2(sc, f):
    """cv2.aruco.Board over the start map's corners (float32) + matchImagePoints + cv2.solvePnP(ITERATIVE) for frame f's mapped,
    non-duplicated detections: (ok, rvec, tvec)."""
    import cv2

    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    O = object_points(sc)
    ids = [int(v) for v in sc["fids"][f, :sc["counts"][f]]]
    keep = [j for j, i in enumerate(ids) if i in pos and ids.count(i) == 1]
    board_ids = sorted({ids[j] for j in keep})
    objp = [np.ascontiguousarray((O[pos[i]] @ sc["start_R"][pos[i]].T + sc["start_t"][pos[i]]).astype(np.float32)) for i in board_ids]
    board = cv2.aruco.Board(objp, cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_ARUCO_ORIGINAL), np.array(board_ids, np.int32))
    det = [sc["corners"][f, j].reshape(1, 4, 2).astype(np.float32) for j in keep]
    obj, img = board.matchImagePoints(det, np.array([ids[j] for j in keep], np.int32))
    ok, rv, tv = cv2.solvePnP(obj, img, sc["K"], sc["D"], flags=cv2.SOLVEPNP_ITERATIVE)
    return ok, rv.ravel(), tv.ravel()


def file_entries(sc, start=True):
    """The map as FiducialSlam.loadMap rows: id, x, y, z, roll, pitch, yaw (degrees), variance, num_obs."""
    R, t = (sc["start_R"], sc["start_t"]) if start else (sc["R"], sc["t"])
    rows = []
    for k, i in enumerate(sc["ids"]):
        r = math.atan2(R[k][2, 1], R[k][2, 2])
        p = -math.asin(max(-1.0, min(1.0, R[k][2, 0])))
        y = math.atan2(R[k][1, 0], R[k][0, 0])
        rows.append([int(i), t[k][0], t[k][1], t[k][2], math.degrees(r), math.degrees(p), math.degrees(y), 0.0 if sc["fixed"][k] else 0.01 * (1 + k % 3), 3 + k])
    return rows


def loaded_pose(row):
    """The pose fid_map_load stores for a row, with its arithmetic (tf2 setRPY, then setRotation), so that the host build starts
    from the device map's bits."""
    d2r = 3.14159265358979323846 / 180.0
    hr, hp, hy = row[4] * d2r * 0.5, row[5] * d2r * 0.5, row[6] * d2r * 0.5
    cy, sy, cp, sp, cr, sr = math.cos(hy), math.sin(hy), math.cos(hp), math.sin(hp), math.cos(hr), math.sin(hr)
    x, y, z, w = sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy
    d = x * x + y * y + z * z + w * w
    s = 2.0 / d
    xs, ys, zs = x * s, y * s, z * s
    wx, wy, wz = w * xs, w * ys, w * zs
    xx, xy, xz = x * xs, x * ys, x * zs
    yy, yz, zz = y * ys, y * zs, z * zs
    R = np.array([[1.0 - (yy + zz), xy - wz, xz + wy], [xy + wz, 1.0 - (xx + zz), yz - wx], [xz - wy, yz + wx, 1.0 - (xx + yy)]])
    return R, np.array(row[1:4], np.float64)


def as_loaded(sc):
    """sc with its start map replaced by the poses fid_map_load makes of file_entries(sc)."""
    out = dict(sc)
    P = [loaded_pose(r) for r in file_entries(sc)]
    out["start_R"] = np.array([p[0] for p in P])
    out["start_t"] = np.array([p[1] for p in P])
    return out


def map_error(sc, R, t, ref=0):
    """RMS position (m) and rotation (rad) error of the entries other than `ref` against the truth, both expressed in entry
    ref's frame (the gauge of a map is its origin)."""
    def rel(Ra, ta, Rb, tb):
        return Ra.T @ Rb, Ra.T @ (tb - ta)
    dp, dr = [], []
    for i in range(len(sc["ids"])):
        if i == ref:
            continue
        Rg, tg = rel(R[ref], t[ref], R[i], t[i])
        Rt, tt = rel(sc["R"][ref], sc["t"][ref], sc["R"][i], sc["t"][i])
        dp.append(np.sum((tg - tt) ** 2))
        dr.append(np.sum(rot_delta(Rt, Rg) ** 2))
    return math.sqrt(np.mean(dp)), math.sqrt(np.mean(dr))
