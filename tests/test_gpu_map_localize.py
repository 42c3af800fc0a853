"""fid_map_localize on the device: against the host build of map_localize.cuh and against cv2 on the host tests' scenes; a map
loaded by fid_map_load (stale id hash: linear search) and the same map after a fold rebuilt the hash; an asynchronous fold is
seen; reruns are bit-identical; the refusals and the frame cap; and end to end, from rendered frames through
fid_detect_pose_batch and the fold, the joint pose's position error next to the fold's robot pose on the same read-only map."""
import os

import numpy as np
import pytest

import map_ba_cases as mc
import map_localize_cases as lc
from test_gpu_map_ba import _render
from test_hostsim_map_localize import MOUNT, _check_frames
from fiducials_b200 import _lib
from fiducials_b200.node import Detector, FiducialSlam, default_params

pytestmark = pytest.mark.gpu
IDENT = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]


def _slam(sc, cap=256):
    s = FiducialSlam(max_fiducials=cap)
    s.loadMap(mc.file_entries(sc))
    return s


def _loc(s, sc, **kw):
    ov = {int(i): float(l) for i, l in zip(sc["ov_ids"], sc["ov_lens"])}
    return s.localize(sc["counts"], sc["fids"], sc["corners"], sc["K"], sc["D"], sc["fiducial_len"], ov, **kw)


def _loaded(sc):
    """The scene as the device holds it after fid_map_load of mc.file_entries (the start map)."""
    out = mc.as_loaded(sc)
    out["var"] = lc.entry_variances(sc)
    return out


def _same_as_host(d, h):
    used = h["status"] == 1
    assert np.array_equal(d["status"], h["status"]) and np.array_equal(d["start"], h["start"]) and np.array_equal(d["n_markers"], h["n_markers"])
    assert np.array_equal(d["cov_ok"], h["cov_ok"]) and np.array_equal(d["have_base"], h["have_base"])
    dp = max(np.abs(d["rvec"][used] - h["rvec"][used]).max(initial=0), np.abs(d["tvec"][used] - h["tvec"][used]).max(initial=0))
    dc = np.abs(d["covariance"][used] - h["covariance"][used]).max(initial=0) / max(np.abs(h["covariance"][used]).max(initial=0), 1e-300)
    de = np.abs(d["image_error"][used] / h["image_error"][used] - 1).max(initial=0)
    print("device - host: pose %.2e, covariance %.2e (relative to its largest entry), image error %.2e" % (dp, dc, de))
    assert dp <= 1e-7 and dc <= 1e-6 and de <= 1e-9


@pytest.mark.parametrize("kw", [dict(seed=1, dist=True, noise=0.5), dict(seed=2, walls=3, oblique=True, noise=0.5),
                                dict(seed=4, overrides=True, noise=0.5, n_markers=25), dict(seed=5, visible=1, noise=0.5)],
                         ids=["fold-dist", "fold-walls", "fold-overrides", "one-marker"])
def test_device_matches_host_and_cv2(kw):
    kw = dict(kw)
    sc = _loaded(mc.make_scene(kw.pop("seed"), n_frames=30, **kw))
    s = _slam(sc)
    for cam_base in (None, MOUNT):
        d = _loc(s, sc, T_camBase=cam_base)
        h, p0, used = lc.hs_localize(sc, cam_base=cam_base)
        _same_as_host(d, h)
        assert _check_frames(sc, d, p0, used, range(len(d)), cam_base=cam_base) >= 20  # the device records against cv2


def test_edited_frames_and_variance_bound():
    sc, _ = lc.with_edits(_loaded(mc.make_scene(7, dist=True, noise=0.5, n_frames=12)))
    s = _slam(sc)
    for mv in (-1.0, 0.015):
        d = _loc(s, sc, max_entry_variance=mv)
        h, p0, used = lc.hs_localize(sc, max_entry_variance=mv)
        _same_as_host(d, h)
        assert 0 in d["status"]


def test_hash_rebuilt_by_a_fold_and_reruns_bit_identical():
    """After fid_map_load the id hash is stale and the kernel searches linearly; an empty message through the fold rebuilds the
    hash without changing an entry: the records are bit-identical either way, and on reruns."""
    sc = _loaded(mc.make_scene(11, dist=True, noise=0.5, n_frames=40, n_markers=25))
    s = _slam(sc)
    a = _loc(s, sc, T_camBase=MOUNT)
    b = _loc(s, sc, T_camBase=MOUNT)
    s.transformCallback([], IDENT, IDENT)
    c = _loc(s, sc, T_camBase=MOUNT)
    assert a.tobytes() == b.tobytes() == c.tobytes()


def test_pending_asynchronous_fold_is_seen():
    """A localization right after an asynchronous fold sees the folded map: the same records as after a synchronous one, and not
    those of the map before it."""
    sc = _loaded(mc.make_scene(51, n_markers=9, n_frames=30))
    det = Detector(max_width=64, max_height=64)
    tfs = (_lib.fid_transform * (len(sc["counts"]) * _lib.FID_MAX_MARKERS))()
    counts = np.zeros(len(sc["counts"]), np.int32)
    for f in range(6):
        n = int(sc["counts"][f])
        out = det.pose(sc["fids"][f, :n], sc["corners"][f, :n] + 0.7, sc["K"], sc["D"], sc["fiducial_len"])  # shifted corners: the fold moves entries
        for j in range(n):
            tfs[f * _lib.FID_MAX_MARKERS + j] = out[j]
        counts[f] = n
    before = _loc(_slam(sc), sc)
    res = []
    for asynchronous in (False, True):
        s = _slam(sc)
        s.update_frames(counts, tfs, IDENT, IDENT, asynchronous=asynchronous)
        res.append(_loc(s, sc))
    assert res[0].tobytes() == res[1].tobytes() and res[0].tobytes() != before.tobytes()


def test_refusals_and_frame_cap():
    sc = _loaded(mc.make_scene(61, n_markers=9, n_frames=8))
    s = _slam(sc)
    lib = _lib.load()

    def status(**kw):
        a = dict(counts=sc["counts"], fids=sc["fids"], corners=sc["corners"], K=sc["K"], D=sc["D"], instance=0)
        a.update(kw)
        try:
            s.localize(a["counts"], a["fids"], a["corners"], a["K"], a["D"], instance=a["instance"])
        except _lib.FidError as e:
            return e.status
        return 0

    assert status() == 0
    K0 = sc["K"].copy()
    K0[0, 0] = 0
    assert status(K=K0) == -1
    bad = sc["corners"].copy()
    bad[0, 0, 0, 0] = np.nan
    assert status(corners=bad) == -1
    c = sc["counts"].copy()
    c[0] = sc["fids"].shape[1] + 1
    assert status(counts=c) == -1
    assert status(instance=1) == -1
    wide = np.full((8, 257), -1, np.int32)
    assert status(counts=np.zeros(8, np.int32), fids=wide, corners=np.zeros((8, 257, 4, 2), np.float32)) == -1
    n = 65537
    out = np.full(n, 0x5A, np.uint8)  # nothing written past a refusal
    import ctypes as C

    from fiducials_b200.node import _camera

    z = np.zeros(n, np.int32)
    ids = np.zeros((n, 1), np.int32)
    cr = np.zeros((n, 1, 8), np.float32)
    cam = _camera(sc["K"], sc["D"])
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    rc = lib.fid_map_localize(s.h, 0, n, p(z), p(ids), p(cr), 1, C.byref(cam), 0.14, 0, None, None, -1.0, None,
                              C.cast(out.ctypes.data, C.POINTER(_lib.fid_localization)))
    assert rc == -5 and np.all(out == 0x5A)


def test_end_to_end_joint_pose_next_to_the_fold():
    """Rendered 1080p frames -> fid_detect_pose_batch -> the fold builds the map -> the map saved and loaded read-only -> per frame
    the fold's robot pose (transformCallback) and the joint pose (localize) on the same map.  Camera positions against the truth,
    in the world frame through the fold's origin entry; both printed (DESIGN.md f17), a loose bound only."""
    dict_id, flen = 7, 0.2
    sc = mc.make_scene(91, n_markers=25, n_frames=60, noise=0.0, visible=10, oblique=True, size=(1920, 1080), f=900.0, fiducial_len=flen)
    frames = np.stack([_render(sc, f, dict_id) for f in range(len(sc["counts"]))])
    det = Detector(default_params(dictionary=dict_id), 0, 1920, 1080, 8)
    counts, ids, corners, tfs = det.detect_pose_batch(frames, sc["K"], sc["D"], flen)
    build = FiducialSlam(max_fiducials=64)
    build.update_frames(counts, tfs, IDENT, IDENT)
    path = os.path.join(os.environ.get("TMPDIR", "/tmp"), "fid_loc_map_%d.txt" % os.getpid())
    build.saveMap(path)
    ro = FiducialSlam(max_fiducials=64, read_only_map=True)
    ro.loadMapFile(path)
    os.remove(path)
    ents = {e.fiducial_id: e for e in ro.entries()}
    origin = [i for i, e in ents.items() if e.variance == 0.0][0]
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    eo = ents[origin]
    R_mo = mc.loaded_pose([0, eo.x, eo.y, eo.z, np.degrees(eo.rx), np.degrees(eo.ry), np.degrees(eo.rz)])[0]
    R_wo, t_wo = sc["R"][pos[origin]], sc["t"][pos[origin]]
    R_wm = R_wo @ R_mo.T
    t_wm = t_wo - R_wm @ np.array([eo.x, eo.y, eo.z])
    loc = ro.localize(counts, ids, corners, sc["K"], sc["D"], flen)
    e_joint, e_fold = [], []
    for f in range(len(counts)):
        msg = [dict(fiducial_id=int(t.fiducial_id), translation=list(t.translation), rotation=list(t.rotation), image_error=t.image_error, object_error=t.object_error,
                    fiducial_area=t.fiducial_area) for t in (tfs[f * _lib.FID_MAX_MARKERS + j] for j in range(counts[f]))]
        robot = ro.transformCallback(msg, IDENT, IDENT)
        truth = -sc["cams"][f][0].T @ sc["cams"][f][1]
        if robot.valid and loc[f]["status"] == 1:
            e_fold.append(np.linalg.norm(R_wm @ np.array(robot.t[:]) + t_wm - truth))
            e_joint.append(np.linalg.norm(R_wm @ loc[f]["t"] + t_wm - truth))
    e_joint, e_fold = np.array(e_joint), np.array(e_fold)
    print("camera position error (m) over %d frames: joint median %.4f p95 %.4f; fold median %.4f p95 %.4f" %
          (len(e_joint), np.median(e_joint), np.percentile(e_joint, 95), np.median(e_fold), np.percentile(e_fold, 95)))
    assert len(e_joint) >= 40 and np.median(e_joint) < 0.2
