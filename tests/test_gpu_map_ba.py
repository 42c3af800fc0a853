"""fid_map_bundle_adjust on the device: against the host build of map_ba.cuh (the same computation up to the rounding of the
reduced system's tensor-core Cholesky) and bit-identical on reruns; against scipy on part of the CPU sweep; the write-back into
the map (free entries only; variances, observation counts, links and the other entries untouched); frames that see only fixed
entries; the caps and refusals; FiducialSlam.bundle_adjust against the C call; and end to end, from rendered 1080p frames through
fid_detect_pose_batch and the fold, a map closer to the truth than the fold's (and in rotation than fid_map_refine's)."""
import math

import numpy as np
import pytest

import map_ba_cases as mc
import ctypes as C

from fiducials_b200 import _lib, synth
from fiducials_b200.node import Detector, FiducialSlam, _camera, default_params

pytestmark = pytest.mark.gpu

# device against host: the reduced system is summed and factored blockwise on the tensor cores, so values agree to rounding
# amplified by its condition, not bit for bit (the bound the calibrations use; the measured value is in DESIGN.md f16)
HOST_TOL = 1e-6


def _slam(sc, cap=256):
    s = FiducialSlam(max_fiducials=cap)
    s.loadMap(mc.file_entries(sc))
    return s


def _ba(s, sc, criteria=None):
    ov = {int(i): float(l) for i, l in zip(sc["ov_ids"], sc["ov_lens"])}
    return s.bundle_adjust(sc["counts"], sc["fids"], sc["corners"], sc["K"], sc["D"], sc["fiducial_len"], ov, criteria=criteria)


def _entries(s):
    return {e.fiducial_id: (e.num_obs, e.x, e.y, e.z, e.rx, e.ry, e.rz, e.variance) for e in s.entries()}


def _R_of(e):
    row = [0, e[1], e[2], e[3], math.degrees(e[4]), math.degrees(e[5]), math.degrees(e[6])]
    return mc.loaded_pose(row)[0]


def _rel(a, b):
    """Differences relative to the pose scale: a small rvec or tvec component is compared in radians or metres (max(|b|, 1))."""
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b)) / np.maximum(np.abs(b), 1.0), initial=0.0))


@pytest.mark.parametrize("seed,nm,nf,walls,dist", [(2, 9, 30, 0, True), (4, 12, 40, 3, True), (7, 64, 400, 0, False)])
def test_device_matches_host_and_reruns_are_bit_identical(seed, nm, nf, walls, dist):
    sc = mc.as_loaded(mc.make_scene(seed, n_markers=nm, n_frames=nf, walls=walls, dist=dist, oblique=bool(walls)))
    h = mc.hs_bundle_adjust(sc)
    assert h["rc"] == 0
    outs = []
    for _ in range(2):
        s = _slam(sc)
        st, rv, tv, status, sd = _ba(s, sc)
        outs.append((rv.tobytes(), tv.tobytes(), status.tobytes(), np.array([sd[i] for i in sorted(sd)]).tobytes(), repr(sorted(_entries(s).items())),
                     st.final_rms, st.iterations))
    assert outs[0] == outs[1]
    assert np.array_equal(status, h["status"])
    # the iterations agree while the steps stay above rounding level; with the default epsilon (1e-12) the last accept / reject
    # decisions compare costs that differ in their last bits, and device and host may take a different number of them
    coarse = (3, 100, 1e-7)
    hc = mc.hs_bundle_adjust(sc, criteria=coarse)
    stc = _ba(_slam(sc), sc, criteria=coarse)[0]
    assert stc.iterations == hc["iterations"], (stc.iterations, hc["iterations"])
    assert st.frames_used == h["frames_used"] and st.markers_used == h["markers_used"] and st.observations_used == h["observations"]
    used = status == 1
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    ent = _entries(s)
    d_frames = max(_rel(rv[used], h["rvecs"][used]), _rel(tv[used], h["tvecs"][used]))
    d_map = max([_rel(e[1:4], h["t"][pos[i]]) for i, e in ent.items()] + [_rel(_R_of(e), h["R"][pos[i]]) for i, e in ent.items()])
    free = [i for i in ent if np.all(h["std"][pos[i]] > 0)]
    d_std = max(float(np.max(np.abs(sd[i] / h["std"][pos[i]] - 1))) for i in free)
    d_rms = abs(st.final_rms / h["final_rms"] - 1)
    print("device - host: frames %.2e, map %.2e, std %.2e, rms %.2e" % (d_frames, d_map, d_std, d_rms))
    assert abs(st.initial_rms / h["initial_rms"] - 1) <= HOST_TOL
    assert max(d_frames, d_map, d_std, d_rms) <= HOST_TOL
    for i in ent:
        if i not in free:
            assert np.all(sd[i] == 0)

def test_device_matches_scipy():
    sc = mc.as_loaded(mc.make_scene(3, n_markers=16, n_frames=40, noise=1.0, oblique=True, overrides=True))
    s = _slam(sc)
    st, rv, tv, status, sd = _ba(s, sc)
    i0 = mc.hs_bundle_adjust(sc, criteria="init")
    used = [f for f in range(len(sc["counts"])) if status[f] == 1]
    ref = mc.scipy_bundle_adjust(sc, {f: mc.rot(i0["rvecs"][f]) for f in used}, {f: i0["tvecs"][f] for f in used})
    ent = _entries(s)
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    got = dict(observations=st.observations_used, final_rms=st.final_rms, R=np.array(sc["start_R"]).copy(), t=np.array(sc["start_t"]).copy(),
               std=np.zeros((len(sc["ids"]), 6)))
    for i, e in ent.items():
        got["t"][pos[i]] = e[1:4]
        got["R"][pos[i]] = _R_of(e)
        got["std"][pos[i]] = sd[i]
    # the rotations come back through fid_map_entries' roll / pitch / yaw: compare them at that precision
    cost = st.final_rms ** 2 * 4 * st.observations_used
    assert abs(cost / ref["cost"] - 1) <= 1e-9
    for i in ref["free"]:
        d = np.r_[mc.rot_delta(ref["R"][i], got["R"][i]), got["t"][i] - ref["t"][i]]
        assert np.all(np.abs(d[3:]) <= 1e-4 * ref["std"][i][3:]) and np.all(np.abs(d[:3]) <= 1e-4 * ref["std"][i][:3] + 1e-12)
        assert np.all(np.abs(got["std"][i] / ref["std"][i] - 1) <= 1e-4)


def test_write_back_leaves_everything_else_alone():
    a = mc.make_scene(21, n_markers=9, n_frames=30)
    b = mc.make_scene(22, n_markers=4, n_frames=8, n_fixed=0)
    sc = mc.as_loaded(mc.join_disconnected(a, b))
    s = _slam(sc)
    links0 = s.links()
    before = _entries(s)
    st, rv, tv, status, sd = _ba(s, sc)
    after = _entries(s)
    assert s.links() == links0
    nb = len(b["ids"])
    unreached = {int(i) for i in sc["ids"][-nb:]}
    fixed = {int(i) for i, f in zip(sc["ids"], sc["fixed"]) if f}
    assert st.markers_unreached == nb
    for i in before:
        assert before[i][0] == after[i][0] and before[i][7] == after[i][7]  # num_obs, variance
        if i in unreached or i in fixed:
            assert before[i] == after[i] and np.all(sd[i] == 0)
        else:
            assert before[i] != after[i] and np.all(sd[i] > 0)


def test_refusals_and_caps():
    sc = mc.as_loaded(mc.make_scene(41, n_markers=4, n_frames=10))
    s = _slam(sc)
    before = _entries(s)
    bad = dict(sc)
    bad["corners"] = sc["corners"].copy()
    bad["corners"][2, 0, 1, 0] = np.nan
    with pytest.raises(_lib.FidError):
        _ba(s, bad)
    badK = dict(sc)
    badK["K"] = np.zeros((3, 3))
    with pytest.raises(_lib.FidError):
        _ba(s, badK)
    big = dict(sc)
    n = 65537
    big["counts"], big["fids"], big["corners"] = np.zeros(n, np.int32), np.zeros((n, 1), np.int32), np.zeros((n, 1, 4, 2), np.float32)
    with pytest.raises(_lib.FidError) as e:
        _ba(s, big)
    assert e.value.status == -5  # FID_ERR_CAPACITY
    assert _entries(s) == before
    nofix = dict(sc)
    nofix["fixed"] = np.zeros(len(sc["ids"]), bool)
    s2 = _slam(nofix)
    with pytest.raises(_lib.FidError):
        _ba(s2, nofix)


def test_pending_asynchronous_update_is_waited_for():
    """A bundle adjustment after an asynchronous fold sees the folded map: the same as after a synchronous one."""
    sc = mc.as_loaded(mc.make_scene(51, n_markers=9, n_frames=30))
    det = Detector(max_width=64, max_height=64)
    res = []
    for asynchronous in (False, True):
        s = _slam(sc)
        tfs = (_lib.fid_transform * (len(sc["counts"]) * _lib.FID_MAX_MARKERS))()
        counts = np.zeros(len(sc["counts"]), np.int32)
        for f in range(3):
            n = int(sc["counts"][f])
            out = det.pose(sc["fids"][f, :n], sc["corners"][f, :n], sc["K"], sc["D"], sc["fiducial_len"])
            for j in range(n):
                tfs[f * _lib.FID_MAX_MARKERS + j] = out[j]
            counts[f] = n
        s.update_frames(counts, tfs, asynchronous=asynchronous)
        _ba(s, sc)
        res.append(_entries(s))
    assert res[0] == res[1]


def test_frames_that_see_only_fixed_entries():
    sc = mc.as_loaded(mc.make_scene(61, n_markers=4, n_frames=12, n_fixed=4))
    s = _slam(sc)
    before = _entries(s)
    st, rv, tv, status, sd = _ba(s, sc)
    h = mc.hs_bundle_adjust(sc)
    assert st.markers_used == 0 and st.frames_used == h["frames_used"] > 0 and st.converged == 1
    assert _entries(s) == before and all(np.all(v == 0) for v in sd.values())
    used = status == 1
    assert _rel(rv[used], h["rvecs"][used]) <= HOST_TOL and _rel(tv[used], h["tvecs"][used]) <= HOST_TOL


def test_wrapper_returns_the_c_call_values():
    sc = mc.as_loaded(mc.make_scene(71, n_markers=9, n_frames=30, overrides=True))
    ov = {int(i): float(l) for i, l in zip(sc["ov_ids"], sc["ov_lens"])}
    st, rv, tv, status, sd = _ba(_slam(sc), sc)
    s2 = _slam(sc)
    lib = _lib.load()
    F, mm = sc["fids"].shape
    counts, fids = np.ascontiguousarray(sc["counts"], np.int32), np.ascontiguousarray(sc["fids"], np.int32)
    cr = np.ascontiguousarray(sc["corners"], np.float32)
    oi, ol = np.ascontiguousarray(list(ov.keys()), np.int32), np.ascontiguousarray(list(ov.values()), np.float64)
    cam = _camera(sc["K"], sc["D"])
    st2 = _lib.fid_ba_stats()
    rv2, tv2, status2 = np.zeros((F, 3)), np.zeros((F, 3)), np.zeros(F, np.int32)
    ents = s2.entries()
    sd2 = np.zeros((len(ents), 6))
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    assert lib.fid_map_bundle_adjust(s2.h, 0, F, p(counts), p(fids), p(cr), mm, C.byref(cam), float(sc["fiducial_len"]), len(oi), p(oi), p(ol), None, C.byref(st2),
                                     p(rv2), p(tv2), p(status2), p(sd2)) == 0
    assert rv.tobytes() == rv2.tobytes() and tv.tobytes() == tv2.tobytes() and status.tobytes() == status2.tobytes()
    assert np.array([sd[e.fiducial_id] for e in ents]).tobytes() == sd2.tobytes()
    fields = [f for f, _ in _lib.fid_ba_stats._fields_ if f != "device_ms"]  # device time differs between calls
    assert [getattr(st, f) for f in fields] == [getattr(st2, f) for f in fields]


def test_caps_on_free_markers_and_observations():
    # 1 030 free markers seen: more than FID_BA_MAX_FREE
    sc = mc.as_loaded(mc.make_scene(81, n_markers=1031, n_frames=700, visible=10))
    s = _slam(sc, cap=1100)
    before = _entries(s)
    with pytest.raises(_lib.FidError) as e:
        _ba(s, sc)
    assert e.value.status == -5 and _entries(s) == before
    # 65 536 frames x 65 distinct mapped ids: 4 259 840 observations, more than FID_BA_MAX_OBS
    small = mc.as_loaded(mc.make_scene(82, n_markers=65, n_frames=4))
    s = _slam(small)
    before = _entries(s)
    big = dict(small)
    n = 65536
    big["counts"] = np.full(n, 65, np.int32)
    big["fids"] = np.ascontiguousarray(np.broadcast_to(small["ids"].astype(np.int32), (n, 65)))
    big["corners"] = np.zeros((n, 65, 4, 2), np.float32)
    with pytest.raises(_lib.FidError) as e:
        _ba(s, big)
    assert e.value.status == -5 and _entries(s) == before


def _render(sc, f, dict_id, supersample=2):
    """Frame f of the scene at its size: every visible marker warped through the homography of its projected corners, as
    synth.make_frame draws them (quiet zone of one cell)."""
    W, H = sc["size"]
    cells = synth.dictionary_info(dict_id)[0] + 2
    img = np.full((H, W), 200.0, np.float32)
    offs = (np.arange(supersample) + 0.5) / supersample - 0.5
    for j in range(sc["counts"][f]):
        quad = sc["corners"][f, j].astype(np.float64)
        bits = synth.marker_bits(dict_id, int(sc["fids"][f, j]))
        q = 1.0 / cells
        Hm = synth._homography([(0, 0), (1, 0), (1, 1), (0, 1)], quad)
        Hinv = np.linalg.inv(Hm)
        x0, x1 = max(int(quad[:, 0].min()) - 15, 0), min(int(quad[:, 0].max()) + 16, W)
        y0, y1 = max(int(quad[:, 1].min()) - 15, 0), min(int(quad[:, 1].max()) + 16, H)
        py, px = np.mgrid[y0:y1, x0:x1].astype(np.float64)
        acc, cov = np.zeros(py.shape), np.zeros(py.shape)
        for oy in offs:
            for ox in offs:
                X, Y = px + ox, py + oy
                w = Hinv[2, 0] * X + Hinv[2, 1] * Y + Hinv[2, 2]
                u = (Hinv[0, 0] * X + Hinv[0, 1] * Y + Hinv[0, 2]) / w
                v = (Hinv[1, 0] * X + Hinv[1, 1] * Y + Hinv[1, 2]) / w
                inq = (u >= -q) & (u < 1 + q) & (v >= -q) & (v < 1 + q)
                inm = (u >= 0) & (u < 1) & (v >= 0) & (v < 1)
                ci, cj = np.clip((u * cells).astype(np.int64), 0, cells - 1), np.clip((v * cells).astype(np.int64), 0, cells - 1)
                acc += np.where(inq, np.where(inm, np.where(bits[cj, ci] > 0, 235.0, 20.0), 235.0), 0.0)
                cov += inq
        a = cov / supersample ** 2
        img[y0:y1, x0:x1] = img[y0:y1, x0:x1] * (1 - a) + acc / supersample ** 2
    g = np.clip(np.rint(img + np.random.default_rng(f).normal(0, 2.0, img.shape)), 0, 255).astype(np.uint8)
    return np.repeat(g[:, :, None], 3, axis=2)


def test_end_to_end_rendered_frames_map_beats_fold_and_refine():
    """Rendered 1080p frames of a 5 x 5 ceiling grid along the lawn-mower path -> fid_detect_pose_batch -> the fold (autoInit pins
    the origin) -> fid_map_bundle_adjust.  In the origin marker's frame, the map's RMS position and rotation errors against the
    truth are lower than the fold's, and the rotation error lower than fid_map_refine's on the same messages; its position error is
    not (ratios printed and recorded in DESIGN.md f16)."""
    dict_id, flen = 7, 0.2
    sc = mc.make_scene(91, n_markers=25, n_frames=60, noise=0.0, visible=10, oblique=True, size=(1920, 1080), f=900.0, fiducial_len=flen)
    frames = np.stack([_render(sc, f, dict_id) for f in range(len(sc["counts"]))])
    det = Detector(default_params(dictionary=dict_id), 0, 1920, 1080, 8)
    counts, ids, corners, tfs = det.detect_pose_batch(frames, sc["K"], sc["D"], flen)
    assert counts.sum() >= 0.8 * sc["counts"].sum()  # oblique views of small markers: most, not all, are found
    msgs = []
    for f in range(len(counts)):
        msgs.append([tfs[f * _lib.FID_MAX_MARKERS + j] for j in range(counts[f])])
    ident = [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0]  # the camera is the base: both tf lookups succeed (updatePose needs them)
    fold = FiducialSlam(max_fiducials=64)
    fold.update_frames(counts, tfs, ident, ident)
    ref = FiducialSlam(max_fiducials=64)
    ref.update_frames(counts, tfs, ident, ident)
    ref.refine([[dict(fiducial_id=int(t.fiducial_id), translation=list(t.translation), rotation=list(t.rotation), image_error=t.image_error,
                      object_error=t.object_error, fiducial_area=t.fiducial_area) for t in m] for m in msgs])
    ba = FiducialSlam(max_fiducials=64)
    ba.update_frames(counts, tfs, ident, ident)
    st, rv, tv, status, sd = ba.bundle_adjust(counts, ids, corners, sc["K"], sc["D"], flen)
    assert st.converged == 1 and st.final_rms < 0.5
    pos = {int(i): k for k, i in enumerate(sc["ids"])}
    origin = [e.fiducial_id for e in fold.entries() if e.variance == 0.0]
    assert len(origin) == 1

    def errors(slam):
        ents = {e.fiducial_id: e for e in slam.entries()}
        keep = [i for i in ents if i in pos]
        assert len(keep) >= 10, sorted(ents)
        sub = dict(sc)
        sub["ids"] = np.array(keep)
        sub["R"] = np.array([sc["R"][pos[i]] for i in keep])
        sub["t"] = np.array([sc["t"][pos[i]] for i in keep])
        R = np.array([_R_of((0, ents[i].x, ents[i].y, ents[i].z, ents[i].rx, ents[i].ry, ents[i].rz)) for i in keep])
        t = np.array([[ents[i].x, ents[i].y, ents[i].z] for i in keep])
        return mc.map_error(sub, R, t, ref=keep.index(origin[0]))

    e_fold, e_ref, e_ba = errors(fold), errors(ref), errors(ba)
    print("map error (m, rad): fold %s, fid_map_refine %s, bundle adjustment %s; ratios ba/fold %.3f %.3f, ba/refine %.3f %.3f" %
          (e_fold, e_ref, e_ba, e_ba[0] / e_fold[0], e_ba[1] / e_fold[1], e_ba[0] / e_ref[0], e_ba[1] / e_ref[1]))
    assert e_ba[0] < e_fold[0] and e_ba[1] < e_fold[1] and e_ba[1] < e_ref[1]
    # position against fid_map_refine: not better on this scene (measured 1.24x on an H100, DESIGN.md f16), so only bounded
    assert e_ba[0] < 1.5 * e_ref[0]
