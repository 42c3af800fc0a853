#!/usr/bin/env python
"""Lift the reference's own test fixtures into committed golden vectors, so that the tests run without
the reference checkout:  python tests/golden/make_golden.py <reference checkout>

Inputs (all under the reference checkout, read-only):
  aruco_detect/test/test_images/tag_01_d7_14cm.png, tag_245-246_d7_14cm.png  (aruco_images_test.cpp)
  fiducial_slam/test/test_images/403.jpg                                    (auto_init_403_test.cpp)
  fiducial_slam/test/aruco_images.bag      (one 1280x960 JPEG frame + CameraInfo)
  fiducial_slam/test/aruco_transforms.bag  (the golden FiducialTransformArray for that frame)

Output: per frame, the decoded BGR8 pixels (decoded exactly as the reference tests do,
cv::imread(IMREAD_COLOR) / cv_bridge BGR8) as two lossless WebP halves, tests/golden/frames/<name>_top.webp
and <name>_bottom.webp (each file stays well under 1 MB), and tests/golden/reference_kat.npz with the
camera K/D, dictionary, fiducial_len and the cv2-4.13 oracle's outputs (oracle/aruco_oracle.py).

The answers of the reference's compiled Map (tests/golden/map_ref/*.npz) are recorded separately, where
oracle/_ref/libmap_ref.so was built:  FID_RECORD_MAP_REF=1 python -m pytest tests/test_map_ref.py, and
oracle.map_ref.use_tape(tests.test_gpu_slam.MAP_REF_TAPE) around tests.test_gpu_slam.c5_reference_answers().
"""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import aruco_oracle as ao  # noqa: E402
from oracle import rosbag_lite as rb  # noqa: E402

# aruco_detect/test/aruco_images_test.cpp:24-27
TEST_K = [1006.126285753055, 0.0, 655.8639244150409, 0.0, 1004.015433012594, 490.6140221242933, 0.0, 0.0, 1.0]
TEST_D = [0.1349735087283542, -0.2335869827451621, 0.0006697030315075139, 0.004846737465872353, 0.0]


def pack(out, name, bgr, K, D, dict_id, flen):
    h = bgr.shape[0] // 2
    for part, pixels in (("top", bgr[:h]), ("bottom", bgr[h:])):
        ok, webp = cv2.imencode(".webp", np.ascontiguousarray(pixels), [cv2.IMWRITE_WEBP_QUALITY, 101])  # quality > 100: lossless
        assert ok and np.array_equal(cv2.imdecode(webp, cv2.IMREAD_COLOR), pixels)
        with open(os.path.join(ROOT, "tests/golden/frames", "%s_%s.webp" % (name, part)), "wb") as f:
            f.write(webp.tobytes())
    ids, corners, rvecs, tvecs, fields = ao.detect_and_pose(bgr, dict_id, K, D, flen)
    out[name + "_K"] = np.array(K, np.float64)
    out[name + "_D"] = np.array(D, np.float64)
    out[name + "_dict"] = np.array(dict_id)
    out[name + "_len"] = np.array(flen)
    out[name + "_ids"] = ids
    out[name + "_corners"] = corners
    out[name + "_rvecs"] = rvecs
    out[name + "_tvecs"] = tvecs
    out[name + "_quat"] = np.array([f["rotation"] for f in fields]).reshape(-1, 4)
    out[name + "_errs"] = np.array([[f["image_error"], f["object_error"], f["fiducial_area"]] for f in fields]).reshape(-1, 3)
    print(name, bgr.shape, "ids", ids.tolist())


def main(ref):
    out = {}
    os.makedirs(os.path.join(ROOT, "tests/golden/frames"), exist_ok=True)
    for name, rel, flen in [
        ("tag01", "aruco_detect/test/test_images/tag_01_d7_14cm.png", 0.145),
        ("tag245", "aruco_detect/test/test_images/tag_245-246_d7_14cm.png", 0.145),
        ("img403", "fiducial_slam/test/test_images/403.jpg", 0.145),
    ]:
        bgr = cv2.imread(os.path.join(ref, rel), cv2.IMREAD_COLOR)
        pack(out, name, bgr, TEST_K, TEST_D, 7, flen)
    # bag pair
    cam = None
    frame = None
    for topic, typ, raw in rb.read_bag(os.path.join(ref, "fiducial_slam/test/aruco_images.bag")):
        if typ == "sensor_msgs/CameraInfo" and cam is None:
            cam = rb.parse_camera_info(raw)
        elif typ == "sensor_msgs/CompressedImage":
            ci = rb.parse_compressed_image(raw)
            frame = cv2.imdecode(np.frombuffer(ci["data"], np.uint8), cv2.IMREAD_COLOR)
            out["bag_image_seq"] = np.array(ci["header"]["seq"])
    pack(out, "bag", frame, cam["K"], cam["D"][:5], 7, 0.14)
    msgs = rb.read_bag(os.path.join(ref, "fiducial_slam/test/aruco_transforms.bag"))
    assert len(msgs) == 1
    fta = rb.parse_fiducial_transform_array(msgs[0][2])
    out["bag_golden_ids"] = np.array([t["fiducial_id"] for t in fta["transforms"]], np.int32)
    out["bag_golden_t"] = np.array([t["translation"] for t in fta["transforms"]])
    out["bag_golden_q"] = np.array([t["rotation"] for t in fta["transforms"]])
    out["bag_golden_errs"] = np.array([[t["image_error"], t["object_error"], t["fiducial_area"]] for t in fta["transforms"]])
    out["bag_golden_image_seq"] = np.array(fta["image_seq"])
    print("bag golden ids", out["bag_golden_ids"].tolist(), "frame", fta["header"]["frame_id"], "image_seq", fta["image_seq"])
    np.savez(os.path.join(ROOT, "tests/golden/reference_kat.npz"), **out)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        raise SystemExit(__doc__)
    main(sys.argv[1])
