"""CPU oracle for the aruco_detect + fiducial_slam hot path.

TEST INFRASTRUCTURE ONLY.  Nothing under ``fiducials_b200/`` may import this
package; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` do, and only as the checker or the
timed CPU baseline -- never as the thing shipped.

Parity pinning (see DESIGN.md section "Oracle"):
  * detect/pose: the arithmetic the reference executes at
    aruco_detect/src/aruco_detect.cpp:350 (cv::aruco::detectMarkers), :247
    (cv::solvePnP) and :210 (cv::projectPoints) lives in OpenCV, which is not
    vendored in the reference checkout.  ``aruco_oracle`` drives the OpenCV 4.13 wheel
    of this image (``cv2``) with the reference's parameters
    (aruco_detect.cpp:690-727) and restates the node's own glue arithmetic
    (aruco_detect.cpp:151-221, 447-495).  It is pinned against the reference's
    golden corner vectors (aruco_detect/test/aruco_images_test.cpp:96-109,
    125-147), the 403 map-entry golden
    (fiducial_slam/test/auto_init_403_test.cpp:119-137) and the golden
    FiducialTransformArray inside fiducial_slam/test/aruco_transforms.bag by
    tests/test_oracle_golden.py.
  * map update: ``slam_oracle`` is a numpy/pure-python restatement of
    fiducial_slam/src/map.cpp and transform_with_variance.cpp with tf2
    LinearMath semantics (tf2 is not vendored either), pinned against
    fiducial_slam/test/create_map_aruco.xml:26-33 and the 403 golden.
"""
