"""Regenerate tests/golden/calib_ro_384x30.npz: cv2.calibrateCameraROExtended (OpenCV 4.13) on one seeded printed-board problem
too large to run against cv2 on every test run (384 points x 30 views, m = 1 161 rows in the reduced system; cv2 takes about a
minute on 8 CPU threads).  The inputs are stored with the result, so the fixture does not depend on the generator's cv2 calls.

    python tests/golden/make_calib_ro_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import calib_ro_cases as rc  # noqa: E402

SEED, VIEWS, GRID, SIZE, FIXED = 384, 30, (24, 16), (3840, 2160), 23  # FIXED: the top-right corner


def main():
    O, I, K, D, true = rc.make_printed_problem(SEED, VIEWS, GRID, SIZE, "mild", 0.2, (1.0, 1.004), square=0.015)
    ref = rc.cv2_calibrate_ro(O, I, SIZE, FIXED)
    np.savez_compressed(os.path.join(HERE, "calib_ro_384x30.npz"), board=O[0], img=np.stack(I), size=np.array(SIZE), fixed=FIXED, rms=ref["rms"], K=ref["K"],
                        D=ref["D"], rvecs=ref["rvecs"], tvecs=ref["tvecs"], std_int=ref["std_int"], std_ext=ref["std_ext"], pve=ref["pve"], new_obj=ref["new_obj"],
                        std_obj=ref["std_obj"])
    print("rms", ref["rms"])


if __name__ == "__main__":
    main()
