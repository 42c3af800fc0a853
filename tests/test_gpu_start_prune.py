"""Table stage of the start-crack pruning (FID_START_PRUNE=1, start_prune_table.h) on the device, strict.  It is off by default
because on H100 it costs the threshold kernel more than it saves the border walk (DESIGN.md section 4); it must still be exact."""
import numpy as np
import pytest

from fiducials_b200 import synth
from oracle import aruco_oracle as ao

pytestmark = pytest.mark.gpu


def test_start_prune_table_keeps_candidates_and_detections(monkeypatch):
    """Identical quad candidates and detections with and without the table stage, equal to the oracle's, with a third of the start
    cracks gone (tests/test_hostsim_contours.py proves the same on the CPU harness)."""
    from fiducials_b200.node import Detector, default_params

    W, H, n, d = synth.CONFIGS["C3"]
    bgr = synth.make_config_frame("C3", 2)[0]
    runs = []
    for prune in ("0", "1"):
        monkeypatch.setenv("FID_START_PRUNE", prune)  # read by fid_create
        det = Detector(default_params(dictionary=d), 0, W, H, 1)
        try:
            ids, corners = det.detect(bgr)
            starts = det.last_counters()["start_cracks"]
            cands = det.debug_candidates()
        finally:
            det.close()
        runs.append((ids, corners, starts, cands))
    (ids0, c0, starts0, cands0), (ids1, c1, starts1, cands1) = runs
    assert ids0.tolist() == ids1.tolist() and np.array_equal(c0, c1)
    assert all(np.array_equal(a, b) for a, b in zip(cands0, cands1))
    rids, rc = ao.detect(bgr, d)
    assert ids1.tolist() == rids.tolist() and len(ids1) > 0 and np.abs(c1 - rc).max() <= 1e-3
    assert starts1 < 0.8 * starts0, (starts0, starts1)
