"""Opt-in device paths that were written after the round's GPU budget was spent and have therefore never run on a GPU.  The file
sorts last on purpose: whatever these tests do, every other GPU test has already run.  Non-strict xfail: a pass is reported
as XPASS, a failure does not fail the suite."""
import numpy as np
import pytest

from fiducials_b200 import synth
from oracle import aruco_oracle as ao

pytestmark = pytest.mark.gpu


@pytest.mark.xfail(strict=False, reason="opt-in path (FID_START_PRUNE=1): proven on the CPU harness; not a default, so a failure here does not fail the suite")
def test_opt_in_start_prune_table_keeps_results(monkeypatch):
    """Table stage of the start pruning (start_prune_table.h; tests/test_hostsim_contours.py proves it on the CPU): identical quad
    candidates and detections with a third of the start cracks gone."""
    from fiducials_b200.node import Detector, default_params

    W, H, n, d = synth.CONFIGS["C3"]
    bgr = synth.make_config_frame("C3", 2)[0]
    base = Detector(default_params(dictionary=d), 0, W, H, 1)
    ids0, c0 = base.detect(bgr)
    starts0 = base.last_counters()["start_cracks"]
    base.close()
    monkeypatch.setenv("FID_START_PRUNE", "1")
    det = Detector(default_params(dictionary=d), 0, W, H, 1)
    ids1, c1 = det.detect(bgr)
    starts1 = det.last_counters()["start_cracks"]
    det.close()
    assert ids0.tolist() == ids1.tolist() and np.array_equal(c0, c1)
    rids, rc = ao.detect(bgr, d)
    assert ids1.tolist() == rids.tolist() and np.abs(c1 - rc).max() <= 1e-3
    assert starts1 < 0.8 * starts0
