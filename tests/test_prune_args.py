"""PointFusion's pruning keywords: argument errors are raised in __init__, before any compute (no GPU needed)."""
import math

import pytest

import gradslam_b200 as gs


@pytest.mark.parametrize("kw,exc", [
    (dict(stable_confidence=1.0), ValueError),
    (dict(max_unstable_age=2), ValueError),
    (dict(stable_confidence="1", max_unstable_age=2), TypeError),
    (dict(stable_confidence=True, max_unstable_age=2), TypeError),
    (dict(stable_confidence=1.0, max_unstable_age=2.0), TypeError),
    (dict(stable_confidence=1.0, max_unstable_age=False), TypeError),
    (dict(stable_confidence=-0.5, max_unstable_age=2), ValueError),
    (dict(stable_confidence=math.nan, max_unstable_age=2), ValueError),
    (dict(stable_confidence=1.0, max_unstable_age=-1), ValueError),
])
def test_keyword_errors(kw, exc):
    with pytest.raises(exc):
        gs.PointFusion(odom="gt", device="cpu", **kw)


def test_keywords_accepted_and_off_by_default():
    slam = gs.PointFusion(odom="gt", device="cpu", stable_confidence=0, max_unstable_age=0)
    assert (slam.stable_confidence, slam.max_unstable_age) == (0, 0)
    slam = gs.PointFusion(odom="gt", device="cpu", stable_confidence=math.inf, max_unstable_age=5)
    assert slam.max_unstable_age == 5
    slam = gs.PointFusion(odom="gt", device="cpu")
    assert slam.stable_confidence is None and slam.max_unstable_age is None
    with pytest.raises(TypeError):
        gs.ICPSLAM(odom="gt", device="cpu", stable_confidence=1.0, max_unstable_age=1)
