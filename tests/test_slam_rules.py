"""Host-side rules of the SLAM driver (vmap_b200.slam): which rows the tracker takes."""
from vmap_b200.slam import tracker_groups


def test_background_row_is_tracked_only_as_a_do_bg_model():
    groups = [("objects", [1, None, 0, -1, 7]), ("background", [0]), ("only_zero", [0, None])]
    assert tracker_groups(groups, do_bg=True) == [("objects", [1, None, 0, None, 7]), ("background", [0]),
                                                  ("only_zero", [0, None])]
    assert tracker_groups(groups, do_bg=False) == [("objects", [1, None, None, None, 7]), ("background", [None]),
                                                   ("only_zero", [None, None])]
