"""CPU tests: the stream ids a fleet's remove_streams accepts (scoring.fleet_removal), and the old -> new id map."""
import numpy as np
import pytest


def test_removal_map_renumbers_the_survivors():
    from mtad_gat_pytorch_b200.scoring import fleet_removal
    keep, mapping = fleet_removal([0, 2], 5, "remove")
    assert keep.tolist() == [1, 3, 4] and mapping.tolist() == [-1, 0, -1, 1, 2]
    keep, mapping = fleet_removal(np.array([4, 1], np.int32), 5, "remove")          # any order, any integer dtype
    assert keep.tolist() == [0, 2, 3] and mapping.tolist() == [0, -1, 1, 2, -1]
    assert fleet_removal(3, 5, "remove")[1].tolist() == [0, 1, 2, -1, 3]


@pytest.mark.parametrize("ids", [[5], [-1], [1, 1], [0.0], [True], [], "a", [[0], [1]], [0, 1, 2, 3, 4]])
def test_removal_refuses_bad_ids(ids):
    from mtad_gat_pytorch_b200.scoring import fleet_removal
    with pytest.raises(ValueError, match="^remove: "):
        fleet_removal(ids, 5, "remove")
