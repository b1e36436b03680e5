"""CPU: the host decisions of a sharded DetectionCollector (detect.shard_merge_plan, detect.check_same_setup), taken
from the block every rank gathers, so that every rank decides alike: the union of the added flags that gives the dict
order, the duplicate-frustum and capacity verdicts, and the construction check over a gloo group of two processes."""
import os

import numpy as np
import pytest


def test_union_of_added_flags():
    from frustum_convnet_b200.detect import shard_merge_plan
    added = np.zeros((3, 10), bool)
    added[0, [0, 1, 2]] = True
    added[1, [3, 4]] = True                    # rank 2 added nothing
    added[0, 9] = True
    got = shard_merge_plan([5, 0, 0], [8, 8, 8], added)
    assert got.dtype == bool and got.tolist() == [True] * 5 + [False] * 4 + [True]
    assert not shard_merge_plan([0, 0], [1, 1], np.zeros((2, 4), bool)).any()
    assert shard_merge_plan([3], [3], np.ones((1, 2), bool)).all()        # a group of one


def test_frustum_added_on_two_ranks():
    from frustum_convnet_b200.detect import shard_merge_plan
    added = np.zeros((3, 8), bool)
    added[0, :4] = added[1, 3:6] = added[2, 5:] = True          # frustums 3 and 5 overlap; 3 is named
    with pytest.raises(ValueError, match=r"frustum 3 was added on ranks 0 and 1;"):
        shard_merge_plan([1, 1, 1], [9, 9, 9], added)
    added = np.zeros((2, 8), bool)
    added[:, 7] = True
    with pytest.raises(ValueError, match=r"frustum 7 was added on ranks 0 and 1;"):     # before the capacity verdict
        shard_merge_plan([100, 0], [1, 1], added)


def test_capacity_overflow_names_the_rank_and_the_capacity_needed():
    from frustum_convnet_b200.detect import shard_merge_plan
    added = np.eye(3, dtype=bool)
    assert shard_merge_plan([4, 6, 0], [4, 6, 1], added).all()            # exactly at capacity
    with pytest.raises(RuntimeError, match=r"rank 1: 7 rows were produced, the capacity is 6 \(needs capacity >= 7\)"):
        shard_merge_plan([4, 7, 9], [4, 6, 1], added)


def test_setup_digests_name_every_field():
    from frustum_convnet_b200.detect import _SETUP_FIELDS, setup_digests
    base = dict(id_list=[1, 1, 2], type_list=["Car", "Car", "Car"], box2d_list=np.arange(12.0).reshape(3, 4),
                dataset="KITTI", method="nms", thresh=0.1, top_k=300)
    d0 = setup_digests(**base)
    assert len(d0) == len(_SETUP_FIELDS)
    # the same values in other containers agree: numpy ids, float64 boxes, 'top' for any method but 'nms'
    assert setup_digests(**dict(base, id_list=np.array([1, 1, 2]), box2d_list=list(np.arange(12.0)))) == d0
    assert setup_digests(**dict(base, method="top")) == setup_digests(**dict(base, method="other"))
    for field, value in (("id_list", [1, 2, 2]), ("type_list", ["Car", "Van", "Car"]),
                         ("box2d_list", np.arange(12.0).reshape(3, 4) + 0.5), ("dataset", "SUNRGBD"),
                         ("method", "top"), ("thresh", 0.25), ("top_k", 100)):
        d = setup_digests(**dict(base, **{field: value}))
        assert [f for f, a, b in zip(_SETUP_FIELDS, d0, d) if a != b] == [field], field
    d = setup_digests(**dict(base, id_list=[1, 1], type_list=["Car", "Car"], box2d_list=np.zeros((2, 4))))
    assert "num_frustums" in [f for f, a, b in zip(_SETUP_FIELDS, d0, d) if a != b]


def _setup_worker(rank, world, port, out_dir):
    import torch.distributed as dist
    from spawn_group import init_group
    from frustum_convnet_b200.detect import check_same_setup, setup_digests
    init_group(rank, world, port, "gloo")
    try:
        base = dict(id_list=[3, 3, 4], type_list=["Car"] * 3, box2d_list=np.ones((3, 4)), dataset="KITTI",
                    method="nms", thresh=0.1, top_k=300)
        got = []
        for case in ({}, {"thresh": 0.3}, {"id_list": [3, 4, 4]}):
            args = dict(base, **case) if rank == world - 1 else base
            try:
                check_same_setup(None, setup_digests(**args))
                got.append("ok")
            except ValueError as e:
                got.append(str(e))
        with open(os.path.join(out_dir, "rank%d.txt" % rank), "w") as f:
            f.write("\n".join(got))
    finally:
        dist.destroy_process_group()


def test_differing_construction_raises_the_same_error_on_every_rank(tmp_path):
    from spawn_group import run_group
    run_group(_setup_worker, 2, (str(tmp_path),), timeout=300)
    got = [open(os.path.join(tmp_path, "rank%d.txt" % r)).read().split("\n") for r in range(2)]
    assert got[0] == got[1]
    assert got[0][0] == "ok"
    assert got[0][1].startswith("DetectionCollector: rank 1 of the group was constructed with a different thresh ")
    assert "different id_list than rank 0" in got[0][2]
