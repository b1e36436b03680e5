"""GPU: a DetectionCollector over a process group (detect.py, ``group=``).  Every rank adds its shard_slice chunk of
every batch; each rank's merged ``finalize_device()`` must equal, bit for bit, one single-process collector that added
every rank's chunks (rows, segment offsets, keep counts, dict order, ``to_dict()``), and so must what the evaluators and
the refinement extractor make of it.  The errors of a sharded pass (a frustum added on two ranks, a rank over its
capacity, ranks constructed differently) must raise the same message on every rank and leave the group usable.

gloo groups of 2 and 3 processes share one GPU; the NCCL group needs one GPU per rank and is skipped on fewer than 2."""
import os
import pickle
import traceback

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR
from det_shard_sets import add_shard, rebatch, recorded_pass

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ inputs
def _golden_pass(name, dataset, run):
    from oracle.make_golden_detect import batches
    from test_detect_cpu import fixture_runs
    from test_gpu_detect import _cuda_batches
    g = dict(np.load(os.path.join(GOLDEN_DIR, "detect_%s.npz" % name)))
    ids, types = [int(i) for i in g["id_list"]], [str(t) for t in g["type_list"]]
    method, use_ref, use_rgb, _ = fixture_runs(g)[run]
    ctor = ((ids, types, g["box2d"]), dict(dataset=dataset, method=method, thresh=float(g["thresh"])))
    return ctor, [(outs, d, first) for first, outs, d in _cuda_batches(batches(g, use_ref, use_rgb))]


def _random_pass(seed, method, **kw):
    """Lists of 1, 513 and 1680 rows (test_gpu_detect._random_case) in batches of 5 over 22 frustums."""
    from test_gpu_detect import _cuda_batches, _random_case
    bt, ids, types, box2d = _random_case(seed)
    ctor = ((ids, types, box2d), dict(dataset="KITTI", method=method, thresh=0.25, **kw))
    return ctor, [(outs, d, first) for first, outs, d in _cuda_batches(bt)]


# ------------------------------------------------------------------------------------------------ one pass
def _merged_and_single(pg, dev, rank, world, ctor, adds, owner=None):
    """-> (this rank's merged result, a single collector's result over every rank's chunks)."""
    from frustum_convnet_b200.detect import DetectionCollector
    (args, kw) = ctor
    kw = dict(kw, device=dev)
    col = DetectionCollector(*args, group=pg, **kw)
    add_shard(col, adds, rank, world, owner)
    merged = col.finalize_device()
    one = DetectionCollector(*args, **kw)
    for r in range(world):
        add_shard(one, adds, r, world, owner)
    return merged, one.finalize_device()


def _check_identical(a, b):
    assert a.num_rows == b.num_rows and a.num_segments == b.num_segments
    assert torch.equal(a.seg_offsets, b.seg_offsets) and torch.equal(a.keep_count, b.keep_count)
    assert np.array_equal(a.host_seg_offsets, b.host_seg_offsets)
    assert np.array_equal(a.host_keep_count, b.host_keep_count)
    # the kept rows: under 'nms' a segment's rows past its keep count are never written
    kept = np.concatenate([np.arange(o, o + k) for o, k in zip(b.host_seg_offsets[:-1], b.host_keep_count)] +
                          [np.zeros(0, np.int64)])
    kept = torch.from_numpy(kept.astype(np.int64)).to(b.rows.device)
    assert torch.equal(a.rows[kept].view(torch.int32), b.rows[kept].view(torch.int32))
    assert np.array_equal(a.order, b.order) and a.segments == b.segments
    da, db = a.to_dict(), b.to_dict()
    assert list(da) == list(db)
    for i in db:
        assert list(da[i]) == list(db[i]), i
        for c in db[i]:
            assert da[i][c].tobytes() == db[i][c].tobytes(), (i, c)


def _check_kitti(a, b):
    assert a.evaluated == b.evaluated
    for m in b.precision:
        assert a.precision[m].keys() == b.precision[m].keys()
        for c in b.precision[m]:
            assert a.precision[m][c].tobytes() == b.precision[m][c].tobytes(), (m, c)
            assert np.array_equal(a.ap[m][c], b.ap[m][c]) and np.array_equal(a.n_gt[m][c], b.n_gt[m][c])
    assert a.aos.keys() == b.aos.keys() and all(a.aos[c].tobytes() == b.aos[c].tobytes() for c in b.aos)
    assert a.lines() == b.lines()


def _check_sunrgbd(a, b):
    assert a.classes == b.classes and a.nd == b.nd and a.npos == b.npos
    for c in b.classes:
        assert a.rec[c].tobytes() == b.rec[c].tobytes() and a.prec[c].tobytes() == b.prec[c].tobytes(), c
        assert a.ap[c] == b.ap[c], c


def _check_refine(a, b):
    assert len(a) == len(b) and np.array_equal(a.job_index, b.job_index) and np.array_equal(a.counts, b.counts)
    assert a.id_list == b.id_list and a.type_list == b.type_list
    for n in ("points", "offsets", "lists", "frustum_records", "record_words"):
        assert torch.equal(getattr(a, n), getattr(b, n)), n
    assert (a.label is None) == (b.label is None) and (a.label is None or torch.equal(a.label, b.label))


# ------------------------------------------------------------------------------------------------ the cases
def _cases(pg, dev, rank, world):
    """(name, fn) pairs run in order on every rank; fn raises on a mismatch, or returns None or the string every rank
    must agree on (the error a sharded pass raised; "counts": this rank's rows)."""
    from det_feed_sets import collector_for, kitti_set
    from frustum_convnet_b200 import refine_extract as rx
    from frustum_convnet_b200.detect import DetectionCollector
    from test_gpu_det_eval_feed import _sun_set, kitti_gt, sun_gt
    from test_gpu_refine_cascade import _scene

    def same(ctor, adds, owner=None):
        def run():
            _check_identical(*_merged_and_single(pg, dev, rank, world, ctor, adds, owner))
        return run

    def error(ctor, adds, *, dup=False, thresh=None, ids=None):
        def run():
            (args, kw) = ctor
            if rank == world - 1 and thresh is not None:
                kw = dict(kw, thresh=thresh)
            if rank == world - 1 and ids is not None:
                args = (ids,) + tuple(args[1:])
            try:
                col = DetectionCollector(*args, group=pg, **dict(kw, device=dev))
                if dup:                                  # ranks 0 and 1 both add the first batch
                    if rank < 2:
                        outs, d, first = adds[0]
                        col.add(outs, d, first=first)
                else:
                    add_shard(col, adds, rank, world)
                col.finalize_device()
            except (ValueError, RuntimeError) as e:
                return "%s: %s" % (type(e).__name__, e)
            return "no error"
        return run

    def kitti():
        gts, dets = kitti_set(300, seed=7)
        (ctor, adds), _ = recorded_pass(lambda: collector_for(dets, "KITTI", device=dev))
        merged, one = _merged_and_single(pg, dev, rank, world, ctor, rebatch(adds, 32))
        _check_identical(merged, one)
        ev = kitti_gt(list(range(len(gts))), gts)
        _check_kitti(ev.evaluate_collected(merged), ev.evaluate_collected(one))

    def sunrgbd():
        classes, gt_rows, gt_ids, dets = _sun_set(300, 11, True)
        (ctor, adds), _ = recorded_pass(lambda: collector_for(dets, "SUNRGBD", device=dev))
        merged, one = _merged_and_single(pg, dev, rank, world, ctor, rebatch(adds, 32))
        _check_identical(merged, one)
        ev = sun_gt(gt_rows, gt_ids, classes)
        _check_sunrgbd(ev.evaluate_collected(merged), ev.evaluate_collected(one))

    def refine():
        (ctor, adds), (scans, calibs, hws, ids, gt, _) = recorded_pass(lambda: _scene(31, n_frames=6))
        merged, one = _merged_and_single(pg, dev, rank, world, ctor, rebatch(adds, 4))
        _check_identical(merged, one)
        x = rx.RefineFrustumExtractor(("Car", "Pedestrian", "Cyclist"))
        a, b = x.from_collected(scans, calibs, hws, ids, merged), x.from_collected(scans, calibs, hws, ids, one)
        assert len(b) > 0
        _check_refine(a, b)
        _check_refine(x.from_matched_collected(scans, calibs, hws, ids, merged, gt, remove_diff=True),
                      x.from_matched_collected(scans, calibs, hws, ids, one, gt, remove_diff=True))

    def no_rows():
        (ctor, adds), _ = recorded_pass(lambda: collector_for({7: {"Car": np.zeros((3, 12), np.float32)}}, "KITTI",
                                                          device=dev))
        merged, one = _merged_and_single(pg, dev, rank, world, ctor, rebatch(adds, 1))
        assert merged.num_rows == 0 and len(merged.order) == 1
        _check_identical(merged, one)

    def counts():
        """this rank's rows of the capacity case: the message must name the first rank over 100."""
        (args, kw), adds = _random_pass(5, "nms")
        col = DetectionCollector(*args, **dict(kw, device=dev))
        add_shard(col, adds, rank, world)
        torch.cuda.synchronize()
        return str(int(col.counter.item()))

    cases = []
    for name, dataset in (("kitti", "KITTI"), ("sunrgbd", "SUNRGBD")):
        for run in range(4):
            cases.append(("golden_%s_%d" % (name, run), same(*_golden_pass(name, dataset, run))))
    for method in ("nms", "top"):
        cases.append(("random_%s" % method, same(*_random_pass(5, method))))
    cases.append(("one_rank_adds_everything", same(*_random_pass(6, "nms"), owner=0)))
    cases.append(("last_rank_adds_everything", same(*_random_pass(6, "top"), owner=world - 1)))
    cases += [("no_rows", no_rows), ("kitti_ap", kitti), ("sunrgbd_ap", sunrgbd), ("refine", refine)]
    rp = _random_pass(5, "nms")
    cases += [("err_duplicate", error(*rp, dup=True)),
              ("err_capacity", error(*_random_pass(5, "nms", capacity=100))), ("counts", counts),
              ("err_thresh", error(*rp, thresh=0.3)),
              ("err_id_list", error(*rp, ids=list(rp[0][0][0][1:]) + [99])),
              ("after_errors", same(*rp))]
    return cases


def _worker(rank, world, port, backend, out_dir):
    import torch.distributed as dist
    from spawn_group import init_group
    dev = torch.device("cuda", rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    init_group(rank, world, port, backend, **({"device_id": dev} if backend == "nccl" else {}))
    got = {}
    try:
        for name, fn in _cases(dist.group.WORLD, dev, rank, world):
            try:
                got[name] = fn()
            except Exception:
                got[name] = "FAILED " + traceback.format_exc()
    finally:
        with open(os.path.join(out_dir, "rank%d.pkl" % rank), "wb") as f:
            pickle.dump(got, f)
        dist.destroy_process_group()


def _run(backend, world, tmp_path):
    from spawn_group import run_group
    run_group(_worker, world, (backend, str(tmp_path)), timeout=900)
    got = [pickle.load(open(os.path.join(tmp_path, "rank%d.pkl" % r), "rb")) for r in range(world)]
    failed = ["rank %d %s: %s" % (r, k, v) for r in range(world) for k, v in got[r].items()
              if isinstance(v, str) and v.startswith("FAILED")]
    assert not failed, "\n".join(failed)
    names = list(got[0])
    assert "after_errors" in names and all(list(g) == names for g in got)
    for k in names:
        assert all(g[k] == got[0][k] for g in got) or k == "counts", (k, [g[k] for g in got])
    r = got[0]
    assert r["err_duplicate"].startswith("ValueError: DetectionCollector: frustum 0 was added on ranks 0 and 1;")
    over = [(q, int(g["counts"])) for q, g in enumerate(got) if int(g["counts"]) > 100]
    assert over, "no rank overflowed"
    assert r["err_capacity"] == ("RuntimeError: DetectionCollector: record capacity exceeded on rank %d: %d rows were "
                                 "produced, the capacity is 100 (needs capacity >= %d)" % (over[0] + over[0][1:]))
    assert r["err_thresh"].startswith("ValueError: DetectionCollector: rank %d of the group was constructed with a "
                                      "different thresh than rank 0" % (world - 1))
    assert "rank %d of the group was constructed with a different id_list than rank 0" % (world - 1) in r["err_id_list"]


@pytest.mark.parametrize("world", [2, 3])
def test_gloo_ranks_on_one_gpu(world, tmp_path):
    _run("gloo", world, tmp_path)


def test_nccl_one_gpu_per_rank(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    _run("nccl", 2, tmp_path)
