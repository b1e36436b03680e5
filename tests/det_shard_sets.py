"""Detection passes that several ranks share: a pass is a DetectionCollector's constructor arguments and its adds,
recorded from any helper that builds and fills a collector (det_feed_sets.collector_for, ...), which each rank then
replays on its chunk of every batch."""
import contextlib


@contextlib.contextmanager
def _recording():
    """Collectors made inside the block remember their constructor arguments and their adds."""
    from frustum_convnet_b200 import detect
    made, base = [], detect.DetectionCollector

    class Recorder(base):
        def __init__(self, *args, **kw):
            super().__init__(*args, **kw)
            self.ctor, self.adds = (args, kw), []
            made.append(self)

        def add(self, outputs, data_dicts, first):
            super().add(outputs, data_dicts, first)
            self.adds.append((outputs, data_dicts, first))

    detect.DetectionCollector = Recorder
    try:
        yield made
    finally:
        detect.DetectionCollector = base


def recorded_pass(make):
    """make() builds and fills one collector -> ((constructor (args, kwargs), adds [(outputs, data_dicts, first)]),
    make's result)."""
    with _recording() as made:
        res = make()
    col = made[-1]
    return (col.ctor, col.adds), res


def rebatch(adds, batch):
    """The same adds cut into batches of `batch` frustums."""
    out = []
    for outs, d, first in adds:
        B = int(outs[0].shape[0])
        for lo in range(0, B, batch):
            hi = min(B, lo + batch)
            out.append((tuple(o[lo:hi] for o in outs), {k: v[lo:hi] for k, v in d.items()}, first + lo))
    return out


def add_shard(col, adds, rank, world, owner=None):
    """Add rank's shard_slice chunk of every batch (owner: that rank takes every batch whole, the others nothing)."""
    from frustum_convnet_b200.sharding import shard_slice
    for outs, d, first in adds:
        B = int(outs[0].shape[0])
        if owner is None:
            sl = shard_slice(B, rank, world)
        else:
            sl = slice(0, B) if rank == owner else slice(B, B)
        col.add(tuple(o[sl] for o in outs), {k: v[sl] for k, v in d.items()}, first=first + sl.start)
