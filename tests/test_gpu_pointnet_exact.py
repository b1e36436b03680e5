"""GPU: fcn_pointnet_tiles called directly, compared BIT-EXACTLY with the float64 reference of tests/exact_ref.py.

Integer operands keep every partial sum exact (R1: TF32 rounding is the identity; R2: the layer outputs really
round, ties included), so any difference is a kernel bug, not rounding.  The cases choose what the workload
fixtures leave to chance: section boundaries at every row offset (rows 8 / 16 / 64 / 128 of a warp half, warp,
warpgroup and tile), sections split across tiles, every row of a short section being the arg-max of some
channel, all-negative and empty sections, partial tiles with NaN in the unused record slots, b > 0,
feat_pitch > T and ld_feat > C3 with sentinels that must survive, decoy tiles past the device tile count,
a single tile, an odd tile count on 2-CTA clusters and enough tiles for >= 3 rounds per CTA."""
import ctypes as C

import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

CONFIGS = [(64, 64, 128), (128, 128, 256), (256, 256, 512)]
# (precision, regime, tile rows); precision 2 = 2-CTA clusters (streamed-weight configs only), 0 = fp32 SIMT
MODES = [(1, "R1", 128), (1, "R2", 128), (2, "R1", 128), (2, "R2", 128), (0, "R1", 64)]
EDGE_LENGTHS = list(range(1, 21)) + [31, 32, 33, 63, 64, 65, 127, 128, 129, 200]


def dev():
    return torch.device("cuda:0")


def _cuts(tile_rows):
    if tile_rows == 128:
        return (128, 127, 65, 128, 64, 63, 9, 8, 7, 1, 128)
    return (64, 63, 9, 8, 7, 1, 64, 33)


def _edge_frustums(seed):
    """Three frustums with the edge lengths end to end (ascending, shuffled, descending), all-negative and
    empty sections between them."""
    g = torch.Generator().manual_seed(seed)
    pos = [(n, "pos") for n in EDGE_LENGTHS]
    extra = [(5, "neg"), (0, "pos"), (17, "neg"), (1, "neg")]
    a = pos[:10] + extra[:2] + pos[10:] + extra[2:]
    perm = torch.randperm(len(a), generator=g).tolist()
    return [a, [a[i] for i in perm], a[::-1]]


def run(case, precision):
    from frustum_convnet_b200 import _lib
    d = X.pointnet_device_weights(case.W, dev())
    d["rows"] = case.rows.to(dev())
    d["tiles"] = case.tiles.to(dev())
    d["ntiles"] = torch.tensor([case.ntiles], dtype=torch.int32, device=dev())
    d["out"] = case.feat_init.to(dev())
    a = X.pointnet_args(case, d, precision)
    _lib.call("fcn_pointnet_tiles", C.byref(a), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d["out"].cpu()


def check(case, precision, what):
    got = run(case, precision)
    exp = X.pointnet_pooled_ref(case)
    assert X.bits_equal(got, exp), "%s:\n%s" % (what, X.describe_mismatch(got, exp))


def _modes(dims):
    return [m for m in MODES if not (m[0] == 2 and dims[0] < 128)]


PARAMS = [pytest.param(dims, *m, id="%d-%d-%d-p%d-%s" % (dims + m[:2])) for dims in CONFIGS for m in _modes(dims)]


@pytest.mark.parametrize("dims,precision,regime,tile_rows", PARAMS)
def test_pointnet_sections_and_tiles_exact(dims, precision, regime, tile_rows):
    W = X.make_pointnet_weights(*dims, regime, seed=sum(dims) + len(regime))
    case = X.make_pointnet_case(W, _edge_frustums(1), tile_rows, _cuts(tile_rows), seed=2)
    if precision == 2 and case.ntiles % 2 == 0:          # a rank without a tile in the last unit
        case = X.make_pointnet_case(W, _edge_frustums(1) + [[(3, "pos")]], tile_rows, _cuts(tile_rows), seed=2)
    assert precision != 2 or case.ntiles % 2 == 1
    check(case, precision, "edge sections")


@pytest.mark.parametrize("dims,precision,regime,tile_rows", PARAMS)
def test_pointnet_single_tile_exact(dims, precision, regime, tile_rows):
    """ntiles = 1 (tile of 9 rows: one row past the first 8-row half), decoys past it."""
    W = X.make_pointnet_weights(*dims, regime, seed=7 + sum(dims))
    case = X.make_pointnet_case(W, [[(4, "pos"), (5, "pos")]], tile_rows, (tile_rows,), seed=3)
    assert case.ntiles == 1
    check(case, precision, "single tile")


@pytest.mark.parametrize("dims,precision,regime,tile_rows",
                         [p for p in PARAMS if p.values[2] == "R1"])
def test_pointnet_many_rounds_exact(dims, precision, regime, tile_rows):
    """>= 3 tiles per persistent CTA slot: the streamed weight ring wraps its phase many times."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = 2 if (dims[0] <= 64 and precision != 0) else 1
    need = 3 * sms * ctas + 7
    W = X.make_pointnet_weights(*dims, regime, seed=11 + sum(dims))
    g = torch.Generator().manual_seed(12)
    frustums = []
    rows = 0
    while rows < need * tile_rows:
        secs = [(int(n), "pos") for n in torch.randint(1, 70, (40,), generator=g)]
        frustums.append(secs)
        rows += sum(n for n, _ in secs)
    case = X.make_pointnet_case(W, frustums, tile_rows, (tile_rows, tile_rows, tile_rows - 1, 17), seed=13,
                                ensure_argmax=False)
    assert case.ntiles >= 3 * sms * ctas
    check(case, precision, "%d tiles" % case.ntiles)
