"""mcl3dl_kernel_launches over one call of the map build, the incremental map append and scan preparation: one per
kernel launch and one per device-wide CUB call (include/mcl3dl_b200.h).  Each expected count is a sum with one term per
launch or CUB call the path makes, in the order engine.cu makes them."""
import numpy as np
import pytest

from mcl_3dl_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng_mod():
    from mcl_3dl_b200 import engine
    engine.load_library()
    return engine


def launches(e, fn):
    n0 = e.kernel_launches()
    out = fn()
    return e.kernel_launches() - n0, out


def map_params(eng_mod):
    return (eng_mod.LikParams(dist_weight=(1, 1, 5)),
            eng_mod.beam_params_from_reference(num_points_default=8, dda_grid_size=0.2, use_raycast_using_dda=True))


# voxel_grid: scan_bbox_kernel, scan_key_kernel, SortPairs, SortKeys, scan_heads_kernel, ExclusiveSum, scan_centroid_kernel
VOXEL_GRID = 1 + 1 + 1 + 1 + 1 + 1 + 1
# the rest of scan preparation with both sampled scans non-empty: scan_clip_flags_kernel, ExclusiveSum (likelihood clip),
# ExclusiveSum (beam clip), scan_compact_kernel x 2, scan_sample_kernel x 2
CLIP_AND_SAMPLE = 1 + 1 + 1 + 2 + 2


@pytest.mark.parametrize("downsample,want", [((0.3, 0.3, 0.3), VOXEL_GRID + CLIP_AND_SAMPLE), ((0.0, 0.0, 0.0), CLIP_AND_SAMPLE)])
def test_scan_prepare(eng_mod, downsample, want):
    rng = np.random.default_rng(5)
    raw = synth.make_points(rng.uniform([-3, -3, -1], [3, 3, 1], (5000, 3)).astype(np.float32), rng.integers(0, 2, 5000))
    e = eng_mod.Engine((0,))
    sp = eng_mod.ScanParams(downsample=downsample, lik_num_points=96, beam_num_points=6, seed=3)
    n, info = launches(e, lambda: e.scan_prepare(raw, sp))
    e.close()
    assert info["n_lik"] == 96 and info["n_beam"] == 6
    assert (info["n_downsampled"] < len(raw)) == (downsample[0] > 0)
    assert n == want


# build_map_on_device's grids other than the NN field, with a likelihood and a DDA beam model
BBOX = 1                          # bbox_kernel
NN_CSR = 1 + 1 + 1 + 1            # nn_key_kernel, SortPairs, InclusiveSum, nn_gather_kernel
NEAR_LIK = 1                      # near_mark_kernel of the likelihood screen (k = 2)
DDA = 1 + 1 + 1 + 1               # dda_key_kernel, SortPairs, InclusiveSum, dda_gather_kernel


@pytest.fixture(scope="module")
def world():
    s = synth.scene(50_000, 1, 0, 0, seed=41)
    return s["map"]


def test_set_map_with_the_nn_field(eng_mod, world):
    e = eng_mod.Engine((0,))
    n, _ = launches(e, lambda: e.set_map(world, *map_params(eng_mod)))
    assert e.near_field_info()[0][0] == 2 and e.nn_field_info()["bytes"] > 0
    e.close()
    # build_nn_field: near_mark_kernel, nnf_count_kernel, DeviceReduce::Sum, DeviceScan::ExclusiveSum, nnf_base_kernel,
    # nnf_fill_kernel (no nn_row3_kernel: the field is staged)
    nn_field = 1 + 1 + 1 + 1 + 1 + 1
    assert n == BBOX + NN_CSR + NEAR_LIK + nn_field + DDA


def test_incremental_map_append_that_reselects_cells(eng_mod, world):
    e = eng_mod.Engine((0,))
    e.set_map(world, *map_params(eng_mod))
    xyz = np.stack([world["x"], world["y"], world["z"]], axis=1)
    lo, hi = xyz.min(0), xyz.max(0)
    inner = xyz[np.all((xyz > lo + 0.2 * (hi - lo)) & (xyz < hi - 0.2 * (hi - lo)), axis=1)][:300]
    patch = synth.make_points(inner + np.float32(0.01))  # inside both bounding boxes: every lattice stays
    n, info = launches(e, lambda: e.map_append(patch))
    e.close()
    assert info["incremental"] == 1 and info["cells_reselected"] > 0
    # update_nn_field: near_mark_kernel, nnf_mark_kernel, then over the marked cells nnf_count_kernel,
    # DeviceReduce::Sum, DeviceScan::ExclusiveSum, nnf_base_kernel, nnf_fill_kernel
    nn_field = 1 + 1 + 1 + 1 + 1 + 1 + 1
    assert n == BBOX + NN_CSR + NEAR_LIK + nn_field + DDA
