"""-m gpu: the three streaming-ring rasterizers (whole sorted store, segment table in parameters, culled device table) share one
body; one seeded store drawn through each of them gives the same level-0 z-buffer bit for bit, at every ring depth
("raster_stages") and for both register budgets of the whole-store kernel ("raster_occupancy" 4 selects the 56-register build)."""
import pytest
import torch

from read_b200 import _lib as L
from read_b200 import ops, synth

pytestmark = pytest.mark.gpu
N, W, H, LEVELS = 3_000_001, 512, 256, 4         # ~2930 chunks: several per CTA, so the ring wraps; the last chunk is partial


@pytest.fixture(scope="module")
def scene():
    d = torch.device("cuda", 0)
    xyz = torch.from_numpy(synth.street_scene(N, seed=11)).to(d)
    return ops.SortedPoints(xyz), ops.SegmentedPoints([(xyz, torch.arange(N, device=d))])


def _level0(B, draw):
    pyr = ops.Pyramid(B, W, H, LEVELS, torch.device("cuda", 0))
    pyr.clear()
    draw(pyr)
    torch.cuda.synchronize()
    return pyr.level(0).clone()


@pytest.mark.parametrize("occupancy", [0, 4])
@pytest.mark.parametrize("stages", [2, 3])
@pytest.mark.parametrize("B", [1, 3])
def test_whole_store_segments_and_culled_table_are_bit_identical(scene, B, stages, occupancy):
    sorted_store, seg_store = scene
    m = torch.from_numpy(synth.total_matrix(*synth.camera_batch(W, H, list(range(3, 3 + B))))).to(torch.device("cuda", 0))
    seg_m = m.reshape(1, B, 4, 4).contiguous()
    lib = L.load()
    try:
        L.check(lib.read_set_option(b"raster_stages", stages))
        L.check(lib.read_set_option(b"raster_occupancy", occupancy))
        want = _level0(B, lambda pyr: ops.raster_project_sorted(pyr, sorted_store, m))
        seg = _level0(B, lambda pyr: ops.raster_project_segments(pyr, seg_store, seg_m))
        culled = _level0(B, lambda pyr: ops.raster_project_segments_culled(pyr, seg_store, seg_m))
    finally:
        L.check(lib.read_set_option(b"raster_stages", 2))
        L.check(lib.read_set_option(b"raster_occupancy", 0))
    drawn = want.view(B, -1) != 0x7FFFFFFFFFFFFFFF
    assert bool(drawn.float().mean(1).min() > 0.2), drawn.float().mean(1)        # every view sees the scene
    assert torch.equal(seg, want)
    assert torch.equal(culled, want)
