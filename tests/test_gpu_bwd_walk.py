"""GPU: the blend backward's per-batch walk of the quarter-warp lists against the CPU oracle.

Each 4x2 pixel block of a warp walks its own list over a whole batch of 256 tile-list entries, moving from group to group
of 32 on its own cursor.  The scenes here make those lists as unequal as possible: a stack of faint Gaussians of about a
pixel, all on the ray of one pixel, gives the tile of that pixel a list of several hundred entries (several batches) that
only the 4x2 block holding that pixel blends, while the other blocks of its warp see a few ordinary Gaussians or nothing."""
import numpy as np
import pytest
import torch

import gof_synth
from test_gpu_oracle import check, run_both

pytestmark = pytest.mark.gpu


def stacked_scene(width, height, n_base, n_stack, seed, pixel):
    """An ordinary scene of n_base small Gaussians plus n_stack faint ones of ~1 pixel at depths spread along the ray
    through `pixel` (x, y)."""
    cam, gs = gof_synth.make_scene(dict(P=n_base, width=width, height=height, seed=seed, sigma_px=1.5), view=2)
    center = torch.as_tensor(cam.camera_center).to(torch.float64).reshape(3)
    # the ray through the pixel centre, from the inverse of the world-to-view transform (row-vector convention)
    wv = torch.as_tensor(cam.world_view_transform).to(torch.float64).reshape(4, 4)
    px, py = pixel
    d_view = torch.tensor([(2.0 * (px + 0.5) / width - 1.0) * cam.tanfovx, (2.0 * (py + 0.5) / height - 1.0) * cam.tanfovy,
                           1.0, 0.0], dtype=torch.float64)
    d = (d_view @ torch.linalg.inv(wv))[:3]
    g = torch.Generator().manual_seed(seed + 1)
    depth = 2.5 + 3.0 * torch.rand(n_stack, 1, generator=g, dtype=torch.float64)
    means = center + depth * d
    scales = (0.4 * depth / cam.focal_x) * (0.8 + 0.4 * torch.rand(n_stack, 3, generator=g, dtype=torch.float64))
    rot = torch.randn(n_stack, 4, generator=g, dtype=torch.float64)
    rot = rot / rot.norm(dim=1, keepdim=True)
    opac = 0.01 + 0.02 * torch.rand(n_stack, 1, generator=g, dtype=torch.float64)
    shs = torch.zeros(n_stack, 16, 3, dtype=torch.float64)
    shs[:, 0, :] = (torch.rand(n_stack, 3, generator=g, dtype=torch.float64) * 2.0 - 1.0) * 1.77
    f32 = lambda t: t.to(torch.float32)   # noqa: E731
    extra = {"means3D": f32(means), "scales": f32(scales), "rotations": f32(rot), "opacities": f32(opac), "shs": f32(shs)}
    gs = dict(gs, **{k: torch.cat([gs[k], extra[k]]).contiguous() for k in extra})
    return cam, gs


@pytest.mark.parametrize("width,height,n_base,pixel,seed", [
    (150, 90, 1500, (37, 21), 7),    # a tile in the interior
    (147, 83, 800, (145, 81), 8),    # the bottom-right tile, cut by the image border
])
def test_backward_walk_unequal_quarter_lists(width, height, n_base, pixel, seed):
    dev = torch.device("cuda")
    cam, gs = stacked_scene(width, height, n_base, 900, seed, pixel)
    got, out, oradii, st, d = run_both(cam, gs, dev, seed=seed)
    lens = st["ranges"][:, 1].astype(np.int64) - st["ranges"][:, 0]
    assert lens.max() > 512, "the stacked tile must span several batches"
    px, py = pixel
    assert st["n_contrib"][0][py, px] > 256, "the stacked pixel must blend entries of more than one batch"
    check(got, out, oradii, st, d)
