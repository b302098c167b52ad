"""The scene table of the pose and focal-length gradient tests (test_gpu_camera_grad.py, test_gpu_focal_grad.py).

name -> (scene factory, options), the options of test_gpu_grad_stagewise.run: bg, kernel_size, scale_modifier and colors_seed
(precomputed colours).  The table holds
  - test_gpu_grad_stagewise's scenes: SH degrees 0-3, C1, precomputed colours with a background, mip filter and scale modifier,
    screen-filling Gaussians, the camera inside the cloud, stacked lists of about 1 000 entries (several 256-entry batches),
    C2 view 3 and C3 view 5 (1920x1080: 8 160 tiles, 7 813 camera rows).  Its bucket_* scenes become plain_* at the same P:
    a GradBucket refuses pose and focal-length gradients;
  - _integrate_scenes.saturation_scene (pixels that saturate at list positions 3, 32, 33, 256 and 257: group and batch
    boundaries) and threshold_scene (alphas at the 1/255 threshold and the 0.99 clamp);
  - near_plane: the camera inside the cloud with Gaussians just beyond the 0.2 near cull, where view2gaussian's chain rule
    cancels hardest (a pixel-wide Gaussian at depth 0.2 has scales of ~1e-3, 1 / scale^2 ~ 1e6);
  - rows_<P>: the camera reduction k_camera_grad_sum (64 groups of 16 threads over ceil(P / 128) rows) with one row, one row
    exactly full, two rows, exactly 64 rows, 65 rows and 66 rows (every group but one with two rows);
  - image_<W>x<H>: the focal reduction k_focal_grad_sum (1 024 threads over the tiles) with one tile of one pixel, one full
    tile, two tiles of which one has one column, and 1 023, 1 024 and 1 025 tiles; C3 view 5 is its 8 160-tile 1080p case;
  - ragged_4097: P not a multiple of the 128-Gaussian CTA, an odd image size and a background."""
import numpy as np
import torch

import _integrate_scenes as iscenes
import gof_oracle
import gof_synth
from test_gpu_grad_stagewise import SCENES as STAGEWISE
from test_gpu_grad_stagewise import _inside_scene


def _near_plane_scene():
    """The camera_inside scene (6 000 Gaussians around a camera at radius 0.8, SH degree 3) and 300 Gaussians of 0.5 to 4
    pixels at view depths in (0.2, 0.3]: just in front of the near cull (tz <= 0.2 is culled)."""
    cam, gs = _inside_scene()
    rng = np.random.default_rng(61)
    n = 300
    xy = np.stack([rng.uniform(0, cam.image_width, n), rng.uniform(0, cam.image_height, n)], 1)
    near = iscenes.blobs(cam, xy, rng.uniform(0.2005, 0.3, n), rng.uniform(0.5, 4.0, n), rng.uniform(0.05, 0.9, n), seed=62)
    near["shs"][:, 1:, :] = torch.from_numpy(rng.uniform(-0.3, 0.3, (n, 15, 3)).astype(np.float32))
    return cam, iscenes.concat([gs, near])


def _small(P, W, H, seed, view, **kw):
    return lambda: gof_synth.make_scene(dict(P=P, width=W, height=H, seed=seed, **kw), view=view)


SCENES = {
    **{k: v for k, v in STAGEWISE.items() if not v[1].get("bucket")},
    **{f"plain_{k[len('bucket_'):]}": (v[0], {}) for k, v in STAGEWISE.items() if v[1].get("bucket")},
    "saturation": (iscenes.saturation_scene, {}),
    "threshold": (iscenes.threshold_scene, {}),
    "near_plane": (_near_plane_scene, {}),
    **{f"rows_{P}": (_small(P, 96, 64, 70 + i, 2 * i + 1), {}) for i, P in enumerate((1, 127, 128, 129, 64 * 128, 64 * 128 + 1,
                                                                                     65 * 128 + 1))},
    "image_1x1": (_small(300, 1, 1, 80, 5, sigma_px=0.5), {}),
    **{f"image_{W}x{H}": (_small(P, W, H, 81 + i, 6 + i), {}) for i, (W, H, P) in enumerate(((16, 16, 400), (17, 16, 400),
                                                                                            (496, 528, 60_000),
                                                                                            (512, 512, 60_000),
                                                                                            (400, 656, 60_000)))},
    "ragged_4097": (_small(4097, 203, 117, 17, 4), dict(bg=(0.3, 0.6, 0.9))),
}


def inputs(name, colors=False):
    """(cam, gs, the keyword arguments of _util.fwd_args) of scene `name`; colors=True adds precomputed colours (seed 5) to a
    scene that has none."""
    make, opt = SCENES[name]
    cam, gs = make()
    P = gs["means3D"].shape[0]
    seed = opt.get("colors_seed", 5 if colors else None)
    rgb = None if seed is None else torch.rand(P, 3, generator=torch.Generator().manual_seed(seed))
    return cam, gs, dict(kernel_size=opt.get("kernel_size", 0.0), scale_modifier=opt.get("scale_modifier", 1.0),
                         bg=opt.get("bg", (0.0, 0.0, 0.0)), colors_precomp=rgb)


def oracle_scene(cam, gs, kw, v2g=None):
    """gof_oracle.Scene of the same inputs."""
    rgb = kw["colors_precomp"]
    return gof_oracle.Scene(cam.image_width, cam.image_height, cam.tanfovx, cam.tanfovy, cam.world_view_transform,
                            cam.full_proj_transform, cam.camera_center, gs["means3D"], gs["opacities"], scales=gs["scales"],
                            rotations=gs["rotations"], shs=None if rgb is not None else gs["shs"], colors_precomp=rgb,
                            sh_degree=gs["sh_degree"], kernel_size=kw["kernel_size"], scale_modifier=kw["scale_modifier"],
                            bg=kw["bg"], v2g_precomp=v2g)
