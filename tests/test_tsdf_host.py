"""CPU: host-side pieces of gof_tsdf -- the reference's intrinsics formula and the PLY writer."""
import numpy as np
import pytest
import torch

import gof_synth

gof_tsdf = pytest.importorskip("gof_tsdf")


@pytest.mark.parametrize("wh", [(1600, 1200), (320, 240), (161, 97)])
def test_intrinsics_match_the_reference_formula(wh):
    W, H = wh
    for v in gof_synth.make_surface_views(W, H, 7):
        ndc2pix = torch.tensor([[W / 2, 0, 0, (W - 1) / 2], [0, H / 2, 0, (H - 1) / 2], [0, 0, 0, 1]]).float().T
        intrins = (v.projection_matrix @ ndc2pix)[:3, :3].T            # extract_mesh_tsdf.py:49-55, float32
        want = (intrins[0, 0].item(), intrins[1, 1].item(), intrins[0, 2].item(), intrins[1, 2].item())
        assert gof_tsdf.intrinsics_from_view(v) == want


def test_extrinsic_is_world_view_transform_transposed():
    v = gof_synth.make_surface_views(64, 48, 3)[1]
    E = gof_tsdf.extrinsic_from_view(v)
    assert torch.equal(E, v.world_view_transform.t())
    assert torch.equal(E[3], torch.tensor([0.0, 0.0, 0.0, 1.0]))


def test_write_ply_round_trips(tmp_path):
    rng = np.random.default_rng(0)
    mesh = {"vertices": torch.from_numpy(rng.standard_normal((50, 3)).astype(np.float32)),
            "faces": torch.from_numpy(rng.integers(0, 50, (80, 3))),
            "colors": torch.from_numpy(rng.uniform(-0.1, 1.1, (50, 3)).astype(np.float32))}
    path = tmp_path / "m.ply"
    gof_tsdf.write_ply(str(path), mesh)
    data = path.read_bytes()
    assert data.startswith(b"ply\nformat binary_little_endian 1.0\n")
    back = gof_tsdf.read_ply(str(path))
    assert np.array_equal(back["vertices"], mesh["vertices"].numpy())
    assert np.array_equal(back["faces"], mesh["faces"].numpy())
    c = mesh["colors"].numpy()
    assert np.array_equal(back["colors_u8"], np.clip(c * np.float32(255), 0, 255).astype(np.uint8))
    empty = {"vertices": torch.zeros(0, 3), "faces": torch.zeros(0, 3, dtype=torch.int64), "colors": torch.zeros(0, 3)}
    gof_tsdf.write_ply(str(path), empty)
    back = gof_tsdf.read_ply(str(path))
    assert back["vertices"].shape == (0, 3) and back["faces"].shape == (0, 3)


def test_volume_rejects_cpu():
    with pytest.raises(RuntimeError):
        gof_tsdf.TSDFVolume(device="cpu")
