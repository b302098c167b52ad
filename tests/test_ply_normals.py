"""CPU: gof_tsdf.write_ply / read_ply with vertex normals (float nx ny nz after x y z), and without them byte for byte the
format the mesh evaluators load."""
import numpy as np
import torch

import gof_tsdf


def _mesh(seed=3, V=9, F=6):
    g = torch.Generator().manual_seed(seed)
    return {"vertices": torch.randn(V, 3, generator=g), "faces": torch.randint(0, V, (F, 3), generator=g),
            "colors": torch.rand(V, 3, generator=g)}


def _expected_bytes(mesh):
    """The PLY without normals, laid out by hand: header, then per vertex 3 little-endian floats and 3 bytes, then per face a
    count byte and 3 int32."""
    v = mesh["vertices"].numpy().astype("<f4")
    rgb = np.clip(mesh["colors"].numpy().astype(np.float32) * np.float32(255.0), 0, 255).astype(np.uint8)
    f = mesh["faces"].numpy().astype("<i4")
    head = ("ply\nformat binary_little_endian 1.0\n"
            f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
            "property uchar red\nproperty uchar green\nproperty uchar blue\n"
            f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n").encode("ascii")
    body = b"".join(v[i].tobytes() + rgb[i].tobytes() for i in range(v.shape[0]))
    body += b"".join(b"\x03" + f[i].tobytes() for i in range(f.shape[0]))
    return head + body


def test_without_normals_the_file_is_unchanged(tmp_path):
    for mesh in (_mesh(), dict(_mesh(4), normals=None)):
        path = tmp_path / "m.ply"
        gof_tsdf.write_ply(str(path), mesh)
        assert path.read_bytes() == _expected_bytes(mesh)
        back = gof_tsdf.read_ply(str(path))
        assert "normals" not in back
        assert np.array_equal(back["vertices"], mesh["vertices"].numpy())
        assert np.array_equal(back["faces"], mesh["faces"].numpy())


def test_normals_round_trip(tmp_path):
    mesh = _mesh(5)
    n = torch.nn.functional.normalize(torch.randn(9, 3, generator=torch.Generator().manual_seed(6)), dim=1)
    n[2] = 0.0   # a vertex without a normal
    mesh["normals"] = n
    path = tmp_path / "n.ply"
    gof_tsdf.write_ply(str(path), mesh)
    data = path.read_bytes()
    head = data[:data.index(b"end_header\n")].decode("ascii").splitlines()
    props = [ln.split()[-1] for ln in head if ln.startswith("property") and "list" not in ln]
    assert props == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    back = gof_tsdf.read_ply(str(path))
    assert np.array_equal(back["vertices"], mesh["vertices"].numpy())
    assert np.array_equal(back["normals"], n.numpy())
    assert np.array_equal(back["faces"], mesh["faces"].numpy())
    plain = tmp_path / "p.ply"
    gof_tsdf.write_ply(str(plain), _mesh(5))
    assert np.array_equal(back["colors_u8"], gof_tsdf.read_ply(str(plain))["colors_u8"])
