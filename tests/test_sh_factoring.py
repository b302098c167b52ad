"""CPU: the factored SH gradient of the view-parallel exchange is pinned on the REFERENCE's own backward output.  The golden
fixtures (tests/golden/*.npz, generated from the live reference extension by make_golden.py) hold, for one view, the reference's
dL_dcolors, its clamp flags and its dL_dsh: the claim that the exchange rests on -- dL_dsh[k][c] = w_k(dir(mean, camera)) *
(dL_dcolor[c] unless clamped), backward.cu:45-139 -- must reproduce the reference's dL_dsh from the other two."""
import os

import numpy as np
import pytest
import torch

import _golden
import gof_dp

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("name", ["f0_sh3", "f1_sh1_mip_bg", "f3_sh0_inside"])
def test_reference_dsh_is_the_outer_product_of_basis_and_masked_dcolor(name):
    d = _golden.load(os.path.join(GOLD, name + ".npz"))
    degree = int(d["cfg"]["sh_degree"])
    means = torch.from_numpy(d["means3D"]).double()
    cam = torch.from_numpy(d["campos"]).double()
    rgb = torch.from_numpy(d["grad_dcolors"]).double() * (1.0 - torch.from_numpy(d["clamped"].astype(np.float64)))
    want = torch.from_numpy(d["grad_dsh"]).double()
    dirs = means - cam
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    w = gof_dp.sh_grad_weights_torch(dirs, degree)                         # [P, (degree+1)^2]
    got = torch.zeros_like(want)
    got[:, :w.shape[1], :] = w[:, :, None] * rgb[:, None, :]
    assert float(want.abs().max()) > 0
    assert float((got - want).abs().max()) <= 2e-6 * float(want.abs().max())
    assert float(want[:, w.shape[1]:, :].abs().max()) == 0.0 if w.shape[1] < 16 else True    # nothing above the active degree

    # the record form: header (camera centre, degree) + three colour planes, expanded by the routine the CPU buckets use
    P = means.shape[0]
    plane = (P + 63) // 64 * 64
    rec = torch.zeros(gof_dp.SH_SLOT_HEADER + 3 * plane, dtype=torch.float64)
    rec[:3], rec[3] = cam, float(degree)
    rec[gof_dp.SH_SLOT_HEADER:].view(3, plane)[:, :P] = rgb.t()
    again = gof_dp.sh_grad_from_views_torch(means, [rec], P, 16)
    assert float((again - want).abs().max()) <= 2e-6 * float(want.abs().max())
