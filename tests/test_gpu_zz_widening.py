"""Parity of the widened rows (SURVEY 8f): the callers' post-processing (class map) and the data pipeline's index
generation (vox2pix) on the device.  Kept in their own file, collected after the hot-path parity tests."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def test_class_map_matches_host_postprocessing():
    """OccDepth.class_map vs the reference callers' host-side post-processing (generate_output.py:94-97)"""
    import numpy as np
    from occdepth_b200.models.OccDepth import OccDepth
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(2, 20, 17, 9, 5, generator=g) * 3
    logits[0, 7, 3, 2, 1] = logits[0, 4, 3, 2, 1] = 50.0             # an exact tie: the first index wins
    want = np.argmax(torch.softmax(logits, dim=1).numpy(), axis=1).astype(np.uint16)
    got = OccDepth.class_map(logits.cuda()).cpu().numpy()
    assert got.dtype == np.uint16 and got.shape == want.shape
    assert got[0, 3, 2, 1] == 4
    # softmax may merge logits that differ by < 1 ulp of the sum; everywhere else the maps are identical
    diff = got != want
    assert diff.mean() < 1e-4
    if diff.any():
        p = torch.softmax(logits, dim=1).numpy()
        b, x, y, z = np.nonzero(diff)
        assert np.all(p[b, got[diff], x, y, z] == p[b, want[diff], x, y, z])
    # the submission writer's label remap (generate_kitti_submission.py:79) in the same launch
    inv_map = np.array([0, 10, 11, 15, 18, 20, 30, 31, 32, 40, 44, 48, 49, 50, 51, 70, 71, 72, 80, 81], dtype=np.int32)
    sub = OccDepth.class_map(logits.cuda(), inv_map).cpu().numpy()
    assert np.array_equal(sub, inv_map[got.reshape(-1)].astype(np.uint16).reshape(got.shape))


def test_vox2pix_device_matches_reference_outputs():
    """occdepth_b200.data.vox2pix (occd_vox2pix_fwd) vs the committed outputs of the reference's numba vox2pix:
    indices, FOV mask and depth bit for bit (tests/golden/vox2pix.pt, oracle/gen_golden.py)"""
    import numpy as np
    from occdepth_b200.data import vox2pix
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vox2pix.pt"))
    for name, c in gold.items():
        pix, fov, z = vox2pix(c["cam_E"].numpy(), c["cam_k"].numpy(), c["vox_origin"].numpy(), c["voxel_size"],
                              c["img_W"], c["img_H"], c["scene_size"], c["pattern_id"])
        assert pix.is_cuda and pix.dtype == torch.int64 and fov.dtype == torch.bool and z.dtype == c["pix_z"].dtype
        assert torch.equal(pix.cpu(), c["pix"].long()), name
        assert torch.equal(fov.cpu(), c["fov"]), name
        assert np.array_equal(z.cpu().numpy(), c["pix_z"].numpy(), equal_nan=True), name


def test_normalize_rgb_device_matches_torchvision():
    """occdepth_b200.data.normalize_rgb vs the datasets' ToTensor + Normalize (kitti_dataset.py:164-171,376-402)"""
    import numpy as np
    from torchvision import transforms
    from occdepth_b200.data import IMAGENET_MEAN, IMAGENET_STD, normalize_rgb
    g = np.random.default_rng(1)
    img = g.integers(0, 256, size=(40, 61, 3), dtype=np.uint8)
    img[0, :256 % 61] = 0
    H, W = 37, 50
    ref = transforms.Compose([transforms.ToTensor(), transforms.Normalize(mean=list(IMAGENET_MEAN), std=list(IMAGENET_STD))])(
        (np.array(img, dtype=np.float32) / 255.0)[:H, :W, :])
    got = normalize_rgb(img, H, W)
    assert got.is_cuda and got.dtype == torch.float32 and tuple(got.shape) == (3, H, W)
    assert torch.equal(got.cpu(), ref)
