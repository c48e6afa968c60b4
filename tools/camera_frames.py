"""Camera frames for OccDepth.predict_frame / serving.CameraPipeline and the batch the reference's host route builds
from the same frame (numpy normalisation as kitti_dataset.py:376-402, the numpy vox2pix of oracle.projection,
nyu_dataset.py's load_depth and pose algebra, the collate layout).  Shared by tests/test_gpu_camera_pipeline.py and
tools/camera_bench.py; seeded, so every caller sees the same frames."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tools")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

MEAN, STD = np.array([0.485, 0.456, 0.406], np.float32), np.array([0.229, 0.224, 0.225], np.float32)
NYU_K = np.array([[518.8579, 0, 320], [0, 518.8579, 240], [0, 0, 1]])


def host_img(img_u8, H, W):
    """kitti_dataset.py:376-402 / nyu_dataset.py:225-245 with torchvision's transform restated in numpy -> (3, H, W)"""
    x = (np.array(img_u8, dtype=np.float32) / 255.0)[:H, :W, :]
    return torch.from_numpy(np.ascontiguousarray(((x - MEAN) / STD).transpose(2, 0, 1)))


def load_depth(depth, maxDepth=10):
    depth = depth / 8000.0
    depth = depth.astype("float32")
    depth[depth > maxDepth] = maxDepth
    depth[depth < 0] = 0
    return depth


def host_batch(m, frame, geo):
    """the collated batch (B = 1) the reference's dataset builds from the same frame"""
    from oracle.projection import vox2pix
    H, W = geo["img_hw"]
    imgs = frame["img"]
    batch = {"img": torch.stack([host_img(im, H, W) for im in imgs]).unsqueeze(0)}
    ps = m.project_scale
    if m.dataset == "NYU":
        T0 = np.linalg.inv(frame["cam_pose"])
        poses = [T0]
        if "depth" in frame:
            T01 = np.array([[1, 0, 0, -0.1], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
            poses.append(T01 @ T0)
            batch["gt_depth"] = torch.as_tensor(np.stack([load_depth(frame["depth"])])).unsqueeze(0)
            batch["virtual_bf"] = torch.stack([torch.from_numpy(np.array(0.1 * 518.8579))])
        Ks, origin = [NYU_K] * len(poses), frame["vox_origin"]
        voxel, scene = 0.08, (4.8, 4.8, 2.88)
        batch.update(cam_k=[torch.from_numpy(np.array([NYU_K])).double()],
                     T_velo_2_cam=[torch.from_numpy(T0[None]).float()], ida_mats=[torch.eye(4)[None]],
                     vox_origin=torch.stack([torch.from_numpy(origin).double()]))
    else:
        poses, Ks = list(frame["T_velo_2_cam"]), list(frame["cam_k"])
        origin, voxel, scene = geo["vox_origin"], geo["voxel_size"], geo["scene_size"]
        V = len(poses)
        batch.update(cam_k=[torch.from_numpy(frame["cam_k"]).double()],
                     T_velo_2_cam=[torch.from_numpy(frame["T_velo_2_cam"]).float()],
                     ida_mats=[torch.eye(4).unsqueeze(0).repeat(V, 1, 1)])
    pix, fov = [], []
    for T, K in zip(poses, Ks):
        p, f, _ = vox2pix(T, K, origin, voxel, W, H, scene, geo.get("pattern_id", 0))
        pix.append(torch.from_numpy(p))
        fov.append(torch.from_numpy(f))
    batch["projected_pix_%d" % ps] = [torch.stack(pix)]
    batch["fov_mask_%d" % ps] = [torch.stack(fov)]
    import shipped_configs
    return shipped_configs.to_cuda(batch)


def kitti_geometry(H, W, full):
    scene = tuple(s * 0.2 for s in full)
    return dict(img_hw=(H, W), vox_origin=np.array([0.0, -scene[1] / 2.0, -2.0]), voxel_size=0.4, scene_size=scene)


def kitti_frame(V, H, W, seed, shift=0.0):
    """seeded uint8 images a little larger than the crop, synthetic.kitti_calib calibrations (float64, as the dataset
    holds them); `shift` moves the cameras along the lidar's y axis"""
    import synthetic
    g = np.random.default_rng(seed)
    K, Ts = synthetic.kitti_calib(W, H)
    T = np.stack([t.astype(np.float64) for t in Ts[:V]])
    T[:, 0, 3] += shift
    return {"img": g.integers(0, 256, size=(V, H + 3, W + 5, 3), dtype=np.uint8), "cam_k": np.stack([K] * V), "T_velo_2_cam": T}


def nyu_frame(seed, with_depth=True):
    """one uint8 image, a pose whose view covers ~45 % of the voxels, and a uint16 depth PNG"""
    g = np.random.default_rng(seed)
    origin = np.array([-2.0, 0.5, -0.1])
    pose = np.eye(4)
    pose[:3, :3] = [[1, 0, 0], [0, 0, 1], [0, -1, 0]]        # camera z -> world y, camera y -> world -z
    pose[:3, 3] = origin + np.array([2.4, 0.3, 1.4])
    f = {"img": g.integers(0, 256, size=(1, 480, 640, 3), dtype=np.uint8), "cam_pose": pose, "vox_origin": origin,
         "cam_k": NYU_K}
    if with_depth:
        f["depth"] = g.integers(4000, 60000, size=(480, 640), dtype=np.uint16)
    return f
