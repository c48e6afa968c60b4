"""The X-window entry points of the FlospDepth prior (occd_frustum_sample_window_fwd,
occd_grid_sample_prior_window_fwd): for random windows, both output orders, computed and caller-given grids and one
or two views, the window equals the matching slice of the whole grid's output bit for bit, and the whole-grid
window equals the unwindowed entry point."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GRID = (23, 20, 7)                 # 3220 voxels: not a multiple of the 256-thread block
IMG_HW = (96, 320)
DMIN, DMAX, DN = 2.0, 58.0, 16
PC_MIN, PC_MAX = (0.0, -25.6, -2.0), (51.2, 25.6, 4.4)


def L():
    from occdepth_b200 import _lib
    return _lib.lib()


def st():
    from occdepth_b200 import _lib
    return _lib.stream_ptr()


def _table(V):
    """[V, 40] camera tables: KITTI-like lidar->camera transforms 10 m into the grid (voxels behind the camera and
    closer than dmin take the out-of-range path), a stereo partner for view 1, a cropping ida"""
    vs = [(b - a) / n for a, b, n in zip(PC_MIN, PC_MAX, GRID)]
    G = torch.eye(4)
    G[0, 0], G[1, 1], G[2, 2] = vs
    G[:3, 3] = torch.tensor(PC_MIN)
    rows = []
    for v in range(V):
        T = torch.tensor([[0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, 1.2], [1.0, 0.0, 0.0, -10.0], [0.0, 0.0, 0.0, 1.0]])
        if v == 1:
            T[0, 3] = -0.54
        K4 = torch.tensor([[120.0, 0.0, 160.0, 0.0], [0.0, 120.0, 48.0, 0.0], [0.0, 0.0, 1.0, 0.0],
                           [0.0, 0.0, 0.0, 1.0]])
        ida = torch.tensor([[0.9, 0.0, 0.0, -8.0], [0.0, 0.9, 0.0, -4.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])
        rows.append(torch.cat([(T @ G)[:3].reshape(-1), K4[:3].reshape(-1), ida.reshape(-1)]))
    return torch.stack(rows).cuda()


def _run(depth, src, V, given, x0, Xl, perm, mean_mode=1, whole_entry=False):
    X, Y, Z = GRID
    h, w = depth.shape[2:]
    out = torch.full((Xl * Y * Z,), float("nan"), device="cuda")
    if given:
        if whole_entry:
            rc = L().occd_grid_sample_prior_fwd(depth.data_ptr(), src.data_ptr(), V, DN, h, w, X, Y, Z, mean_mode,
                                                out.data_ptr(), perm, st())
        else:
            rc = L().occd_grid_sample_prior_window_fwd(depth.data_ptr(), src.data_ptr(), V, DN, h, w, X, Y, Z, x0, Xl,
                                                       mean_mode, out.data_ptr(), perm, st())
    elif whole_entry:
        rc = L().occd_frustum_sample_fwd(depth.data_ptr(), src.data_ptr(), V, DN, h, w, X, Y, Z, float(IMG_HW[1]),
                                         float(IMG_HW[0]), DMIN, DMAX, mean_mode, out.data_ptr(), perm, st())
    else:
        rc = L().occd_frustum_sample_window_fwd(depth.data_ptr(), src.data_ptr(), V, DN, h, w, X, Y, Z, x0, Xl,
                                                float(IMG_HW[1]), float(IMG_HW[0]), DMIN, DMAX, mean_mode,
                                                out.data_ptr(), perm, st())
    assert rc == 0, L().occd_last_error()
    torch.cuda.synchronize()
    return out.cpu()


def _slice(full, x0, Xl, perm):
    X, Y, Z = GRID
    v = full.view(X, Z, Y) if perm else full.view(X, Y, Z)
    return v[x0:x0 + Xl].reshape(-1)


@pytest.mark.parametrize("V", [1, 2])
@pytest.mark.parametrize("given", [False, True], ids=["computed", "given"])
@pytest.mark.parametrize("perm", [0, 1])
def test_window_equals_the_slice_of_the_whole_grid(V, given, perm):
    X, Y, Z = GRID
    g = torch.Generator().manual_seed(7 * V + 2 * int(given) + perm)
    h, w = 12, 40
    depth = torch.randn(V, DN, h, w, generator=g).softmax(1).cuda()
    if given:
        # grids partly outside [-1, 1], some on cell boundaries
        src = (torch.rand(V, X * Y * Z, 3, generator=g) * 2.4 - 1.2)
        src[:, ::5] = torch.round(src[:, ::5] * 8) / 8
        src = src.cuda()
    else:
        src = _table(V)
    full = _run(depth, src, V, given, 0, X, perm)
    assert torch.isfinite(full).all()
    old = _run(depth, src, V, given, 0, X, perm, whole_entry=True)
    assert torch.equal(full.view(torch.int32), old.view(torch.int32))
    windows = [(0, 1), (X - 1, 1), (0, X - 1), (1, X - 1)]
    for _ in range(8):
        x0 = int(torch.randint(0, X, (1,), generator=g))
        windows.append((x0, int(torch.randint(1, X - x0 + 1, (1,), generator=g))))
    for x0, Xl in windows:
        got = _run(depth, src, V, given, x0, Xl, perm)
        want = _slice(full, x0, Xl, perm)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (x0, Xl)
