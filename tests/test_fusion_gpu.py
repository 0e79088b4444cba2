"""TSDFVolume on the device against the fp64 oracle (oracle/fusion.py): integration voxel by voxel, brick coverage, order
and pool-size invariance, marching cubes, and run_fusion.py end to end."""
import os

import numpy as np
import pytest
import torch

import fusion_scenes as S
from oracle import fusion as OF

pytestmark = pytest.mark.gpu

LO, V, SHAPE = (-2.0, -1.6, 0.0), 0.05, (80, 64, 112)
MAX_DEPTH = 4.0
TOL = 1e-5


def _volume(**kw):
    from scsfm.fusion import TSDFVolume
    hi = np.asarray(LO) + np.asarray(SHAPE) * V
    return TSDFVolume(LO, hi, V, max_depth=MAX_DEPTH, **kw)


def _all_voxels(shape=SHAPE):
    ijk = np.stack(np.meshgrid(*[np.arange(n) for n in shape], indexing="ij"), -1).reshape(-1, 3)
    return torch.from_numpy(ijk).cuda()


def _dense(vol, shape=SHAPE):
    tsdf, w, rgb = vol.sample(_all_voxels(shape))
    return (tsdf.cpu().numpy().reshape(shape), w.cpu().numpy().reshape(shape), rgb.cpu().numpy().reshape(shape + (3,)))


def _allocated(vol, shape=SHAPE):
    a = np.zeros(shape, bool)
    ijk = vol.brick_voxels().cpu().numpy()
    a[ijk[:, 0], ijk[:, 1], ijk[:, 2]] = True
    return a


def _oracle(depth, color, K, T):
    g = OF.Grid(LO, V, SHAPE)
    amb = np.zeros(SHAPE, bool)
    for f in range(len(depth)):
        _, a = OF.integrate(g, depth[f], K[f], T[f], 4 * V, MAX_DEPTH, color[f])
        amb |= a
    return g, amb


def _close(a, b):
    """Within 1e-5 relative, measured against max(|b|, 1): tsdf lies in [-1, 1], where the fp32 error of the projection is
    absolute (the depth difference divided by trunc), so for tsdf this is 1e-5 of the field's range; rgb (0..255) is compared
    truly relative wherever it is at least 1."""
    return np.abs(a - b) <= TOL * np.maximum(np.abs(b), 1.0)


@pytest.mark.parametrize("shared_k", [False, True])
def test_integration_matches_the_fp64_oracle_voxel_by_voxel(shared_k):
    depth, color, K, T = S.street(11 + shared_k, 6)
    if shared_k:
        K = np.broadcast_to(K[0], K.shape).copy()
    vol = _volume()
    vol.integrate(torch.from_numpy(depth).cuda()[:, None], K[0] if shared_k else torch.from_numpy(K), torch.from_numpy(T),
                  torch.from_numpy(color).cuda())
    g, amb = _oracle(depth, color, K, T)
    tsdf, w, rgb = _dense(vol)
    keep = ~amb
    assert amb.mean() < 1e-3, amb.mean()
    assert (g.w > 0).sum() > 20000 and (g.w == 0).sum() > 20000
    assert np.array_equal(w[keep], g.w[keep])
    assert _close(tsdf[keep], g.tsdf[keep]).all(), np.abs(tsdf - g.tsdf)[keep].max()
    assert _close(rgb[keep], g.rgb[keep]).all(), np.abs(rgb - g.rgb)[keep].max()
    # coverage: every voxel the oracle updates is in an allocated brick, and voxels in no brick read w = 0
    alloc = _allocated(vol)
    assert alloc[g.w > 0].all()
    assert not alloc.all() and np.all(w[~alloc] == 0) and np.all(tsdf[~alloc] == 0) and np.all(rgb[~alloc] == 0)
    assert vol.num_bricks == alloc.sum() // 512
    # voxels outside the box read zeros too
    out = vol.sample(torch.tensor([[-1, 0, 0], [0, SHAPE[1], 0], [5, 5, 10 ** 6]], device="cuda"))
    assert all(float(x.abs().sum()) == 0 for x in out)


def test_scene_has_the_cases_it_is_meant_to_cover():
    depth, color, K, T = S.street(11, 6)
    assert (depth == 0).any() and np.isnan(depth).any() and (depth > MAX_DEPTH).any()
    assert len(np.unique(K[:, 0, 0])) > 1
    g = OF.Grid(LO, V, SHAPE)
    inv = np.linalg.inv(T[0])
    assert ((g.centres() @ inv[:3, :3].T + inv[:3, 3])[..., 2] <= 0).any()      # voxels behind the camera
    # surface points of the frames outside the box: the frusta leave it
    H, W = depth.shape[1:]
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    hi = np.asarray(LO) + np.asarray(SHAPE) * V
    for f in range(len(depth)):
        d = np.nan_to_num(depth[f].astype(np.float64))
        ok = (d > 0) & (d <= MAX_DEPTH)
        pc = np.stack([(u - K[f, 0, 2]) / K[f, 0, 0] * d, (v - K[f, 1, 2]) / K[f, 1, 1] * d, d], -1)[ok]
        pw = pc @ T[f][:3, :3].T + T[f][:3, 3]
        assert np.any((pw < LO) | (pw > hi)) and np.any(np.all((pw > LO) & (pw < hi), 1))


def _integrate_split(depth, color, K, T, splits, **kw):
    vol = _volume(**kw)
    d, c = torch.from_numpy(depth).cuda(), torch.from_numpy(color).cuda()
    i = 0
    for n in splits:
        vol.integrate(d[i:i + n], torch.from_numpy(K[i:i + n]), T[i:i + n], c[i:i + n])
        i += n
    return vol


def test_order_invariance_and_pool_growth_are_bitwise(monkeypatch):
    from scsfm.fusion import TSDFVolume
    depth, color, K, T = S.street(5, 16)
    ref = _integrate_split(depth, color, K, T, [16])
    want = _dense(ref)
    alloc = _allocated(ref)
    for splits in ([1] * 16, [3, 13]):
        got = _dense(_integrate_split(depth, color, K, T, splits))
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, want)), splits
    monkeypatch.setattr(TSDFVolume, "_INITIAL_BRICKS", 1)
    small = _integrate_split(depth, color, K, T, [16])
    assert small._pool.shape[0] >= small.num_bricks > 200
    got = _dense(small)
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, want))
    assert np.array_equal(_allocated(small), alloc)
    assert (want[1] > 0).sum() > 0


def _mesh_vs_oracle(vol, shape):
    verts, faces, colors, keys = vol.mesh(with_keys=True)
    tsdf, w, rgb = _dense(vol, shape)
    tris, ov = OF.marching_cubes(tsdf, w, rgb, vol.lo, vol.voxel_size)
    keys = keys.cpu().numpy()
    got = OF.canonical_triangles(keys[faces.cpu().numpy()])
    assert np.array_equal(got, OF.canonical_triangles(tris))
    assert np.array_equal(keys, np.array(sorted(ov), np.int64))
    pos = np.stack([ov[k][0] for k in keys])
    col = np.stack([ov[k][1] for k in keys])
    v = verts.cpu().numpy().astype(np.float64)
    # the kernel computes the vertex in fp64 and stores it in fp32: 1e-6 voxel plus the fp32 rounding of the coordinate
    assert np.all(np.abs(v - pos) <= 1e-6 * vol.voxel_size + np.abs(pos) * 2.0 ** -24)
    assert np.array_equal(colors.cpu().numpy(), col)
    return verts, faces, colors


def test_mesh_matches_the_oracle_on_the_street():
    depth, color, K, T = S.street(7, 8)
    vol = _integrate_split(depth, color, K, T, [8])
    assert vol.dims == SHAPE
    verts, faces, _ = _mesh_vs_oracle(vol, SHAPE)
    assert len(faces) > 5000


def test_fused_sphere_from_twelve_directions_is_closed():
    from scsfm.fusion import TSDFVolume
    c, v = (1.2, 1.2, 1.2), 0.04
    depth, K, T = S.sphere_views(c, 0.5)
    vol = TSDFVolume((0, 0, 0), (2.4, 2.4, 2.4), v)
    vol.integrate(torch.from_numpy(depth).cuda(), K, T)
    verts, faces, _ = _mesh_vs_oracle(vol, vol.dims)
    assert OF.euler_characteristic(faces.cpu().numpy()) == 2
    r = np.linalg.norm(verts.cpu().numpy() - np.asarray(c), axis=1)
    assert np.abs(r - 0.5).max() < v


def test_input_checks():
    vol = _volume()
    d = torch.ones(2, 8, 8, device="cuda")
    T = np.tile(np.eye(4), (2, 1, 1))
    K = np.eye(3)
    with pytest.raises(ValueError, match="depth"):
        vol.integrate(d.cpu(), K, T)
    with pytest.raises(TypeError, match="depth"):
        vol.integrate(d.double(), K, T)
    with pytest.raises(ValueError, match="depth"):
        vol.integrate(d[0], K, T)
    with pytest.raises(ValueError, match="K"):
        vol.integrate(d, np.eye(4), T)
    with pytest.raises(ValueError, match="cam_to_world"):
        vol.integrate(d, K, T[:1])
    bad = T.copy()
    bad[1, 0, 3] = np.nan
    with pytest.raises(ValueError, match="cam_to_world"):
        vol.integrate(d, K, bad)
    with pytest.raises(TypeError, match="color"):
        vol.integrate(d, K, T, torch.zeros(2, 8, 8, 3, device="cuda"))
    with pytest.raises(ValueError, match="color"):
        vol.integrate(d, K, T, torch.zeros(2, 8, 8, 3, dtype=torch.uint8))
    with pytest.raises(TypeError, match="ijk"):
        vol.sample(torch.zeros(3, 3, dtype=torch.int32, device="cuda"))
    with pytest.raises(ValueError, match="ijk"):
        vol.sample(torch.zeros(3, 2, dtype=torch.int64, device="cuda"))
    assert vol.num_bricks == 0 and [len(x) for x in vol.mesh()] == [0, 0, 0]


def test_run_fusion_writes_the_mesh_of_the_volume(tmp_path):
    from PIL import Image
    import models
    import run_fusion
    from scsfm import inference_io as io
    from scsfm.fusion import TSDFVolume
    from scsfm.infer import Predictor
    H, W, n = 64, 128, 9
    rng = np.random.default_rng(3)
    seq = tmp_path / "seqs" / "04"
    os.makedirs(seq / "image_2")
    for i in range(n):
        Image.fromarray(rng.integers(0, 256, (H, W, 3), dtype=np.uint8)).save(seq / "image_2" / ("%06d.png" % i))
    torch.manual_seed(0)
    net = models.DispResNet(18, False)
    torch.save({"state_dict": net.state_dict()}, tmp_path / "disp.tar")
    T = np.tile(np.eye(4), (n, 1, 1))
    T[:, 2, 3] = np.arange(n) * 0.3
    T[:, 0, 3] = np.sin(np.arange(n)) * 0.1
    np.savetxt(tmp_path / "poses.txt", T[:, :3].reshape(n, 12), fmt="%1.8e")
    out = tmp_path / "m.ply"
    args = ["--pretrained-dispnet", str(tmp_path / "disp.tar"), "--dataset-dir", str(tmp_path / "seqs") + "/", "--sequence", "04",
            "--img-height", str(H), "--img-width", str(W), "--poses", str(tmp_path / "poses.txt"), "--voxel-size", "0.05",
            "--max-depth", "30", "--intrinsics", "60", "60", "63.5", "31.5", "--batch-size", "4", "--output", str(out)]
    run_fusion.main(args)
    v, f, c = io.read_ply(str(out))
    # the same predictions and poses through TSDFVolume directly
    net.to("cuda").set_conv_mode("tf32x3").eval()
    pred = Predictor(net)
    frames = np.stack([io.load_frame(str(seq / "image_2" / ("%06d.png" % i)), H, W) for i in range(n)])
    poses = io.read_poses(str(tmp_path / "poses.txt"))
    P = np.tile(np.eye(4), (n, 1, 1))
    P[:, :3] = poses
    vol = TSDFVolume(P[:, :3, 3].min(0) - 30, P[:, :3, 3].max(0) + 30, 0.05, max_depth=30)
    K = np.array([[60, 0, 63.5], [0, 60, 31.5], [0, 0, 1]])
    with torch.no_grad():
        for i0, i1 in io.batches(n, 4):
            vol.integrate(1 / pred(io.network_input(frames[i0:i1])), K, P[i0:i1], torch.from_numpy(frames[i0:i1]).cuda())
    verts, faces, colors = vol.mesh()
    assert len(f) > 0
    assert (len(v), len(f)) == (len(verts), len(faces))
    assert np.array_equal(v, verts.cpu().numpy()) and np.array_equal(f, faces.cpu().numpy())
