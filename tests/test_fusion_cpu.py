"""Dense reconstruction without a device: the fp64 oracle on analytic scenes, the marching-cubes table, the C ABI's argument
checks, calib.txt scaling, PLY round trips and run_fusion.py's refusals."""
import ctypes
import os
import sys

import numpy as np
import pytest

from oracle import fusion as OF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_plane_gives_the_signed_distance_inside_the_band_only():
    v, trunc = 0.1, 0.35
    g = OF.Grid((-1.6, -1.6, 0.05), v, (32, 32, 40))
    K = np.array([[40.0, 0, 31.5], [0, 40.0, 31.5], [0, 0, 1]])
    depth = np.full((64, 64), 2.0)
    upd, amb = OF.integrate(g, depth, K, np.eye(4), trunc, 80.0)
    z = g.centres()[..., 2]
    x, y = g.centres()[..., 0], g.centres()[..., 1]
    u, vv = np.floor(40 * x / z + 31.5 + 0.5), np.floor(40 * y / z + 31.5 + 0.5)
    seen = (u >= 0) & (u < 64) & (vv >= 0) & (vv < 64)
    band = seen & (np.abs(2.0 - z) <= trunc)
    assert np.array_equal(upd, band) and band.sum() > 1000
    assert np.array_equal(g.tsdf[band], (2.0 - z[band]) / trunc)
    assert np.all(g.w[band] == 1) and np.all(g.w[~band] == 0) and np.all(g.tsdf[~band] == 0)


def _sphere_grid(n=48, v=0.05, r=1.03, c=(1.21, 1.2, 1.19)):
    g = OF.Grid((0.0, 0.0, 0.0), v, (n, n, n))
    d = np.linalg.norm(g.centres() - np.asarray(c), axis=-1) - r
    return g, d, c, r


def test_oracle_marching_cubes_on_a_sphere_is_closed_welded_and_on_the_surface():
    g, d, c, r = _sphere_grid()
    tris, verts = OF.marching_cubes(d, np.ones_like(d), np.zeros(d.shape + (3,)), g.lo, g.v)
    keys = np.array(sorted(verts))
    faces = np.searchsorted(keys, tris)
    assert len(faces) > 500
    assert OF.euler_characteristic(faces) == 2
    # closed and consistently oriented: every directed edge once, and its reverse once
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    de = set(map(tuple, e.tolist()))
    assert len(de) == len(e) and all((b, a) in de for a, b in de)
    pos = np.stack([verts[k][0] for k in keys])
    # linear interpolation of the sampled distance, 20 voxels to the radius: within 1 % of a voxel of the sphere
    assert np.abs(np.linalg.norm(pos - np.asarray(c), axis=1) - r).max() < 0.01 * g.v


def test_marching_cubes_table_is_the_derived_one():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_mc_tables
    from scsfm import mc_tables
    assert make_mc_tables.rows() == mc_tables.TRI_TABLE
    assert len(mc_tables.TRI_TABLE) == 256 and all(len(r) == 16 and r[-1] == -1 for r in mc_tables.TRI_TABLE)
    for m, row in enumerate(mc_tables.TRI_TABLE):      # the triangles use exactly the edges whose corners differ
        crossing = {e for e, (a, b) in enumerate(mc_tables.EDGES) if ((m >> a) & 1) != ((m >> b) & 1)}
        assert {e for e in row if e >= 0} == crossing, m


def _edge_faces(tris):
    """{undirected edge: list of directed edges} of a triangle list of vertex keys."""
    out = {}
    for t in np.asarray(tris).tolist():
        for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
            out.setdefault((min(a, b), max(a, b)), []).append((a, b))
    return out


def test_every_pair_of_face_sharing_cells_meshes_to_a_manifold():
    """Two cells sharing a face, for every configuration of their 12 corners along each axis (all 256 x 16 x 3 pairs that
    agree on the shared face): no triangle twice, every edge with at most two faces in opposite directions, and every
    edge in the shared face with exactly two, one from each cell."""
    bits = (np.arange(4096)[:, None] >> np.arange(12)[None]) & 1
    for axis in range(3):
        shape = [2, 2, 2]
        shape[axis] = 3
        nx, ny = shape[0], shape[1]
        for m in bits:
            tsdf = np.where(m.reshape(shape), -1.0, 1.0)
            tris, _ = OF.marching_cubes(tsdf, np.ones(shape), np.zeros(tuple(shape) + (3,)), (0, 0, 0), 1.0)
            if not len(tris):
                continue
            canon = OF.canonical_triangles(tris)
            assert len(np.unique(canon, axis=0)) == len(canon), (axis, m)
            for (a, b), dirs in _edge_faces(tris).items():
                assert len(dirs) <= 2 and len(set(dirs)) == len(dirs), (axis, m, a, b, dirs)
                vox = [((k // 3) % nx, (k // 3 // nx) % ny, k // 3 // (nx * ny))[axis] for k in (a, b)]
                in_face = all(v == 1 and k % 3 != axis for v, k in zip(vox, (a, b)))
                assert not in_face or len(dirs) == 2, (axis, m, a, b)


def test_marching_cubes_on_a_rough_field_is_a_manifold():
    """A smoothed random field has many ambiguous faces: the welded mesh still has no doubled triangle and no edge with more
    than two faces, and every edge away from the grid's border has exactly two, in opposite directions."""
    rng = np.random.default_rng(4)
    f = rng.standard_normal((24, 24, 24))
    for ax in range(3):
        f = (np.roll(f, 1, ax) + f + np.roll(f, -1, ax)) / 3
    tris, verts = OF.marching_cubes(f, np.ones_like(f), np.zeros(f.shape + (3,)), (0, 0, 0), 1.0)
    assert len(tris) > 10000
    canon = OF.canonical_triangles(tris)
    assert len(np.unique(canon, axis=0)) == len(canon)
    n = f.shape[0]
    for (a, b), dirs in _edge_faces(tris).items():
        assert len(dirs) <= 2 and len(set(dirs)) == len(dirs)
        ijk = [((k // 3) % n, (k // 3 // n) % n, k // 3 // (n * n)) for k in (a, b)]
        inner = all(0 < c < n - 1 for v in ijk for c in v)
        assert not inner or len(dirs) == 2


def _vol(nb=(4, 4, 4), voxel=0.1):
    from scsfm import fusion
    v = fusion.Volume((ctypes.c_double * 3)(0, 0, 0), voxel, (ctypes.c_float * 3)(0, 0, 0), voxel, 4 * voxel, 80.0,
                      (ctypes.c_int * 3)(*nb))
    return fusion, v


def test_fusion_abi_argument_errors_are_reported_without_a_gpu():
    from scsfm import lib
    fusion, vol = _vol()
    L = fusion._bind()
    n0 = lib.launch_count()
    fake = ctypes.c_void_p(16)
    frames = (fusion.Frame * 17)(*[fusion.Frame(depth=16) for _ in range(17)])
    assert L.scsfm_fusion_alloc(None, 1, 8, 8, ctypes.byref(vol), fake, fake, 1, fake, fake, 4, None) == -1
    assert b"null frames" in L.scsfm_last_error()
    assert L.scsfm_fusion_alloc(frames, 1, 8, 8, ctypes.byref(vol), None, fake, 1, fake, fake, 4, None) == -1
    assert b"null pointer" in L.scsfm_last_error()
    assert L.scsfm_fusion_alloc(frames, 17, 8, 8, ctypes.byref(vol), fake, fake, 1, fake, fake, 4, None) == -1
    assert b"1..16" in L.scsfm_last_error()
    assert L.scsfm_fusion_integrate(frames, 0, 8, 8, ctypes.byref(vol), fake, fake, 1, fake, None) == -1
    assert L.scsfm_fusion_integrate(frames, 2, 0, 8, ctypes.byref(vol), fake, fake, 1, fake, None) == -1
    assert b"image size" in L.scsfm_last_error()
    frames[0].depth = None
    assert L.scsfm_fusion_integrate(frames, 1, 8, 8, ctypes.byref(vol), fake, fake, 1, fake, None) == -1
    assert b"null depth" in L.scsfm_last_error()
    _, bad = _vol(nb=(0, 4, 4))
    assert L.scsfm_fusion_sample(ctypes.byref(bad), fake, fake, fake, 4, fake, None) == -1
    assert b"positive" in L.scsfm_last_error()
    _, big = _vol(nb=(2048, 1024, 1024))
    assert L.scsfm_fusion_mesh_count(ctypes.byref(big), fake, fake, fake, 1, fake, fake, None) == -1
    assert b"2^31" in L.scsfm_last_error()
    _, vol0 = _vol(voxel=0.0)
    assert L.scsfm_fusion_mesh_emit(ctypes.byref(vol0), fake, fake, fake, 1, fake, fake, fake, fake, fake, None) == -1
    assert L.scsfm_fusion_mesh_emit(ctypes.byref(vol), fake, fake, fake, 0, fake, fake, fake, fake, fake, None) == -1
    assert L.scsfm_fusion_sample(ctypes.byref(vol), fake, None, fake, 4, fake, None) == -1
    assert lib.launch_count() == n0
    with pytest.raises(ValueError, match="fusion_sample"):
        lib.check(-1, "scsfm_fusion_sample")


def test_volume_refuses_bad_boxes_before_touching_a_device():
    from scsfm.fusion import TSDFVolume
    with pytest.raises(ValueError, match=r"2\^31 - 1; a voxel size of ([0-9.]+) or more fits"):
        TSDFVolume((-500, -500, -500), (500, 500, 500), 0.05)
    with pytest.raises(ValueError, match="voxel_size"):
        TSDFVolume((0, 0, 0), (1, 1, 1), 0)
    with pytest.raises(ValueError, match="hi must exceed lo"):
        TSDFVolume((0, 0, 0), (1, 0, 1), 0.1)
    with pytest.raises(ValueError, match="lo"):
        TSDFVolume((0, 0, float("nan")), (1, 1, 1), 0.1)
    with pytest.raises(ValueError, match="CUDA"):
        TSDFVolume((0, 0, 0), (1, 1, 1), 0.1, device="cpu")


def test_suggested_voxel_size_fits():
    from scsfm.fusion import TSDFVolume
    with pytest.raises(ValueError) as e:
        TSDFVolume((-600, -100, -600), (600, 100, 600), 0.02)
    fit = float(str(e.value).split("a voxel size of ")[1].split()[0])
    nb = np.ceil(np.array([1200, 200, 1200]) / (8 * fit))
    assert np.prod(nb) <= 2 ** 31 - 1


def _calib(path):
    with open(path, "w") as f:
        for i, fx in enumerate((718.856, 718.856, 718.856, 718.856)):
            f.write("P%d: %g 0 607.1928 %g 0 %g 185.2157 0 0 0 1 0\n" % (i, fx, 45.38 * i, fx))


def test_calib_scaling_is_the_number_the_odometry_preparation_gives(tmp_path):
    from PIL import Image
    from scsfm import inference_io as io
    from scsfm import prepare
    seq = tmp_path / "sequences" / "03"
    for c in ("2", "3"):
        os.makedirs(seq / ("image_" + c))
        Image.fromarray(np.zeros((376, 1241, 3), np.uint8)).save(seq / ("image_" + c) / "000000.png")
    _calib(seq / "calib.txt")
    scenes = prepare.KittiOdom(str(tmp_path), 256, 832).collect(str(seq))
    K = io.odom_intrinsics(str(seq / "calib.txt"), 2, (376, 1241), (256, 832))
    assert K.dtype == np.float32 and np.array_equal(scenes[0].intrinsics, K)
    assert K[0, 0] == np.float32(np.float32(718.856) * (832 / 1241))


def test_ply_written_and_read_back_is_identical(tmp_path):
    from scsfm import inference_io as io
    rng = np.random.default_rng(0)
    verts = rng.standard_normal((57, 3)).astype(np.float32)
    faces = rng.integers(0, 57, (91, 3))
    colors = rng.integers(0, 256, (57, 3)).astype(np.uint8)
    io.write_ply(str(tmp_path / "m.ply"), verts, faces, colors)
    v, f, c = io.read_ply(str(tmp_path / "m.ply"))
    assert np.array_equal(v, verts) and np.array_equal(f, faces) and np.array_equal(c, colors)
    assert open(tmp_path / "m.ply", "rb").read().startswith(b"ply\nformat binary_little_endian 1.0\n")
    io.write_ply(str(tmp_path / "e.ply"), np.zeros((0, 3)), np.zeros((0, 3), np.int64), np.zeros((0, 3)))
    assert [len(x) for x in io.read_ply(str(tmp_path / "e.ply"))] == [0, 0, 0]
    with pytest.raises(ValueError):
        io.write_ply(str(tmp_path / "x.ply"), verts, faces + 57, colors)


def _sequence(tmp_path, n, calib=True):
    from PIL import Image
    seq = tmp_path / "seqs" / "05"
    os.makedirs(seq / "image_2")
    for i in range(n):
        Image.fromarray(np.zeros((64, 96, 3), np.uint8)).save(seq / "image_2" / ("%06d.png" % i))
    if calib:
        _calib(seq / "calib.txt")
    return str(tmp_path / "seqs") + "/"


def _poses(tmp_path, n):
    p = np.tile(np.eye(4)[:3].reshape(1, 12), (n, 1))
    np.savetxt(tmp_path / "poses.txt", p)
    return str(tmp_path / "poses.txt")


def test_run_fusion_refuses_missing_voxel_size_pose_mismatch_and_missing_camera(tmp_path, capsys):
    import run_fusion
    d = _sequence(tmp_path, 4, calib=False)
    base = ["--pretrained-dispnet", "none.tar", "--dataset-dir", d, "--sequence", "05", "--output", str(tmp_path / "o.ply")]
    with pytest.raises(SystemExit):
        run_fusion.main(base + ["--poses", _poses(tmp_path, 4)])
    assert "--voxel-size" in capsys.readouterr().err
    with pytest.raises(SystemExit, match="3 poses for 4 frames"):
        run_fusion.main(base + ["--poses", _poses(tmp_path, 3), "--voxel-size", "0.2"])
    with pytest.raises(SystemExit, match="--intrinsics"):
        run_fusion.main(base + ["--poses", _poses(tmp_path, 4), "--voxel-size", "0.2"])
    with pytest.raises(SystemExit, match="positive"):
        run_fusion.main(base + ["--poses", _poses(tmp_path, 4), "--voxel-size", "0"])


def test_run_fusion_intrinsics_from_calib_or_the_command_line(tmp_path):
    import run_fusion
    d = _sequence(tmp_path, 2)
    seq = os.path.join(d, "05")
    first = os.path.join(seq, "image_2", "000000.png")
    a = run_fusion.parser.parse_args(["--pretrained-dispnet", "x", "--dataset-dir", d, "--poses", "p", "--voxel-size", "1",
                                      "--output", "o", "--img-height", "32", "--img-width", "64"])
    K = run_fusion.intrinsics(a, seq, first)
    assert K[0, 0] == np.float32(np.float32(718.856) * (64 / 96)) and K[1, 2] == np.float32(np.float32(185.2157) * (32 / 64))
    a.no_resize = True
    assert run_fusion.intrinsics(a, seq, first)[0, 0] == np.float32(718.856)
    a.intrinsics = [10.0, 11.0, 12.0, 13.0]
    assert np.array_equal(run_fusion.intrinsics(a, seq, first), [[10, 0, 12], [0, 11, 13], [0, 0, 1]])
