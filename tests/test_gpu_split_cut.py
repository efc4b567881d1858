"""The occlusion split on one GPU cuts the two depth slabs by depth-key VALUE and depth-sorts only the near list and the
far splats that survive the cull against the saturated tiles (DESIGN.md section 4).  Whatever the key distribution --
a cut inside a run of equal keys, every key equal, no far survivor, nearly all survivors, almost nothing visible -- the
frame must be byte-identical to the one-pass frame, and the debug read-backs of the depth order must still be the complete
stable order of all V splats."""
import numpy as np
import pytest

from helpers import make_args, make_generic

pytestmark = pytest.mark.gpu


def _render(ws, ctx, cloud, pos, rot, W, H, fmt, split, clear=(0.1, 0.2, 0.3, 0.4)):
    import torch
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, fmt, cloud["sh_deg"], cloud["compressed"])
    r.set_occlusion_split(split)
    r.prepare(None, pc, make_args(ws, cloud, pos, rot, W, H, fovx, fovy))
    dt = {0: torch.uint8, 1: torch.float16, 2: torch.float32}[fmt]
    t = torch.empty((H, W, 4), dtype=dt, device="cuda")
    r.render(t, pc, clear)
    torch.cuda.synchronize()
    return r, t.cpu().numpy()


def _check_split(ws, orc, ctx, cloud, az, W, H, fmt=None):
    fmt = ws.FORMAT_RGBA32_FLOAT if fmt is None else fmt
    pos, rot = ws.synth.orbit_camera(az)
    r0, img0 = _render(ws, ctx, cloud, pos, rot, W, H, fmt, split=False)
    r1, img1 = _render(ws, ctx, cloud, pos, rot, W, H, fmt, split=True)
    assert np.array_equal(img0.view(np.uint8), img1.view(np.uint8)), "split frame differs from the one-pass frame"
    s0, s1 = r0.stats(), r1.stats()
    V = s0["num_visible"]
    assert s1["num_visible"] == V and s1["num_pairs"] <= s0["num_pairs"]
    keys = r1.read_buffer(ws.BUF_DEPTH_KEYS)
    assert len(keys) == V and np.array_equal(keys, r0.read_buffer(ws.BUF_DEPTH_KEYS))
    sk, order = orc.sort_pairs(keys, np.arange(V, dtype=np.uint32))
    assert np.array_equal(r1.read_buffer(ws.BUF_SORTED_KEYS), sk)
    assert np.array_equal(r1.read_buffer(ws.BUF_SORTED_INDICES), order)
    assert np.array_equal(r0.read_buffer(ws.BUF_SORTED_INDICES), order)
    return V, keys, s0, s1


def _cloud(ws, n, seed, compressed):
    return ws.synth.make_cloud_compressed(n, seed, codebook=512) if compressed else ws.synth.make_cloud(n, seed)


@pytest.mark.parametrize("compressed", [False, True])
def test_cut_inside_a_run_of_equal_keys(ws, orc, ctx, compressed):
    """Half of the cloud at ONE position, nearer than most of the rest: the near quarter ends inside that run of equal
    keys, which must fall on one side of the cut as a whole."""
    cloud = _cloud(ws, 40000, 31, compressed)
    pos, _ = ws.synth.orbit_camera(60.0)
    g = cloud["gaussians"]
    dist = np.linalg.norm(g["xyz"] - pos, axis=1)
    anchor = g["xyz"][np.argsort(dist)[len(dist) * 3 // 10]].copy()
    g["xyz"][::2] = anchor
    V, keys, _, _ = _check_split(ws, orc, ctx, cloud, 60.0, 320, 200)
    vals, cnt = np.unique(keys, return_counts=True)
    run = vals[cnt.argmax()]
    assert cnt.max() >= 0.4 * V, "the run of equal keys is not there"
    nearer = (keys > run).sum()
    assert nearer < V // 4 <= nearer + cnt.max(), "the near quarter does not end inside the run"


@pytest.mark.parametrize("compressed", [False, True])
def test_all_keys_equal(ws, orc, ctx, compressed):
    cloud = _cloud(ws, 3000, 32, compressed)
    cloud["gaussians"]["xyz"][:] = np.float32(0.125)
    V, keys, _, _ = _check_split(ws, orc, ctx, cloud, 20.0, 160, 96)
    assert V > 0 and (keys == keys[0]).all()


def test_dense_scene_no_far_survivor(ws, orc, ctx):
    """The nearest 8 % of the splats are large and opaque: the near slab saturates every tile and the far cull keeps
    nothing, so the frame emits exactly the pairs of the splats above one key boundary, which lies within 15-35 % of V."""
    az, W, H = 30.0, 160, 100
    cloud = ws.synth.make_cloud(40000, 33)
    pos, _ = ws.synth.orbit_camera(az)
    g = cloud["gaussians"]
    depth = (g["xyz"] - pos) @ (-pos / np.linalg.norm(pos))               # view-space z along the camera axis
    front = np.argsort(depth)[: len(depth) * 8 // 100]
    g["opacity"][front] = np.float16(1.0)
    g["cov"][front] = np.array([1, 0, 0, 1, 0, 1], np.float16)
    V, keys, s0, s1 = _check_split(ws, orc, ctx, cloud, az, W, H)
    rc = _render(ws, ctx, cloud, pos, ws.synth.orbit_camera(az)[1], W, H, ws.FORMAT_RGBA32_FLOAT, True)[0].read_buffer(ws.BUF_TILE_RECTS)
    pairs = rc[:, 2].astype(np.int64) * rc[:, 3]
    o = np.argsort(-keys.astype(np.int64), kind="stable")                 # nearest first
    ks, cum = keys[o], np.concatenate([[0], np.cumsum(pairs[o])])
    lo, hi = int(0.15 * V), int(0.35 * V)
    at_boundary = [i for i in range(lo, hi + 1) if i == V or ks[i - 1] != ks[i]]
    assert s1["num_pairs"] in set(cum[at_boundary].tolist()), (s1["num_pairs"], s0["num_pairs"])
    assert s1["num_pairs"] < s0["num_pairs"]


@pytest.mark.parametrize("compressed", [False, True])
def test_sparse_scene_nearly_all_survive(ws, orc, ctx, compressed):
    """A few thousand splats over a large viewport: hardly a tile saturates, almost every far splat is binned."""
    cloud = _cloud(ws, 4000, 34, compressed)
    _, _, s0, s1 = _check_split(ws, orc, ctx, cloud, 250.0, 1280, 720, ws.FORMAT_RGBA16_FLOAT)
    assert s1["num_pairs"] >= 0.9 * s0["num_pairs"]


@pytest.mark.parametrize("compressed,n", [(False, 0), (False, 1), (False, 2), (False, 3), (False, 5),
                                          (True, 0), (True, 2), (True, 3), (True, 5)])   # (the compressed generator needs n != 1)
def test_tiny_visible_sets(ws, orc, ctx, compressed, n):
    cloud = _cloud(ws, n, 35 + n, compressed)
    V, _, _, _ = _check_split(ws, orc, ctx, cloud, 0.0, 64, 48, ws.FORMAT_RGBA8_UNORM)
    assert V <= n


def test_nothing_visible(ws, orc, ctx):
    """V = 0 with a non-empty cloud: the camera looks away."""
    import torch
    cloud = ws.synth.make_cloud(3000, 2)
    _, rot = ws.synth.fixed_camera()
    pos = np.array([0, 0, 3], np.float32)
    imgs = [_render(ws, ctx, cloud, pos, rot, 64, 48, ws.FORMAT_RGBA32_FLOAT, split)[1] for split in (False, True)]
    assert np.array_equal(imgs[0], imgs[1])
    r, _ = _render(ws, ctx, cloud, pos, rot, 64, 48, ws.FORMAT_RGBA32_FLOAT, True)
    assert r.num_visible_points() == 0 and len(r.read_buffer(ws.BUF_SORTED_INDICES)) == 0
    torch.cuda.synchronize()


def test_split_frames_replayed_as_cuda_graph(ws, ctx):
    """With timing off the split frame (cut histogram, two compactions, two depth sorts) is one captured graph; replayed
    back to back on one stream it gives the directly launched frames."""
    import torch
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    ref = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    for x in (r, ref):
        x.set_occlusion_split(True)
    r.set_timing(False)
    ref.set_cuda_graphs(False)
    stream = torch.cuda.Stream()
    cloud = ws.synth.make_cloud(150000, 36)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    W, H = 320, 200
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    outs = []
    for az in (10.0, 130.0, 250.0, 10.0):
        pos, rot = ws.synth.orbit_camera(az)
        args = make_args(ws, cloud, pos, rot, W, H, fovx, fovy)
        t = torch.empty((H, W, 4), dtype=torch.float32, device="cuda")
        r.prepare(stream, pc, args)
        r.render(t, pc, stream=stream)
        t2 = torch.empty_like(t)
        ref.prepare(None, pc, args)
        ref.render(t2, pc)
        outs.append((t, t2))
    torch.cuda.synchronize()
    for t, t2 in outs:
        assert torch.equal(t, t2)
    assert torch.equal(outs[0][0], outs[3][0])
    assert r.stats()["num_pairs"] == ref.stats()["num_pairs"]
