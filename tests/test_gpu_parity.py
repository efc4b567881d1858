"""GPU parity tests: the sm_90a path, called through the C ABI, against the CPU oracle.

Bars (DESIGN.md "Parity"):
  stage 1 raw layout      bit-exact (visible set, 10 halves, depth key, tile rect, V, P)
  stage 2 sort            bit-exact (sorted keys, payload permutation, stability); reference KAT
  binning + tile sort     bit-exact ((tile, slot) pair list, tile ranges)
  stage 3 image           |cuda - oracle| <= 2e-3 + sens(pixel) in f32; sens = oracle's bound on
                          contributions whose discard test a > 2*CUTOFF lies within 1e-4 of the threshold
"""
import os

import numpy as np
import pytest

from helpers import check_all_stages, frame, image_close, make_args, make_generic

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_sort_kat_from_reference(ws, ctx):
    """GPURSSorter::test_sort (gpu_rs.rs:295-331) through the C ABI."""
    z = np.load(os.path.join(GOLDEN, "sort_kat.npz"))
    keys, vals = ws.sort_pairs_host(ctx, z["keys_in"].view(np.uint32).copy(), np.arange(8192, dtype=np.uint32))
    assert np.array_equal(keys.view(np.float32), z["keys_out"])
    assert np.array_equal(vals, np.arange(8191, -1, -1, dtype=np.uint32))


@pytest.mark.parametrize("n", [1, 31, 4095, 4096, 4097, 12289, 1_000_003])
def test_sort_matches_stable_sort(ws, ctx, n):
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 1 << 32, size=n, dtype=np.uint64).astype(np.uint32)
    keys[: n // 3] &= 0x3ff                                   # heavy ties: stability
    keys[n // 2: n // 2 + n // 8] = 0xffffffff                # real keys equal to the pad value
    k, v = ws.sort_pairs_host(ctx, keys.copy(), np.arange(n, dtype=np.uint32))
    o = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[o]) and np.array_equal(v, o.astype(np.uint32))


@pytest.mark.parametrize("bits", [8, 13, 24])
def test_sort_partial_key_bits(ws, ctx, bits):
    rng = np.random.default_rng(bits)
    n = 100_000
    keys = rng.integers(0, 1 << bits, size=n, dtype=np.uint64).astype(np.uint32)
    k, v = ws.sort_pairs_host(ctx, keys.copy(), np.arange(n, dtype=np.uint32), key_bits=bits)
    o = np.argsort(keys, kind="stable")
    assert np.array_equal(k, keys[o]) and np.array_equal(v, o.astype(np.uint32))


def test_golden_frame(ws, orc, ctx):
    """The committed golden vectors (tests/golden/oracle_small.npz)."""
    z = np.load(os.path.join(GOLDEN, "oracle_small.npz"))
    cloud = ws.synth.make_cloud(int(z["n"]), int(z["seed"]))
    pos, rot = ws.synth.orbit_camera(float(z["az"]))
    W, H = int(z["W"]), int(z["H"])
    r, pc, img, _ = frame(ws, ctx, cloud, pos, rot, W, H)
    assert np.array_equal(r.read_buffer(ws.BUF_SPLATS_2D), z["splats"])
    assert np.array_equal(r.read_buffer(ws.BUF_DEPTH_KEYS), z["keys"])
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_INDICES), z["order"])
    assert r.stats()["num_pairs"] == int(z["pairs"])
    assert np.abs(img - z["image"]).max() <= 4e-3 and np.abs(img - z["image"]).mean() <= 2e-5


@pytest.mark.parametrize("n,W,H,az", [(5000, 320, 200, 30.0), (40000, 800, 600, 140.0), (40000, 1200, 799, 250.0), (777, 33, 17, 0.0)])
def test_all_stages_small(ws, orc, ctx, n, W, H, az):
    cloud = ws.synth.make_cloud(n, 100 + n)
    pos, rot = ws.synth.orbit_camera(az)
    check_all_stages(ws, orc, ctx, cloud, pos, rot, W, H)


def test_cfg1_full(ws, orc, ctx):
    """BASELINE.json configs[0]: 100K Gaussians, 800x600, fixed camera."""
    n, W, H, seed, _ = ws.synth.CONFIGS["cfg1"]
    cloud = ws.synth.make_cloud(n, seed)
    pos, rot = ws.synth.fixed_camera()
    check_all_stages(ws, orc, ctx, cloud, pos, rot, W, H)


@pytest.mark.parametrize("deg", [0, 1, 2])
def test_lower_sh_degree(ws, orc, ctx, deg):
    cloud = ws.synth.make_cloud(20000, 5)
    pos, rot = ws.synth.orbit_camera(80.0)
    check_all_stages(ws, orc, ctx, cloud, pos, rot, 400, 300, max_sh_deg=deg)


def test_options_mip_kernel_scaling_walltime(ws, orc, ctx):
    """§8(f) N4 options: mip-splatting compensation, kernel size, gaussian_scaling, walltime reveal."""
    cloud = ws.synth.make_cloud(20000, 6)
    pos, rot = ws.synth.orbit_camera(10.0)
    check_all_stages(ws, orc, ctx, cloud, pos, rot, 400, 300, mip_splatting=True, kernel_size=0.1)
    check_all_stages(ws, orc, ctx, cloud, pos, rot, 400, 300, gaussian_scaling=0.5)
    check_all_stages(ws, orc, ctx, cloud, pos, rot, 400, 300, walltime=0.6)       # partially revealed: NaN axes vanish


def test_options_clipping_box_and_background(ws, orc, ctx):
    """§8(f) N4: an explicit clipping box (preprocess.wgsl:177) through every stage, and the `Display` pass
    (renderer.rs:556-583: the splat frame blended PREMULTIPLIED over a target cleared with the background colour)
    expressed as render(clear = background)."""
    cloud = ws.synth.make_cloud(20000, 12)
    pos, rot = ws.synth.orbit_camera(200.0)
    box = ws.Aabb([-0.5, -1.0, -0.25], [0.75, 0.5, 1.0])
    r, st, _ = check_all_stages(ws, orc, ctx, cloud, pos, rot, 400, 300, clipping_box=box)
    full = frame(ws, ctx, cloud, pos, rot, 400, 300)[0].stats()["num_visible"]
    assert 0 < st["num_visible"] < full
    bg = (0.2, 0.4, 0.6, 1.0)
    _, _, on_bg, _ = frame(ws, ctx, cloud, pos, rot, 400, 300, clear=bg)
    _, _, on_zero, _ = frame(ws, ctx, cloud, pos, rot, 400, 300)
    want = on_zero + (1.0 - on_zero[..., 3:4]) * np.asarray(bg, np.float32)        # src + dst * (1 - src.a)
    assert np.abs(on_bg - want).max() < 2e-6


def test_occlusion_split_is_bit_identical(ws, orc, ctx):
    """Two depth slabs with saturated-tile culling of the far one: same pixels, bit for bit, from fewer pairs."""
    cases = [(ws.synth.make_cloud(150000, 21), 80, 50, 30.0, ws.FORMAT_RGBA32_FLOAT),        # ~400 layers per pixel: the near slab saturates every tile
             (ws.synth.make_cloud(150000, 21), 320, 200, 200.0, ws.FORMAT_RGBA16_FLOAT),
             (ws.synth.make_cloud(20000, 22), 800, 600, 75.0, ws.FORMAT_RGBA8_UNORM),        # sparse: few do
             (ws.synth.make_cloud_compressed(60000, 23), 640, 360, 140.0, ws.FORMAT_RGBA32_FLOAT),
             (ws.synth.make_cloud(5, 24), 64, 48, 0.0, ws.FORMAT_RGBA32_FLOAT),               # split point 0: empty far slab
             (ws.synth.make_cloud(0, 25), 64, 48, 0.0, ws.FORMAT_RGBA32_FLOAT)]
    saved = []
    for cloud, W, H, az, fmt in cases:
        pos, rot = ws.synth.orbit_camera(az)
        clear = (0.1, 0.2, 0.3, 0.4)
        r0, _, img0, _ = frame(ws, ctx, cloud, pos, rot, W, H, fmt=fmt, clear=clear, split=False)
        r1, _, img1, _ = frame(ws, ctx, cloud, pos, rot, W, H, fmt=fmt, clear=clear, split=True)
        assert np.array_equal(img0.view(np.uint8), img1.view(np.uint8))
        s0, s1 = r0.stats(), r1.stats()
        assert s1["num_visible"] == s0["num_visible"] and s1["num_pairs"] <= s0["num_pairs"]
        saved.append(s1["num_pairs"] / max(s0["num_pairs"], 1))
    assert saved[0] < 0.8, saved                         # the dense case really drops pairs
    # a renderer can switch back and forth between frames (the CUDA graph is re-captured)
    cloud, W, H, az, fmt = cases[0]
    pos, rot = ws.synth.orbit_camera(az)
    import torch
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, fmt, 3, False)
    args = make_args(ws, cloud, pos, rot, W, H, fovx, fovy)
    outs = []
    for split in (True, False, True, True):
        r.set_occlusion_split(split)
        r.prepare(None, pc, args)
        t = torch.empty((H, W, 4), dtype=torch.float32, device="cuda")
        r.render(t, pc)
        torch.cuda.synchronize()
        outs.append(t.cpu().numpy())
    assert all(np.array_equal(outs[0], o) for o in outs[1:])


def test_edge_cases(ws, orc, ctx):
    import torch
    pos, rot = ws.synth.fixed_camera()
    # empty cloud
    c0 = ws.synth.make_cloud(0, 1)
    r, pc, img, _ = frame(ws, ctx, c0, pos, rot, 64, 48, clear=(0.25, 0.5, 0.75, 1.0))
    assert r.num_visible_points() == 0 and r.stats()["num_pairs"] == 0
    assert np.allclose(img, (0.25, 0.5, 0.75, 1.0))
    # everything culled (camera looks away)
    c1 = ws.synth.make_cloud(3000, 2)
    r, pc, img, _ = frame(ws, ctx, c1, np.array([0, 0, 3], np.float32), rot, 64, 48)
    assert r.num_visible_points() == 0 and np.count_nonzero(img) == 0
    # one huge splat covering every tile + a few small ones
    c2 = ws.synth.make_cloud(300, 3)
    c2["gaussians"]["cov"][0] = np.array([4, 0.01, 0, 4, 0, 4], np.float16)
    check_all_stages(ws, orc, ctx, c2, pos, rot, 330, 250)


def test_output_formats(ws, orc, ctx):
    cloud = ws.synth.make_cloud(20000, 9)
    pos, rot = ws.synth.orbit_camera(300.0)
    W, H = 400, 300
    clear = (0.1, 0.2, 0.3, 1.0)
    _, _, f32, _ = frame(ws, ctx, cloud, pos, rot, W, H, ws.FORMAT_RGBA32_FLOAT, clear)
    _, _, f16, _ = frame(ws, ctx, cloud, pos, rot, W, H, ws.FORMAT_RGBA16_FLOAT, clear)
    _, _, u8, _ = frame(ws, ctx, cloud, pos, rot, W, H, ws.FORMAT_RGBA8_UNORM, clear)
    assert np.array_equal(f16, f32.astype(np.float16))
    assert np.array_equal(u8, np.rint(np.clip(f32, 0, 1) * 255).astype(np.uint8))


def test_render_to_host_and_reuse(ws, orc, ctx):
    """render_to_host == render + copy; a renderer serves several clouds / viewports in a row
    (sort buffers re-created when the point count changes, renderer.rs:200-211)."""
    import torch
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA16_FLOAT, 3, False)
    for n, W, H in ((3000, 160, 96), (9000, 320, 200), (3000, 160, 96)):
        cloud = ws.synth.make_cloud(n, n)
        pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
        pos, rot = ws.synth.orbit_camera(45.0)
        fovx, fovy = ws.synth.fov_for_viewport(W, H)
        args = make_args(ws, cloud, pos, rot, W, H, fovx, fovy)
        r.prepare(None, pc, args)
        host = torch.empty((H, W, 4), dtype=torch.float16).pin_memory()
        r.render_to_host(host, pc)
        dev = torch.empty((H, W, 4), dtype=torch.float16, device="cuda")
        r.render(dev, pc)
        torch.cuda.synchronize()
        assert torch.equal(dev.cpu(), host)
        ref = orc.render_frame(cloud, pos, rot, W, H, fovx, fovy)
        assert np.abs(host.numpy().astype(np.float32) - ref["image"]).max() < 6e-3


def test_errors(ws, ctx):
    cloud = ws.synth.make_cloud(2000, 4)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    import torch
    t = torch.empty((48, 64, 4), device="cuda")
    with pytest.raises(ws.WsError) as e:
        r._viewport = (64, 48); r.render(t, pc)
    assert e.value.status == ws.WS_ERR_NOT_PREPARED
    rc = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, True)
    pos, rot = ws.synth.fixed_camera()
    args = make_args(ws, cloud, pos, rot, 64, 48, *ws.synth.fov_for_viewport(64, 48))
    with pytest.raises(ws.WsError) as e:
        rc.prepare(None, pc, args)
    assert e.value.status == ws.WS_ERR_MISMATCH
    # pair overflow is reported, never silently dropped
    r.set_pair_capacity(100)
    r.prepare(None, pc, args)
    st = r.stats(allow_overflow=True)
    assert st["pair_overflow"] and st["num_pairs"] > 100
    with pytest.raises(ws.WsError) as e:
        r.stats()
    assert e.value.status == ws.WS_ERR_PAIR_OVERFLOW


def test_determinism(ws, ctx):
    """Bit-reproducible frames (the reference's atomic slot order is not, preprocess.wgsl:262)."""
    cloud = ws.synth.make_cloud(30000, 8)
    pos, rot = ws.synth.orbit_camera(120.0)
    imgs = [frame(ws, ctx, cloud, pos, rot, 512, 288)[2] for _ in range(3)]
    assert np.array_equal(imgs[0], imgs[1]) and np.array_equal(imgs[0], imgs[2])


# ---- compressed (npz / c3dgs) layout: BASELINE.json configs[3] -----------------------------------
def _check_compressed(ws, orc, ctx, cloud, pos, rot, W, H, **kw):
    """preprocess_compressed.wgsl: exact visible set and keys; halves within 1 f16 ulp (expf of the
    scale factor differs between glibc and CUDA by an ulp, which propagates into the axes); the
    image is compared against the oracle composited over the CUDA splats' own order."""
    from helpers import f16_ordered
    r, pc, img, (fovx, fovy) = frame(ws, ctx, cloud, pos, rot, W, H, **kw)
    zn, zf = orc.fit_near_far(pos, cloud["aabb_min"], cloud["aabb_max"])
    cam = orc.camera_uniform(pos, rot, fovx, fovy, zn, zf, W, H)
    st = orc.render_settings(cloud, **kw)
    osplats, okeys, _ = orc.preprocess(cloud, cam, st)
    V = len(okeys)
    assert r.num_visible_points() == V
    splats = r.read_buffer(ws.BUF_SPLATS_2D)
    assert np.array_equal(r.read_buffer(ws.BUF_DEPTH_KEYS), okeys)         # 24-bit integer keys: exact
    d = np.abs(f16_ordered(splats) - f16_ordered(osplats))
    assert d[:, 4:].max() <= 1                                             # centre, colour, opacity
    a = splats.view(np.float16).astype(np.float64); b = osplats.view(np.float16).astype(np.float64)
    for sl in (slice(0, 2), slice(2, 4)):                                  # axes as vectors (see test_oracle)
        na = np.linalg.norm(b[:, sl] * [W, H], axis=1)
        err = np.linalg.norm((a[:, sl] - b[:, sl]) * [W, H], axis=1)
        assert (err <= 4e-3 * na + 1e-3).all()
    sk, order = orc.sort_pairs(okeys, np.arange(V, dtype=np.uint32))
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_KEYS), sk)
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_INDICES), order)
    ref, sens = orc.composite(splats, order, W, H, want_sens=True)          # same splats, oracle compositor
    dd, ok = image_close(img, ref, sens)
    assert ok.all(), "image: %d px outside tolerance, max %.3g" % ((~ok).sum(), dd.max())
    # and against the all-oracle frame with the looser bound the 1-ulp splat differences allow
    ref2 = orc.composite(osplats, order, W, H)
    assert np.abs(img - ref2).max() < 2e-2 and np.abs(img - ref2).mean() < 2e-4
    return r


@pytest.mark.parametrize("identity", [False, True])
def test_compressed_layout(ws, orc, ctx, identity):
    cloud = ws.synth.make_cloud_compressed(30000, 21, codebook=512, identity_index=identity)
    pos, rot = ws.synth.orbit_camera(75.0)
    r = _check_compressed(ws, orc, ctx, cloud, pos, rot, 480, 270)
    assert r.stats()["num_pairs"] > 0


@pytest.mark.parametrize("deg", [0, 1, 2])
def test_compressed_lower_degree_files(ws, orc, ctx, deg):
    """the SH stride of a compressed cloud depends on the FILE's degree (preprocess_compressed.wgsl:147-153)"""
    cloud = ws.synth.make_cloud_compressed(8000, 22, sh_deg=deg, codebook=256)
    pos, rot = ws.synth.orbit_camera(200.0)
    _check_compressed(ws, orc, ctx, cloud, pos, rot, 320, 200, max_sh_deg=deg)


def test_cuda_graph_path_is_identical(ws, orc, ctx):
    """With timing off prepare() replays a CUDA graph; the frames must equal the direct-launch ones, also
    after the cloud / viewport changed (graph rebuild) and when frames are enqueued back to back."""
    import torch
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    ref = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    r.set_timing(False)
    ref.set_cuda_graphs(False)
    stream = torch.cuda.Stream()
    for n, W, H in ((20000, 320, 200), (20000, 320, 200), (35000, 480, 270), (20000, 320, 200)):
        cloud = ws.synth.make_cloud(n, 50 + n)
        pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
        fovx, fovy = ws.synth.fov_for_viewport(W, H)
        outs = []
        for az in (10.0, 130.0, 250.0):                      # three frames in flight on one stream
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
        assert r.stats()["num_pairs"] == ref.stats()["num_pairs"]


# ---- round 2: closed form, the independent f64 renderer and the ROP-faithful oracle, all against the CUDA path --------
def test_analytic_isotropic_gaussian_on_cuda_path(ws, ctx):
    """The closed form of tests/test_oracle.py::test_analytic_isotropic_gaussian_on_axis, evaluated on the CUDA image
    (no oracle involved): an isotropic Gaussian near the optical axis projects to an isotropic 2D Gaussian of
    variance (f sigma / z)^2 + kernel_size, alpha = min(.99, o exp(-r^2 / (2 var))) inside r^2/(2 var) <= 2 CUTOFF."""
    import math
    W = H = 257
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    sigma, o = 0.02, 0.8
    g = np.zeros(1, dtype=ws.synth.GAUSSIAN_DTYPE)
    g["xyz"] = np.asarray((0.013, 0.007, 0.0), np.float32); g["opacity"] = np.float16(o)
    g["cov"] = np.array([sigma * sigma, 0, 0, sigma * sigma, 0, sigma * sigma], np.float16)
    sh = np.zeros((1, 16, 3), np.float16)
    sh[0, 0] = (np.asarray((0.9, 0.4, 0.2), np.float64) - 0.5) / 0.28209479177387814
    cloud = dict(gaussians=g, sh_coefs=sh, num_points=1, sh_deg=3, compressed=False, aabb_min=np.array([-1, -1, -1], np.float32),
                 aabb_max=np.array([1, 1, 1], np.float32), center=np.zeros(3, np.float32))
    pos, rot = ws.synth.fixed_camera()
    for split in (False, True):
        r, pc, img, _ = frame(ws, ctx, cloud, pos, rot, W, H, split=split)
        assert r.num_visible_points() == 1
        f = H / (2 * math.tan(fovy / 2))
        var = (f * sigma / 3.0) ** 2 + 0.3
        cxp = W / 2 + f * 0.013 / 3.0; cyp = H / 2 + f * 0.007 / 3.0
        ys, xs = np.mgrid[0:H, 0:W]
        a = ((xs + 0.5 - cxp) ** 2 + (ys + 0.5 - cyp) ** 2) / (2 * var)
        alpha = np.where(a <= 2 * 2.3539888583335364, np.minimum(0.99, o * np.exp(-a)), 0.0)
        band = np.abs(a - 2 * 2.3539888583335364) < 0.15          # f16 storage of axes / centre moves the footprint edge
        assert np.abs(img[..., 3] - alpha)[~band].max() < 6e-3
        for ch, c in enumerate((0.9, 0.4, 0.2)):
            assert np.abs(img[..., ch] - c * alpha)[~band].max() < 6e-3
        assert img[..., 3].max() > 0.75 and (img[..., 3][a > 2 * 2.3539888583335364 + 0.15] == 0).all()


@pytest.mark.parametrize("az", [30.0, 200.0])
def test_cuda_image_against_independent_f64_renderer(ws, ctx, az):
    """The CUDA frame against oracle/f64_ideal.py (float64, textbook formulation, no shared code or structure with
    ws_oracle.c or the kernels): same bounds as the oracle-vs-ideal CPU test."""
    from oracle import f64_ideal, oracle as orc
    n, W, H = 3000, 160, 120
    cloud = ws.synth.make_cloud(n, 99)
    pos, rot = ws.synth.orbit_camera(az)
    clear = (0.1, 0.2, 0.3, 1.0)
    r, pc, img, (fovx, fovy) = frame(ws, ctx, cloud, pos, rot, W, H, clear=clear)
    zn, zf = orc.fit_near_far(pos, cloud["aabb_min"], cloud["aabb_max"])
    ideal, idx = f64_ideal.render(cloud, pos, rot, W, H, fovx, fovy, zn, zf, clear=clear)
    assert len(idx) == r.num_visible_points()
    d = np.abs(ideal - img)
    assert d.max() < 2e-2 and d.mean() < 1e-3, (d.max(), d.mean())


def test_target_formats_against_rop_faithful_oracle(ws, orc, ctx):
    """What the reference's OWN render target would hold (blend result rounded to the format after every layer,
    renderer.rs:63-67) vs the CUDA path's float compositor with one conversion at the end.  Bounds from the measured
    gap (profiles/r02_rop_gap.json, DESIGN.md section 5): Rgba16Float within 6e-3 of the pixel's largest channel
    (mean 1e-3); Rgba8Unorm on a scene whose colours stay <= 1: within 8 steps of 255 (mean 1.5 steps).  Per-layer
    saturation of colours > 1 in an 8-bit target is NOT reproduced by a front-to-back compositor (DESIGN.md)."""
    n, W, H = 60000, 640, 360
    cloud = ws.synth.make_cloud(n, 77)
    cloud["sh_coefs"] = cloud["sh_coefs"].copy()
    cloud["sh_coefs"][:, 1:, :] = 0                                           # view-independent colour 0.5 + C0 dc ...
    cloud["sh_coefs"][:, 0, :] = np.clip(cloud["sh_coefs"][:, 0, :], -1.7, 1.7)   # ... inside [0.02, 0.98]
    pos, rot = ws.synth.orbit_camera(140.0)
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    ref = orc.render_frame(cloud, pos, rot, W, H, fovx, fovy)
    assert ref["splats"][:, 6:9].view(np.float16).max() <= 1.0
    r8, _, img8, _ = frame(ws, ctx, cloud, pos, rot, W, H, fmt=ws.FORMAT_RGBA8_UNORM, split=True)
    rop8 = orc.composite_rop(ref["splats"], ref["order"], W, H, 0)
    gap8 = np.abs(img8.astype(np.float32) / 255.0 - rop8).max(axis=2)
    assert gap8.max() <= 8.0 / 255.0 + 1e-6 and gap8.mean() <= 1.5 / 255.0, (gap8.max() * 255, gap8.mean() * 255)
    r16, _, img16, _ = frame(ws, ctx, cloud, pos, rot, W, H, fmt=ws.FORMAT_RGBA16_FLOAT, split=True)
    rop16 = orc.composite_rop(ref["splats"], ref["order"], W, H, 1)
    rel = np.abs(img16.astype(np.float32) - rop16).max(axis=2) / np.maximum(np.abs(rop16).max(axis=2), 2.0 ** -10)
    assert rel.max() < 6e-3 + 2e-3 and rel.mean() < 1e-3, (rel.max(), rel.mean())


def test_deferred_frame_status_and_index_validation(ws, ctx):
    """(1) A frame that overflowed the pair capacity cannot fail the asynchronous call that enqueued it; the NEXT
    prepare() whose predecessor's status copy has landed returns WS_ERR_PAIR_OVERFLOW once, without synchronising.
    (2) compressed records with out-of-range codebook indices are rejected at load time (a CUDA gather would fault
    where wgpu's bounds-checked buffers read zeros).  (3) two contexts in one process (per-device kernel attributes)."""
    import torch
    cloud = ws.synth.make_cloud(3000, 4)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    pos, rot = ws.synth.fixed_camera()
    args = make_args(ws, cloud, pos, rot, 64, 48, *ws.synth.fov_for_viewport(64, 48))
    t = torch.empty((48, 64, 4), device="cuda")
    r.set_pair_capacity(100)
    r.prepare(None, pc, args); r.render(t, pc)               # enqueued fine: the overflow happens on the device
    torch.cuda.synchronize()
    with pytest.raises(ws.WsError) as e:
        r.prepare(None, pc, args)                            # reports the EARLIER frame, enqueues nothing
    assert e.value.status == ws.WS_ERR_PAIR_OVERFLOW
    r.set_pair_capacity(0)
    r.prepare(None, pc, args); r.render(t, pc)               # reported once: the renderer keeps working
    torch.cuda.synchronize()
    r.prepare(None, pc, args); r.render(t, pc)
    assert r.stats()["num_pairs"] > 100
    # (2)
    cc = ws.synth.make_cloud_compressed(2000, 9, codebook=64)
    bad = dict(cc); bad["gaussians"] = cc["gaussians"].copy()
    bad["gaussians"]["sh_idx"][17] = 64                      # one past the SH codebook
    with pytest.raises(ws.WsError) as e:
        ws.PointCloud.new(ctx, make_generic(ws, bad))
    assert e.value.status == ws.WS_ERR_INVALID_ARGUMENT
    bad["gaussians"] = cc["gaussians"].copy()
    bad["gaussians"]["geometry_idx"][5] = 0xfffffff0         # a negative i32 in the file
    with pytest.raises(ws.WsError):
        ws.PointCloud.new(ctx, make_generic(ws, bad))
    ws.PointCloud.new(ctx, make_generic(ws, cc))             # the untouched cloud loads
    # (3) a second context on the same device (and on device 1 when there is one) renders the same frame
    img0 = frame(ws, ctx, cloud, pos, rot, 320, 200)[2]
    for dev in range(min(torch.cuda.device_count(), 2)):
        ctx2 = ws.Context(dev)
        with torch.cuda.device(dev):
            pc2 = ws.PointCloud.new(ctx2, make_generic(ws, cloud))
            r2 = ws.GaussianRenderer.new(ctx2, ws.FORMAT_RGBA32_FLOAT, 3, False)
            r2.set_occlusion_split(False)
            a2 = make_args(ws, cloud, pos, rot, 320, 200, *ws.synth.fov_for_viewport(320, 200))
            r2.prepare(None, pc2, a2)
            t2 = torch.empty((200, 320, 4), dtype=torch.float32, device="cuda:%d" % dev)
            r2.render(t2, pc2)
            torch.cuda.synchronize(dev)
            assert np.array_equal(t2.cpu().numpy(), img0)


@pytest.mark.parametrize("scaling,n,W,H", [(6.0, 3000, 640, 360), (10.0, 300, 1920, 1080), (1.0, 40000, 1200, 799)])
def test_binning_large_rectangles(ws, orc, ctx, scaling, n, W, H):
    """bin_expand: rectangles above 32 tiles are expanded by the whole block, small ones by their owner thread, partitions
    with more than 4096 pairs in several chunks -- the (tile, slot) pair list, ranges and image must not care
    (gaussian_scaling blows the splats up: hundreds to thousands of tiles each, screen-filling ones included)."""
    cloud = ws.synth.make_cloud(n, 123 + n)
    pos, rot = ws.synth.orbit_camera(300.0)
    r, st, d = check_all_stages(ws, orc, ctx, cloud, pos, rot, W, H, gaussian_scaling=scaling)
    assert st["num_pairs"] > (20 * st["num_visible"] if scaling > 1 else st["num_visible"])
