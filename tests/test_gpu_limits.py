"""The renderer at the limits of its viewport and pair-count range.

The kernels change behaviour at fixed thresholds that the 1080p / 4K parity tests never cross:
  > 256 tiles          1 -> 2 tile-sort passes (capi.cu begin_frame, binning.cu ndig)
  > 65 536 tiles       2 -> 3 tile-sort passes, a third tile-digit histogram in the expand kernels
  > 262 144 tiles      the far cull reads the per-tile "saturated" byte map from global memory instead of packing it into a
                       bit map in shared memory (binning.cu done_bits_bytes / drop_saturated)
  16 384 px per side   the largest accepted viewport
  frame > 4 GiB        byte offsets of the target past 2^32 (composite.cu epilogue)
  P >= 2^31 / 2^32     64-bit pair totals, saturating partition bases, the overflow report
Bars are those of DESIGN.md section 5 (tests/helpers.check_all_stages).  The scenes fill the whole view of
synth.fixed_camera (eye (0, 0, -3) looking down +z) at depths 2..4 with a 90-degree field of view across the longer
side, so that the edge tiles and the last tile column are covered at every aspect ratio."""
import ctypes as C
import gc
import math
import time

import numpy as np
import pytest

from helpers import check_all_stages, frame, make_args, make_generic, oracle_pairs

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Frames here reach 4 GiB: give the memory back between cases."""
    yield
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _fov(W, H):
    """90 degrees across the longer side, square pixels: focal length max(W, H) / 2 px."""
    f = max(W, H) / 2.0
    return (2.0 * math.atan(W / (2.0 * f)), 2.0 * math.atan(H / (2.0 * f))), f


def _rebox(cloud):
    xyz = cloud["gaussians"]["xyz"]
    cloud["aabb_min"] = np.minimum(xyz.min(axis=0), 0.0).astype(np.float32)     # raw clouds: bbox grown from the zero box
    cloud["aabb_max"] = np.maximum(xyz.max(axis=0), 0.0).astype(np.float32)
    cloud["center"] = xyz.mean(axis=0, dtype=np.float64).astype(np.float32)


def _scene(ws, n, seed, W, H, px=6.0):
    """synth.make_cloud stretched over the view: x and y scaled to 1.05 x the frustum at depth 3 (splats up to 1.6 x
    beyond the edges at depth 2), splat sigmas around `px` pixels (rectangles of a few tiles on either side of the
    16-tile limit of the far cull)."""
    fov, f = _fov(W, H)
    px = min(px, max(W, H) / 4.0)
    cloud = ws.synth.make_cloud(n, seed)
    g = cloud["gaussians"]
    g["xyz"][:, 0] *= np.float32(3.15 * W / (2.0 * f))
    g["xyz"][:, 1] *= np.float32(3.15 * H / (2.0 * f))
    k = px * 3.0 / f / (0.6 * n ** (-1.0 / 3.0))                            # synth's sigma scale -> px pixels at depth 3
    g["cov"] = (g["cov"].astype(np.float32) * np.float32(k * k)).astype(np.float16)
    _rebox(cloud)
    return cloud, fov


def _points_for(W, H):
    """About six layers of splats per pixel (a 6-px-sigma footprint covers ~1400 px)."""
    return int(min(max(6 * W * H // 1400, 300), 300_000))


def _timed(label, fn, *a, **kw):
    t0 = time.perf_counter()
    out = fn(*a, **kw)
    print("%s: %.2f s" % (label, time.perf_counter() - t0))
    return out


def _render(ws, ctx, cloud, pc, args, W, H, split, fmt=None, clear=(0.1, 0.2, 0.3, 0.4)):
    """One frame on the device; a frame that overflows the automatic pair capacity is prepared again with the
    capacity its stats report, so that the list is complete."""
    import torch
    fmt = ws.FORMAT_RGBA32_FLOAT if fmt is None else fmt
    r = ws.GaussianRenderer.new(ctx, fmt, cloud["sh_deg"], cloud["compressed"])
    r.set_occlusion_split(split)
    r.prepare(None, pc, args)
    st = r.stats(allow_overflow=True)
    if st["pair_overflow"]:
        r.set_pair_capacity(st["num_pairs"])
        r.prepare(None, pc, args)
    t = torch.empty((H, W, 4), dtype={0: torch.uint8, 1: torch.float16, 2: torch.float32}[fmt], device="cuda")
    r.render(t, pc, clear)
    torch.cuda.synchronize()
    return r, t, r.stats()


# ---- 1. tile-count thresholds: full-stage parity with the split off, then split == one pass ---------------------------
@pytest.mark.parametrize("W,H", [(4096, 16), (4112, 16), (16, 4112),          # 256 / 257 tiles, one tile column
                                 (16384, 1024), (16384, 1040),                # 2 -> 3 tile-sort passes
                                 (16384, 4096), (16384, 4112),                # far cull: bit map -> byte map
                                 (1, 1), (1, 4097), (4097, 1),
                                 (16383, 4112)])                              # half-width 8191.5: 14 significant bits
def test_viewport_thresholds(ws, orc, ctx, W, H):
    import torch
    n = _points_for(W, H)
    cloud, fov = _scene(ws, n, 1000 + W + H, W, H)
    pos, rot = ws.synth.fixed_camera()
    t0 = time.perf_counter()
    r, st, img = check_all_stages(ws, orc, ctx, cloud, pos, rot, W, H, fov=fov)
    rng_ = r.read_buffer(ws.BUF_TILE_RANGES)
    print("%dx%d: N=%d V=%d P=%d tiles=%d (%.0f%% touched)  image max|d| %.3g mean %.3g, %.1f%% of the tolerance used  oracle %.2f s, check %.2f s" % (
        W, H, n, st["num_visible"], st["num_pairs"], st["num_tiles"], 100.0 * np.mean(rng_[:, 1] > rng_[:, 0]),
        img["max"], img["mean"], 100.0 * img["used"], img["oracle_s"], time.perf_counter() - t0))
    assert st["num_visible"] > 0 and st["num_tiles"] == ((W + 15) // 16) * ((H + 15) // 16)
    del r
    # the occlusion split (cut by key value, far cull on the bit map or, above 2^18 tiles, the byte map): the same bytes
    args = make_args(ws, cloud, pos, rot, W, H, *fov)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r0, t0_, s0 = _render(ws, ctx, cloud, pc, args, W, H, split=False)
    r1, t1_, s1 = _render(ws, ctx, cloud, pc, args, W, H, split=True)
    assert torch.equal(t0_.view(torch.uint8), t1_.view(torch.uint8)), "split frame differs from the one-pass frame"
    assert s1["num_visible"] == s0["num_visible"] and s1["num_pairs"] <= s0["num_pairs"] == st["num_pairs"]


# ---- 2. the far cull on both map layouts -------------------------------------------------------------------------------
def _opaque(g, idx, f, px=300.0):
    """large (sigma ~ px pixels at depth 2.1) opaque splats: a few hundred of them saturate every tile they cover"""
    s = px * 2.1 / f
    g["opacity"][idx] = np.float16(1.0)
    g["cov"][idx] = np.array([s * s, 0, 0, s * s, 0, s * s], np.float16)


def _dense_front(ws, W, H, seed, right_half_only):
    """The nearest 8 % of the splats large and opaque: everywhere, or only those right of the view axis (that half of
    the view, with the last tile column and the bottom-right tile, saturates in the near slab)."""
    n = _points_for(W, H)
    cloud, fov = _scene(ws, n, seed, W, H)
    g = cloud["gaussians"]
    front = np.argsort(g["xyz"][:, 2], kind="stable")[: n * 8 // 100]     # view depth = z + 3
    if right_half_only:
        front = front[g["xyz"][front, 0] > 0]
    _opaque(g, front, _fov(W, H)[1])
    return cloud, fov


def _near_candidates(r1, ws, V):
    """Per key boundary b within 15-35 % of V (nearest first): the pairs of the splats above it (the near list, if the
    cut is there), and the pairs of the splats below it with rectangles above / up to 16 tiles."""
    keys = r1.read_buffer(ws.BUF_DEPTH_KEYS)
    rc = r1.read_buffer(ws.BUF_TILE_RECTS)
    pairs = rc[:, 2].astype(np.int64) * rc[:, 3]
    o = np.argsort(-keys.astype(np.int64), kind="stable")                 # nearest first
    ks, p = keys[o], pairs[o]
    cum = np.concatenate([[0], np.cumsum(p)])
    cum_big = np.concatenate([[0], np.cumsum(np.where(p > 16, p, 0))])
    cum_small = cum - cum_big
    lo, hi = int(0.15 * V), int(0.35 * V)
    out = []
    for b in range(lo, hi + 1):
        if b == V or ks[b - 1] != ks[b]:
            out.append((int(cum[b]), int(cum_big[V] - cum_big[b]), int(cum_small[V] - cum_small[b])))
    assert out, "no key boundary within 15-35 % of V"
    return out


@pytest.mark.parametrize("H", [4096, 4112])
def test_far_cull_partial_saturation(ws, ctx, H):
    """Half of the view saturates in the near slab.  The split frame must be the one-pass frame byte for byte (a splat
    dropped wrongly changes pixels), and the far cull must drop the small far splats of the saturated half only."""
    W = 16384
    cloud, fov = _dense_front(ws, W, H, 2000 + H, right_half_only=True)
    pos, rot = ws.synth.fixed_camera()
    args = make_args(ws, cloud, pos, rot, W, H, *fov)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    import torch
    r0, t0, s0 = _timed("16384x%d one pass" % H, _render, ws, ctx, cloud, pc, args, W, H, split=False)
    r1, t1, s1 = _timed("16384x%d split" % H, _render, ws, ctx, cloud, pc, args, W, H, split=True)
    assert torch.equal(t0.view(torch.uint8), t1.view(torch.uint8)), "split frame differs from the one-pass frame"
    # the scene: the last tile column and the bottom-right tile are saturated (alpha exactly 1 over a clear alpha < 1),
    # the left quarter is not
    alpha = t0[..., 3]
    assert bool((alpha[:, -16:] == 1.0).all()) and bool((alpha[-16:, -16:] == 1.0).all())
    assert float((alpha[:, : W // 4] < 1.0).float().mean()) > 0.5
    V = s0["num_visible"]
    kept = []
    for near, big_far, small_far in _near_candidates(r1, ws, V):
        kept.append((s1["num_pairs"] - near - big_far) / small_far)
    print("16384x%d: V=%d one pass %d pairs, split %d; small far pairs kept %.3f-%.3f" % (
        H, V, s0["num_pairs"], s1["num_pairs"], min(kept), max(kept)))
    assert s1["num_pairs"] < s0["num_pairs"]
    assert 0.2 < min(kept) and max(kept) < 0.8, kept                       # dropping nothing / everything fails


@pytest.mark.parametrize("H", [4096, 4112])
def test_far_cull_full_saturation(ws, ctx, H):
    """Every tile saturates in the near slab: the far cull drops every far splat it tests, so the frame emits exactly
    the near list's pairs plus those of the far splats whose rectangles exceed 16 tiles (drop_saturated tests only
    rectangles up to 16 tiles).  The sharded path at world 1 with the split forced on (position cut, bin_count_kernel's
    cull) gives the same frame."""
    import torch
    W = 16384
    cloud, fov = _dense_front(ws, W, H, 3000 + H, right_half_only=False)
    pos, rot = ws.synth.fixed_camera()
    args = make_args(ws, cloud, pos, rot, W, H, *fov)
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r0, t0, s0 = _timed("16384x%d one pass" % H, _render, ws, ctx, cloud, pc, args, W, H, split=False)
    r1, t1, s1 = _timed("16384x%d split" % H, _render, ws, ctx, cloud, pc, args, W, H, split=True)
    assert torch.equal(t0.view(torch.uint8), t1.view(torch.uint8)), "split frame differs from the one-pass frame"
    assert bool((t0[..., 3] == 1.0).all()), "the scene does not saturate every pixel"
    V = s0["num_visible"]
    want = sorted({near + big_far for near, big_far, _ in _near_candidates(r1, ws, V)})
    print("16384x%d: V=%d one pass %d pairs, split %d; near + large far candidates %s" % (H, V, s0["num_pairs"], s1["num_pairs"], want[:4]))
    assert s1["num_pairs"] in want
    del r1, t1
    sh = ws.ShardedRenderer(ws, ctx, ws.FORMAT_RGBA32_FLOAT, 3, False, pc, cloud["num_points"], (W, H),
                            pair_capacity=s0["num_pairs"])
    sh.r.set_occlusion_split(True)                      # (ws_renderer_shard_frame_to_root decides the split per frame)
    host = torch.zeros((H, W, 4), dtype=torch.float32).pin_memory()
    _timed("16384x%d sharded, world 1, split" % H, lambda: (sh.frame_peer(args, clear=(0.1, 0.2, 0.3, 0.4), host=host), torch.cuda.synchronize()))
    assert torch.equal(host.view(torch.uint8), t0.cpu().view(torch.uint8)), "sharded split frame differs from the one-pass frame"
    assert sh.stats()["num_pairs"] < s0["num_pairs"]


# ---- 3. viewport validation --------------------------------------------------------------------------------------------
def test_largest_viewport_and_rejection(ws, orc, ctx):
    """16384 x 16384 (2^20 tiles, three tile-sort passes) prepares and renders: stage 1, the depth order and the pair list
    against the oracle.  16385 in either dimension is refused before anything is enqueued: the prepared frame stays
    and renders again, and the renderer then renders a normal frame."""
    import torch
    W = H = 16384
    cloud, fov = _scene(ws, 50_000, 4000, W, H)
    pos, rot = ws.synth.fixed_camera()
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA8_UNORM, 3, False)
    r.set_occlusion_split(False)
    r.prepare(None, pc, make_args(ws, cloud, pos, rot, W, H, *fov))
    t = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    _timed("16384x16384 render", lambda: (r.render(t, pc), torch.cuda.synchronize()))
    st = r.stats()
    assert (st["width"], st["height"], st["num_tiles"]) == (W, H, 1 << 20)
    zn, zf = orc.fit_near_far(pos, cloud["aabb_min"], cloud["aabb_max"])
    osplats, okeys, _ = orc.preprocess(cloud, orc.camera_uniform(pos, rot, fov[0], fov[1], zn, zf, W, H), orc.render_settings(cloud))
    assert np.array_equal(r.read_buffer(ws.BUF_SPLATS_2D), osplats) and np.array_equal(r.read_buffer(ws.BUF_DEPTH_KEYS), okeys)
    _, order = orc.sort_pairs(okeys, np.arange(len(okeys), dtype=np.uint32))
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_INDICES), order)
    tiles, slots, _, P = oracle_pairs(orc, osplats, order, W, H)
    assert st["num_pairs"] == P
    assert np.array_equal(r.read_buffer(ws.BUF_PAIR_TILES), tiles) and np.array_equal(r.read_buffer(ws.BUF_PAIR_SLOTS), slots)
    rng_ = r.read_buffer(ws.BUF_TILE_RANGES)
    assert np.array_equal(rng_[:, 1] - rng_[:, 0], np.bincount(tiles, minlength=1 << 20))
    assert int(tiles.max()) > (1 << 20) - 1024                              # the last tile row has pairs
    for bw, bh in ((16385, 16), (16, 16385), (16385, 16385)):
        with pytest.raises(ws.WsError) as e:
            r.prepare(None, pc, make_args(ws, cloud, pos, rot, bw, bh, *_fov(bw, bh)[0]))
        assert e.value.status == ws.WS_ERR_UNSUPPORTED
    st2 = r.stats()
    assert (st2["width"], st2["height"], st2["num_pairs"]) == (W, H, P)
    t2 = torch.empty_like(t)
    r.render(t2, pc)
    torch.cuda.synchronize()
    assert torch.equal(t, t2)
    del t, t2
    small = ws.synth.make_cloud(20000, 4001)
    pcs = ws.PointCloud.new(ctx, make_generic(ws, small))
    spos, srot = ws.synth.orbit_camera(70.0)
    args = make_args(ws, small, spos, srot, 320, 200, *ws.synth.fov_for_viewport(320, 200))
    r.prepare(None, pcs, args)
    a = torch.empty((200, 320, 4), dtype=torch.uint8, device="cuda")
    r.render(a, pcs)
    torch.cuda.synchronize()
    _, _, b, _ = frame(ws, ctx, small, spos, srot, 320, 200, fmt=ws.FORMAT_RGBA8_UNORM, host=False)
    assert torch.equal(a, b)


# ---- 4. row pitch ------------------------------------------------------------------------------------------------------
_SENTINEL = {0: 0xA5, 1: -7.0, 2: -7.0}


@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_padded_row_pitch(ws, ctx, fmt):
    """A target that is a view of a wider tensor (row pitch = its row stride): the frame equals the tight frame and the
    padding keeps its sentinel.  Bad pitches and a misaligned pointer are refused without touching the target.
    render_to_host with a padded host pitch (the 2-D copy) gives the same frame."""
    import torch
    W, H, pad = 333, 201, 13
    cloud, fov = _scene(ws, 2000, 5000 + fmt, W, H)
    pos, rot = ws.synth.fixed_camera()
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, fmt, 3, False)
    r.prepare(None, pc, make_args(ws, cloud, pos, rot, W, H, *fov))
    dt = {0: torch.uint8, 1: torch.float16, 2: torch.float32}[fmt]
    bpp = ws._BPP[fmt]
    clear = (0.1, 0.2, 0.3, 0.4)
    tight = torch.empty((H, W, 4), dtype=dt, device="cuda")
    r.render(tight, pc, clear)
    wide = torch.full((H, W + pad, 4), _SENTINEL[fmt], dtype=dt, device="cuda")
    pitch = wide.stride(0) * wide.element_size()
    r.render(wide.data_ptr(), pc, clear, row_pitch=pitch)
    torch.cuda.synchronize()
    assert torch.equal(wide[:, :W].view(torch.uint8), tight.view(torch.uint8))
    assert bool((wide[:, W:] == _SENTINEL[fmt]).all())
    assert bool((tight != tight[0, 0]).any())                              # a frame with content
    # refused: pitch below W * bpp, not a multiple of the pixel size, past 32 bits; dst not aligned to the pixel size
    before = wide.clone()
    for ptr, p in ((wide.data_ptr(), W * bpp - bpp), (wide.data_ptr(), pitch + bpp // 2), (wide.data_ptr(), pitch + 1),
                   (wide.data_ptr(), (1 << 32) * bpp), (wide.data_ptr() + 1, pitch), (wide.data_ptr() + bpp // 2, pitch)):
        with pytest.raises(ws.WsError) as e:
            r.render(ptr, pc, clear, row_pitch=p)
        assert e.value.status == ws.WS_ERR_INVALID_ARGUMENT, (ptr - wide.data_ptr(), p)
    torch.cuda.synchronize()
    assert torch.equal(wide.view(torch.uint8), before.view(torch.uint8))
    # render_to_host into padded host rows: cudaMemcpy2DAsync
    npdt = {0: np.uint8, 1: np.float16, 2: np.float32}[fmt]
    host = np.full((H, W + 5, 4), _SENTINEL[fmt], dtype=npdt)
    clr = (C.c_double * 4)(*clear)
    L = ws.lib()
    st = L.ws_renderer_render_to_host(r._h, pc._h, C.c_void_p(host.ctypes.data), (W + 5) * bpp, C.byref(clr), None)
    assert st == ws.WS_OK, ws.lib().ws_last_error()
    torch.cuda.synchronize()
    assert np.array_equal(host[:, :W].view(np.uint8), tight.cpu().numpy().view(np.uint8))
    assert (host[:, W:] == npdt(_SENTINEL[fmt])).all()
    assert L.ws_renderer_render_to_host(r._h, pc._h, C.c_void_p(host.ctypes.data), W * bpp - 1, C.byref(clr), None) == ws.WS_ERR_INVALID_ARGUMENT


def test_frame_past_4_gib(ws, ctx):
    """16384 x 16384 RGBA32F with a pitch of W * 16 + 256: the last row starts past byte 2^32.  Compared on the device."""
    import torch
    W = H = 16384
    cloud, fov = _scene(ws, 50_000, 6000, W, H)
    pos, rot = ws.synth.fixed_camera()
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA32_FLOAT, 3, False)
    r.set_occlusion_split(False)
    r.prepare(None, pc, make_args(ws, cloud, pos, rot, W, H, *fov))
    tight = torch.empty((H, W, 4), dtype=torch.float32, device="cuda")
    r.render(tight, pc)
    pitch = W * 16 + 256
    assert (H - 1) * pitch > (1 << 32)
    buf = torch.full((H * pitch,), 0xA5, dtype=torch.uint8, device="cuda")
    _timed("16384x16384 RGBA32F into a padded 4.3 GB target", lambda: (r.render(buf.data_ptr(), pc, row_pitch=pitch), torch.cuda.synchronize()))
    rows = buf.view(H, pitch)
    tb = tight.view(torch.uint8).view(H, W * 16)
    for y0 in range(0, H, 1024):
        assert torch.equal(rows[y0:y0 + 1024, : W * 16], tb[y0:y0 + 1024]), "rows %d.. differ" % y0
        assert bool((rows[y0:y0 + 1024, W * 16:] == 0xA5).all()), "padding of rows %d.. written" % y0
    assert float(tight[-1, :, 3].max()) > 0 and float(tight[:, -1, 3].max()) > 0   # the last row / column have content


# ---- 5. pair counts past 2^31 and 2^32 ---------------------------------------------------------------------------------
def _covering_cloud(ws, n, seed):
    """n splats around the origin (depth ~3), each covering all 2^20 tiles of a 16384 x 16384 view."""
    cloud = ws.synth.make_cloud(n, seed)
    g = cloud["gaussians"]
    g["xyz"] *= np.float32(0.05)
    g["cov"] = np.array([16, 0, 0, 16, 0, 16], np.float16)
    _rebox(cloud)
    return cloud


@pytest.mark.parametrize("n,split,lo,hi", [(3000, False, 1 << 31, 1 << 32),    # signed 32-bit arithmetic
                                           (5000, False, 1 << 32, 1 << 33),    # past 2^32
                                           (7000, True, 1 << 32, 1 << 33)])    # the far slab alone past 2^32
def test_pair_count_past_32_bits(ws, orc, ctx, n, split, lo, hi):
    """An overflowing frame reports the exact number of pairs it needed (64-bit), sets pair_overflow and nothing else
    (no error flag: the look-back watchdog did not fire); a frame nobody inspected reports the overflow at the next
    prepare() exactly once; after set_pair_capacity(0) the renderer gives a fresh renderer's frame."""
    import torch
    W = H = 16384
    cloud = _covering_cloud(ws, n, 7000 + n)
    pos, rot = ws.synth.fixed_camera()
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    args = make_args(ws, cloud, pos, rot, W, H, *_fov(W, H)[0])
    r = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA8_UNORM, 3, False)
    r.set_occlusion_split(split)
    r.set_pair_capacity(1 << 24)
    st = _timed("N=%d split=%s prepare + stats" % (n, split), lambda: (r.prepare(None, pc, args), r.stats(allow_overflow=True))[1])
    rects, P = orc.tile_rects(r.read_buffer(ws.BUF_SPLATS_2D), W, H)
    area = (rects[:, 2] - rects[:, 0] + 1).astype(np.int64) * (rects[:, 3] - rects[:, 1] + 1)
    print("N=%d split=%s: V=%d P=%d (%.2f x 2^32), reported %d" % (n, split, st["num_visible"], P, P / 2.0 ** 32, st["num_pairs"]))
    assert st["num_visible"] == n and (area > 16).all() and lo < P < hi     # no far splat is tested by the cull: P is the split's count too
    if split:
        assert 0.7 * P > (1 << 32)                                          # the far slab (about 3/4) alone passes 2^32
    assert st["pair_overflow"] and st["num_pairs"] == P and st["pair_capacity"] == 1 << 24
    # a frame rendered without stats(): the next prepare() reports it, once
    t = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
    _timed("N=%d split=%s prepare + render" % (n, split), lambda: (r.prepare(None, pc, args), r.render(t, pc), torch.cuda.synchronize()))
    with pytest.raises(ws.WsError) as e:
        r.prepare(None, pc, args)
    assert e.value.status == ws.WS_ERR_PAIR_OVERFLOW
    r.prepare(None, pc, args)
    st = r.stats(allow_overflow=True)
    assert st["pair_overflow"] and st["num_pairs"] == P
    del t
    # automatic capacity again, a small viewport
    r.set_pair_capacity(0)
    small = ws.synth.make_cloud(20000, 7001)
    pcs = ws.PointCloud.new(ctx, make_generic(ws, small))
    spos, srot = ws.synth.orbit_camera(200.0)
    sargs = make_args(ws, small, spos, srot, 320, 200, *ws.synth.fov_for_viewport(320, 200))
    r.prepare(None, pcs, sargs)
    a = torch.empty((200, 320, 4), dtype=torch.uint8, device="cuda")
    r.render(a, pcs)
    fresh = ws.GaussianRenderer.new(ctx, ws.FORMAT_RGBA8_UNORM, 3, False)
    fresh.set_occlusion_split(split)
    fresh.prepare(None, pcs, sargs)
    b = torch.empty_like(a)
    fresh.render(b, pcs)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    s_r, s_f = r.stats(), fresh.stats()
    assert not s_r["pair_overflow"] and s_r["num_pairs"] == s_f["num_pairs"] and s_r["pair_capacity"] == s_f["pair_capacity"]
