"""Shared helpers for the parity tests."""
import numpy as np


def make_generic(ws, cloud):
    return ws.GenericGaussianPointCloud(
        cloud["gaussians"], cloud["sh_coefs"], cloud["sh_deg"], cloud["num_points"],
        ws.Aabb(cloud["aabb_min"], cloud["aabb_max"]), cloud["center"], compressed=cloud["compressed"],
        covars=cloud.get("covars"), quantization=cloud.get("quantization"))


def make_args(ws, cloud, pos, rot, W, H, fovx, fovy, **kw):
    cam = ws.PerspectiveCamera(pos, rot, ws.PerspectiveProjection(fovx, fovy, 0.1, 100.0))
    cam.fit_near_far(ws.Aabb(cloud["aabb_min"], cloud["aabb_max"]))     # as every reference caller does
    return ws.SplattingArgs(cam, (W, H), **kw)


def f16_ordered(bits):
    """map f16 bit patterns to integers that are monotone in the value (for ulp distances)."""
    i = bits.astype(np.int32)
    return np.where(i & 0x8000, 0x8000 - (i & 0x7fff), (i & 0x7fff) + 0x8000)


def oracle_pairs(orc, splats, order, W, H):
    """(tile, slot) pair list sorted by (tile, draw order) from the oracle's stage outputs."""
    rects, P = orc.tile_rects(splats, W, H)
    tx = (W + 15) // 16
    tiles, slots = [], []
    for slot in order:                          # draw order = ascending key, ties by slot
        x0, y0, x1, y1 = rects[slot]
        if x1 < x0:
            continue
        ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        t = (ys * tx + xs).reshape(-1)
        tiles.append(t); slots.append(np.full(t.size, slot, np.uint32))
    if not tiles:
        return np.zeros(0, np.uint32), np.zeros(0, np.uint32), rects, 0
    tiles = np.concatenate(tiles).astype(np.uint32); slots = np.concatenate(slots)
    o = np.argsort(tiles, kind="stable")
    return tiles[o], slots[o], rects, P


def image_close(img, ref, sens, atol=2e-3):
    """|img - ref| <= atol + sens per pixel (sens = oracle's bound on discard-threshold flips)."""
    d = np.abs(img.astype(np.float64) - ref.astype(np.float64)).max(axis=2)
    lim = atol + (sens if sens is not None else 0.0)
    return d, (d <= lim)


def frame(ws, ctx, cloud, pos, rot, W, H, fmt=None, clear=(0, 0, 0, 0), split=False, fov=None, pair_capacity=None, host=True, **kw):
    """One frame through the C ABI.  split=False: one binning + tile sort over all pairs, so that the pair-list
    read-backs and num_pairs are the complete ones the oracle produces (the occlusion split, on by default in the
    product, emits fewer pairs for the same image: test_occlusion_split_is_bit_identical).  fov = (fovx, fovy) in
    radians (default: synth.fov_for_viewport); host=False leaves the frame on the device (a torch tensor)."""
    import torch
    fmt = ws.FORMAT_RGBA32_FLOAT if fmt is None else fmt
    fovx, fovy = ws.synth.fov_for_viewport(W, H) if fov is None else fov
    pc = ws.PointCloud.new(ctx, make_generic(ws, cloud))
    r = ws.GaussianRenderer.new(ctx, fmt, cloud["sh_deg"], cloud["compressed"])
    r.set_occlusion_split(split)
    if pair_capacity:
        r.set_pair_capacity(pair_capacity)
    args = make_args(ws, cloud, pos, rot, W, H, fovx, fovy, **kw)
    r.prepare(None, pc, args)
    dt = {0: torch.uint8, 1: torch.float16, 2: torch.float32}[fmt]
    target = torch.empty((H, W, 4), dtype=dt, device="cuda")
    r.render(target, pc, clear)
    torch.cuda.synchronize()
    return r, pc, (target.cpu().numpy() if host else target), (fovx, fovy)


def check_all_stages(ws, orc, ctx, cloud, pos, rot, W, H, fov=None, **kw):
    """Every stage of a split-off frame against the oracle (DESIGN.md section 5): uniforms, stage 1, depth sort, pair
    list and tile ranges bit-exact; image within 2e-3 + sens per pixel, mean |d| <= 2e-5.  The pair capacity is set to
    the oracle's P, so that the complete list is there to compare however many tiles a splat touches.  The image is
    compared in strips of rows (image_close works in float64).  Returns (renderer, stats, image summary) where the
    summary holds the largest |d|, the mean |d|, the largest share |d| / (atol + sens) of a pixel's tolerance and the
    seconds the oracle took to render the frame."""
    import time
    fovx, fovy = ws.synth.fov_for_viewport(W, H) if fov is None else fov
    t0 = time.perf_counter()
    ref = orc.render_frame(cloud, pos, rot, W, H, fovx, fovy, want_sens=True, **kw)
    oracle_s = time.perf_counter() - t0
    V = len(ref["keys"])
    sk, order = orc.sort_pairs(ref["keys"], np.arange(V, dtype=np.uint32))
    tiles, slots, rects, P = oracle_pairs(orc, ref["splats"], order, W, H)
    r, pc, img, _ = frame(ws, ctx, cloud, pos, rot, W, H, fov=(fovx, fovy), pair_capacity=max(P, 1), host=False, **kw)
    st = r.stats()
    # uniforms as the reference would upload them
    assert np.array_equal(r.camera_uniform().view(np.uint32), np.frombuffer(bytes(ref["cam"]), np.uint32))
    assert r.settings_uniform().tobytes() == bytes(ref["settings"])
    # stage 1
    assert st["num_visible"] == V == r.num_visible_points()
    splats = r.read_buffer(ws.BUF_SPLATS_2D)
    a, b = splats, ref["splats"]
    nan_a = np.isnan(a.view(np.float16)); nan_b = np.isnan(b.view(np.float16))
    assert np.array_equal(nan_a, nan_b)
    assert np.array_equal(a[~nan_a], b[~nan_b]), "stage-1 halves differ from the oracle"
    assert np.array_equal(r.read_buffer(ws.BUF_DEPTH_KEYS), ref["keys"])
    # stage 2 (depth sort)
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_KEYS), sk)
    assert np.array_equal(r.read_buffer(ws.BUF_SORTED_INDICES), order)
    # tile binning
    assert st["num_pairs"] == P
    rc = r.read_buffer(ws.BUF_TILE_RECTS).astype(np.int32)
    mine = np.stack([rc[:, 0], rc[:, 1], rc[:, 0] + rc[:, 2] - 1, rc[:, 1] + rc[:, 3] - 1], 1)
    empty = rc[:, 2] == 0
    assert np.array_equal(empty, rects[:, 2] < rects[:, 0])
    assert np.array_equal(mine[~empty], rects[~empty])
    assert np.array_equal(r.read_buffer(ws.BUF_PAIR_TILES), tiles)
    assert np.array_equal(r.read_buffer(ws.BUF_PAIR_SLOTS), slots)
    rng_ = r.read_buffer(ws.BUF_TILE_RANGES)
    T = ((W + 15) // 16) * ((H + 15) // 16)
    cnt = np.bincount(tiles, minlength=T)
    assert np.array_equal(rng_[:, 1] - rng_[:, 0], cnt)
    # stage 3, in strips of about 2^22 pixels
    rows = max(1, (1 << 22) // W)
    dmax, used, bad, sum_abs = 0.0, 0.0, 0, 0.0
    for y0 in range(0, H, rows):
        part = img[y0:y0 + rows].cpu().numpy()
        refp = ref["image"][y0:y0 + rows]
        d, ok = image_close(part, refp, ref["sens"][y0:y0 + rows])
        dmax = max(dmax, float(d.max()))
        used = max(used, float((d / (2e-3 + ref["sens"][y0:y0 + rows])).max()))
        bad += int((~ok).sum())
        sum_abs += float(np.abs(part.astype(np.float64) - refp).sum())
    mean = sum_abs / (H * W * 4)
    assert bad == 0, "image: %d px outside tolerance, max |d| %.3g" % (bad, dmax)
    assert mean <= 2e-5
    return r, st, dict(max=dmax, mean=mean, used=used, oracle_s=oracle_s)
