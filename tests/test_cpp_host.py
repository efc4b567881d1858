"""The C++ host side above the C ABI (include/websplat_b200.hpp, tools/ws_render.cpp): what can be checked without a GPU --
cameras.json parsing + SceneCamera -> PerspectiveCamera against the Python mirror, the f16 -> u8 conversion + PNG writer,
and the error behaviour without a CUDA device (no CPU fallback)."""
import json
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def tool(ws):
    ws.build_library()                                     # builds libwebsplat_b200.so and web-splat_b200/ws_render
    path = os.path.join(ROOT, "web-splat_b200", "ws_render")
    assert os.path.exists(path)
    return path


def _scene_entries(ws, count=19, W=1920, H=1080):
    fovx, fovy = ws.synth.fov_for_viewport(W, H)
    out = []
    for i in range(count):
        pos, rot = ws.synth.orbit_camera(360.0 * i / count + 3.0, radius=2.5 + 0.2 * i, elev_deg=10.0 + i)
        cam = ws.PerspectiveCamera(pos, rot, ws.PerspectiveProjection(fovx, fovy, 0.01, 100.0))
        out.append(ws.SceneCamera.from_perspective(ws, cam, "view_%02d" % i, 100 - i, (W, H)).to_json())   # ids descend: order != id
    if count > 4:
        out[4]["rotation"] = (np.asarray(out[4]["rotation"]) * np.array([1.0, -1.0, 1.0])).tolist()      # a left-handed entry
    return out


def test_cpp_scene_parser_matches_python_mirror(ws, tool, tmp_path):
    entries = _scene_entries(ws)
    path = tmp_path / "cameras.json"
    path.write_text(json.dumps(entries, indent=1))
    p = subprocess.run([tool, "--parse-scene", str(path)], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    lines = p.stdout.strip().splitlines()
    sc = ws.Scene.from_json(str(path))
    head = lines[0].split()
    assert int(head[1]) == sc.num_cameras() == len(entries) and abs(float(head[3]) - sc.extend()) < 1e-5 * sc.extend()
    cams = sc.cameras()
    assert len(lines) - 1 == len(cams)
    for line, c in zip(lines[1:], cams):                     # both sorted by id
        f = line.split()
        assert int(f[0]) == c.id and f[1] == c.img_name and f[2] == c.split
        assert (int(f[3]), int(f[4])) == ws.scene.render_resolution(c.width, c.height)
        cam = c.to_perspective(ws)
        vals = np.array([float(x) for x in f[5:]])
        assert np.allclose(vals[0:3], cam.position, rtol=0, atol=1e-6)
        q = vals[3:7] if np.dot(vals[3:7], cam.rotation) > 0 else -vals[3:7]
        assert np.allclose(q, cam.rotation, atol=2e-6)
        assert np.allclose(vals[7:10], [cam.projection.fovx, cam.projection.fovy, cam.projection.fov2view_ratio], rtol=1e-6)
    # malformed input is an error, not a crash
    bad = tmp_path / "bad.json"; bad.write_text('[{"id": 1, "img_name": "x"')
    assert subprocess.run([tool, "--parse-scene", str(bad)], capture_output=True, text=True).returncode == 1


def test_cpp_pixel_conversion_and_png_writer(ws, tool, tmp_path):
    W, H = 61, 37
    out = tmp_path / "ramp.png"
    p = subprocess.run([tool, "--png-selftest", str(out), str(W), str(H)], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    i = np.arange(W * H * 4, dtype=np.uint64)
    halves = (((i * 2654435761) & 0xFFFFFFFF) >> 16).astype(np.uint16).view(np.float16).reshape(H, W, 4)
    assert np.isnan(halves).any() and np.isinf(halves).any() and (halves < 0).any() and ((halves > 0) & (halves < 1)).any()
    with np.errstate(invalid="ignore"):
        want = ws.scene.frame_to_rgba8(halves)               # bin/render.rs:234-240 as restated in the Python mirror
    got = ws.scene.decode_png(out.read_bytes())              # checks the chunk CRCs; zlib checks the adler32 of the stored blocks
    assert np.array_equal(got, want)


def test_cpp_tool_errors(ws, tool, tmp_path):
    assert subprocess.run([tool], capture_output=True).returncode == 64
    ply = tmp_path / "c.ply"; ply.write_bytes(ws.synth.ply_bytes(ws.synth.ply_vertices(50, 1, 1), 1))
    cams = tmp_path / "cameras.json"; cams.write_text(json.dumps(_scene_entries(ws, 3, 320, 200)))
    notply = tmp_path / "c.bin"; notply.write_bytes(b"not a splat file")
    p = subprocess.run([tool, str(notply), str(cams), str(tmp_path / "o")], capture_output=True, text=True)
    assert p.returncode == 1 and "Unknown file format" in p.stderr
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except ImportError:
        has_gpu = False
    if not has_gpu:                                          # no CPU fallback: the ABI's status comes back as ws::Error
        p = subprocess.run([tool, str(ply), str(cams), str(tmp_path / "o")], capture_output=True, text=True)
        assert p.returncode == 2 and "status -2" in p.stderr, p.stderr


@pytest.mark.gpu
def test_gpu_cpp_tool_renders_like_the_python_tool(ws, ctx, tool, tmp_path):
    """the C++ host mirror + offline tool on a GPU: PNG for PNG what scripts/render_scene.py writes"""
    n, W, H = 20000, 320, 200
    ply = tmp_path / "cloud.ply"; ply.write_bytes(ws.synth.ply_bytes(ws.synth.ply_vertices(n, 8, 3), 3))
    cams = tmp_path / "cameras.json"; cams.write_text(json.dumps(_scene_entries(ws, 9, W, H)))
    a, b = tmp_path / "cpp", tmp_path / "py"
    p = subprocess.run([tool, str(ply), str(cams), str(a)], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    import sys
    q = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "render_scene.py"), str(ply), str(cams), str(b)], capture_output=True, text=True, timeout=300)
    assert q.returncode == 0, q.stdout + q.stderr
    for split in ("test", "train"):
        names = sorted(os.listdir(a / split))
        assert names == sorted(os.listdir(b / split)) and names
        for nm in names:
            assert np.array_equal(ws.scene.decode_png((a / split / nm).read_bytes()), ws.scene.decode_png((b / split / nm).read_bytes()))


def _fnv1a(b):
    h = 1469598103934665603
    for x in bytes(b):
        h = ((h ^ x) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


@pytest.mark.parametrize("compressed_zip", [False, True])
def test_cpp_npz_reader_matches_numpy(ws, tool, tmp_path, compressed_zip):
    """tools/npz_reader.hpp (zip central directory, zip64 extras as numpy writes them, stored / deflated members, .npy headers)."""
    a = ws.synth.c3dgs_arrays(700, 4, 2, codebook=64)
    a["extra_f8"] = np.float64(2.5); a["extra_i8"] = np.arange(6, dtype=np.int64).reshape(2, 3)
    path = tmp_path / "c.npz"
    (np.savez_compressed if compressed_zip else np.savez)(path, **a)
    p = subprocess.run([tool, "--parse-npz", str(path)], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0, p.stderr
    got = {}
    for line in p.stdout.strip().splitlines():
        left, right = line.split(" | ")
        f = left.split()
        got[f[0]] = (f[1], tuple(int(x) for x in f[2:]), int(right.split()[0]), int(right.split()[1], 16))
    assert set(got) == set(a)
    for k, v in a.items():
        v = np.asarray(v)
        descr, shape, nbytes, h = got[k]
        assert descr == v.dtype.str and shape == v.shape and nbytes == v.nbytes and h == _fnv1a(np.ascontiguousarray(v).tobytes()), k
    # the descriptor the loader hands to ws_pointcloud_create_from_c3dgs (io/npz.rs:29-160)
    q = subprocess.run([tool, "--check-npz", str(path)], capture_output=True, text=True, timeout=60)
    assert q.returncode == 0, q.stderr
    lines = q.stdout.strip().splitlines()
    assert lines[0] == "points 700 covars 64 features 64 sh_deg 2 scaling_factor 1 gaussian_indices 1 feature_indices 1"
    f = lines[1].split()
    assert abs(float(f[1]) - float(a["scaling_scale"])) < 1e-9 and int(f[2]) == a["scaling_zero_point"]
    assert abs(float(f[4]) - float(a["rotation_scale"])) < 1e-9 and int(f[5]) == a["rotation_zero_point"]
    for line, key in zip(lines[2:6], ("features_dc", "features_rest", "opacity", "scaling_factor")):
        zp, sc = line.split()[1:]
        assert int(zp) == a[key + "_zero_point"] and abs(float(sc) - float(a[key + "_scale"])) < 1e-9
    assert lines[6].startswith("meta mip 1 1 kernel 1 0.1") and lines[6].endswith("bg 1 0 0 0")
    assert lines[7] == "gi0 %d gilast %d" % (a["gaussian_indices"][0], a["gaussian_indices"][-1])
    # the older file variant: no scaling factor, no index arrays, no metadata
    b = ws.synth.c3dgs_arrays(50, 5, 0, scaling_factor=False, indices=False, metadata=False)
    path2 = tmp_path / "d.npz"; np.savez(path2, **b)
    q = subprocess.run([tool, "--check-npz", str(path2)], capture_output=True, text=True, timeout=60)
    assert q.returncode == 0 and q.stdout.splitlines()[0] == "points 50 covars 50 features 50 sh_deg 0 scaling_factor 0 gaussian_indices 0 feature_indices 0"
    assert "quant 0 1" in q.stdout.splitlines()[5] and q.stdout.splitlines()[6].startswith("meta mip 0 0 kernel 0 0 bg 0")
    # a missing required member is an error (io/npz.rs:265-275), so is a truncated archive
    del b["rotation"]
    path3 = tmp_path / "e.npz"; np.savez(path3, **b)
    r = subprocess.run([tool, "--check-npz", str(path3)], capture_output=True, text=True)
    assert r.returncode == 1 and "rotation" in r.stderr
    path4 = tmp_path / "f.npz"; path4.write_bytes(path.read_bytes()[:-30])
    assert subprocess.run([tool, "--parse-npz", str(path4)], capture_output=True, text=True).returncode == 1


def test_cpp_readers_survive_damaged_input(ws, tool, tmp_path):
    """the zip / npy / JSON readers of the C++ tool on damaged files: an error exit is fine, a crash (signal) is not."""
    rng = np.random.default_rng(11)
    a = ws.synth.c3dgs_arrays(40, 4, 1, codebook=8)
    src = tmp_path / "g.npz"; np.savez_compressed(src, **a)
    good = src.read_bytes()
    cams = json.dumps(_scene_entries(ws, 3, 320, 200)).encode()
    victim = tmp_path / "v.bin"
    for i in range(240):
        base, flag = (good, "--check-npz") if i % 2 == 0 else (cams, "--parse-scene")
        b = bytearray(base)
        k = rng.integers(0, 3)
        if k == 0:
            for _ in range(rng.integers(1, 8)):
                b[rng.integers(0, len(b))] = rng.integers(0, 256)
        elif k == 1:
            b = b[:rng.integers(0, len(b))]
        else:
            j = rng.integers(0, len(b)); del b[j:j + rng.integers(1, 64)]
        victim.write_bytes(bytes(b))
        p = subprocess.run([tool, flag, str(victim)], capture_output=True, timeout=60)
        assert p.returncode in (0, 1), (flag, p.returncode, p.stderr[-200:])


def test_cpp_npz_reader_rejects_hostile_sizes(ws, tool, tmp_path):
    """The attacker-controlled fields the advisor named (ADVICE r01, tools/npz_reader.hpp): a .npy shape whose byte count
    wraps (2^63, 2), a central-directory name / extra length that runs past the file, a local-header offset and a compressed
    size near 2^64 (zip64), an implausible uncompressed size.  Each must end in the reader's own error (exit 1), never in a
    crash, a hang or a huge allocation."""
    import io
    import struct
    import zipfile

    def npy(shape_text, payload=b"\x00" * 16, descr="<f4"):
        hdr = ("{'descr': '%s', 'fortran_order': False, 'shape': %s, }" % (descr, shape_text)).encode()
        hdr += b" " * ((64 - (10 + len(hdr) + 1) % 64) % 64) + b"\n"
        return b"\x93NUMPY\x01\x00" + struct.pack("<H", len(hdr)) + hdr + payload

    def run(blob):
        f = tmp_path / "h.npz"; f.write_bytes(blob)
        p = subprocess.run([tool, "--parse-npz", str(f)], capture_output=True, text=True, timeout=60)
        assert p.returncode == 1 and "npz:" in p.stderr, (p.returncode, p.stderr[-300:])

    def zip_of(name, data):
        bio = io.BytesIO()
        with zipfile.ZipFile(bio, "w", zipfile.ZIP_STORED) as z:
            z.writestr(name, data)
        return bytearray(bio.getvalue())

    # (1) shapes whose element count times the item size wraps around 2^64, or simply exceeds the member
    for shape in ("(9223372036854775808, 2)", "(4294967296, 4294967296)", "(1000000,)", "(18446744073709551615,)"):
        run(bytes(zip_of("xyz.npy", npy(shape))))
    good = zip_of("xyz.npy", npy("(4,)"))
    cd = good.rfind(b"PK\x01\x02"); eocd = good.rfind(b"PK\x05\x06")
    assert cd > 0 and eocd > cd
    # (2) file-name / extra-field lengths of the central directory entry running past the end of the file
    for off in (28, 30, 32):
        b = bytearray(good); b[cd + off:cd + off + 2] = b"\xff\xff"; run(bytes(b))
    # (3) local header offset and sizes forced through the zip64 extra field to values near 2^64
    b = bytearray(good)
    extra = struct.pack("<HHQQQ", 1, 24, 0xfffffffffffffff0, 0xfffffffffffffff0, 0xfffffffffffffff0)
    entry_end = cd + 46 + struct.unpack("<H", b[cd + 28:cd + 30])[0]
    b[cd + 20:cd + 28] = b"\xff" * 8                          # compressed + uncompressed size = 0xffffffff -> "see zip64 extra"
    b[cd + 42:cd + 46] = b"\xff" * 4                          # local header offset likewise
    b[cd + 30:cd + 32] = struct.pack("<H", len(extra))
    b[entry_end:entry_end] = extra
    run(bytes(b))
    # (4) a zip64 extra field shorter than the values it must hold
    b2 = bytearray(good)
    short = struct.pack("<HHQ", 1, 8, 5)
    b2[cd + 20:cd + 28] = b"\xff" * 8; b2[cd + 42:cd + 46] = b"\xff" * 4
    b2[cd + 30:cd + 32] = struct.pack("<H", len(short)); b2[entry_end:entry_end] = short
    run(bytes(b2))
    # (5) central directory offset / entry count beyond the file
    b3 = bytearray(good); b3[eocd + 16:eocd + 20] = struct.pack("<I", 0x7fffffff); run(bytes(b3))
    b4 = bytearray(good); b4[eocd + 10:eocd + 12] = struct.pack("<H", 60000); run(bytes(b4))
    # (6) a stored member that claims a different uncompressed size
    b5 = bytearray(good); b5[cd + 24:cd + 28] = struct.pack("<I", 0x70000000); run(bytes(b5))
    # and the untouched archive still parses
    f = tmp_path / "ok.npz"; f.write_bytes(bytes(good))
    p = subprocess.run([tool, "--parse-npz", str(f)], capture_output=True, text=True, timeout=60)
    assert p.returncode == 0 and p.stdout.startswith("xyz <f4 4"), p.stderr
