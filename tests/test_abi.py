"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/websplat_b200.h declares, host-only helpers agree with the oracle, and device work fails
LOUDLY without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "websplat_b200.h")).read()
    return sorted(set(re.findall(r"WS_API[^;(]*?\b(ws_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(ws):
    L = ws.lib()
    declared = _declared_symbols()
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(L, name), "libwebsplat_b200.so does not export %s" % name
    assert sorted(ws.EXPORTED_SYMBOLS) == declared


def test_struct_layouts_match_reference_uniforms(ws):
    # SplattingArgs mirror, stats, desc: sizes are part of the ABI
    assert C.sizeof(ws.ws_aabb) == 24
    assert C.sizeof(ws.ws_quantization4) == 64              # pointcloud.rs:389-396, 4 x 16 B
    assert ws.synth.GAUSSIAN_DTYPE.itemsize == 28           # pointcloud.rs:38-45
    assert ws.synth.GAUSSIAN_COMPRESSED_DTYPE.itemsize == 24  # pointcloud.rs:14-24
    assert ws.synth.GAUSSIAN_DTYPE.fields["opacity"][1] == 12 and ws.synth.GAUSSIAN_DTYPE.fields["cov"][1] == 16
    f = ws.synth.GAUSSIAN_COMPRESSED_DTYPE.fields
    assert f["opacity"][1] == 12 and f["scale_factor"][1] == 13 and f["geometry_idx"][1] == 16 and f["sh_idx"][1] == 20


def test_host_helpers_match_oracle(ws, orc):
    rng = np.random.default_rng(5)
    for _ in range(20):
        lo = rng.uniform(-3, 0, 3).astype(np.float32); hi = rng.uniform(0, 3, 3).astype(np.float32)
        pos = rng.uniform(-5, 5, 3).astype(np.float32)
        box = ws.Aabb(lo, hi)
        assert np.float32(box.radius()) == orc.aabb_radius(lo, hi)
        cam = ws.PerspectiveCamera(pos, (1, 0, 0, 0), ws.PerspectiveProjection(1.0, 1.0, 0.1, 100.0))
        cam.fit_near_far(box)
        zn, zf = orc.fit_near_far(pos, lo, hi)
        assert (np.float32(cam.projection.znear), np.float32(cam.projection.zfar)) == (np.float32(zn), np.float32(zf))


def test_status_strings_and_version(ws):
    L = ws.lib()
    assert L.ws_status_string(0) == b"ok"
    assert b"pair" in L.ws_status_string(ws.WS_ERR_PAIR_OVERFLOW)
    assert b"sm_90a" in L.ws_version()


def test_no_cpu_fallback_without_gpu(ws):
    """The product must fail loudly when there is no CUDA device."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(ws.WsError) as e:
        ws.Context(0)
    assert e.value.status == ws.WS_ERR_CUDA


def test_product_does_not_import_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
    pats = (r'#\s*include\s*[<"][^>"]*oracle', r"libws_oracle", r"^\s*from\s+oracle\b", r"^\s*import\s+oracle\b", r"wso_[a-z_]+\s*\(")
    roots = [os.path.join(ROOT, d) for d in ("web-splat_b200", "include", "scripts", "bindings", "tools")]
    files = [os.path.join(ROOT, f) for f in ("bench_multi.py", "websplat_b200.py")]
    for root in roots:
        for dirpath, _, names in os.walk(root):
            files += [os.path.join(dirpath, fn) for fn in names]
    for path in files:
        if path.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp", ".rs", ".sh")):
            txt = open(path, errors="ignore").read()
            for pat in pats:
                assert not re.search(pat, txt, re.M), (path, pat)


def test_header_is_plain_c_and_cxx(tmp_path):
    """the drop-in boundary must be consumable from C (cgo / JNI / Rust bindgen read it as C) and from C++."""
    import subprocess
    inc = os.path.join(ROOT, "include")
    c = tmp_path / "t.c"
    c.write_text('#include "websplat_b200.h"\nint main(void) { ws_splatting_args a; ws_frame_stats s; (void)a; (void)s; return sizeof(ws_pointcloud_desc) > 0 ? 0 : 1; }\n')
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    p = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", inc, str(c)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    cpp = tmp_path / "t.cpp"
    cpp.write_text('#include "websplat_b200.hpp"\nint main() { ws::SplattingArgs a; return a.c().max_sh_deg == 3 ? 0 : 1; }\n')
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    p = subprocess.run([gxx, "-std=c++17", "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-I", inc, str(cpp)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr


def test_ctypes_mirror_has_the_header_s_struct_layouts(ws, tmp_path):
    """sizeof / offsetof of every struct that crosses the boundary: the C header against the ctypes mirror."""
    import ctypes as C
    import subprocess
    structs = {"ws_aabb": ws.ws_aabb, "ws_quantization4": ws.ws_quantization4, "ws_pointcloud_desc": ws.ws_pointcloud_desc,
               "ws_splatting_args": ws.ws_splatting_args, "ws_frame_stats": ws.ws_frame_stats, "ws_c3dgs_arrays": ws.ws_c3dgs_arrays,
               "ws_ply_info": ws.ws_ply_info}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "websplat_b200.h"', 'int main(void) {']
    for name, st in structs.items():
        lines.append('printf("%s %%zu\\n", sizeof(%s));' % (name, name))
        for field, _ in st._fields_:
            lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, field, name, field))
    lines += ['return 0; }']
    src = tmp_path / "layout.c"; src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    gcc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    p = subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True).stdout.splitlines())
    for name, st in structs.items():
        assert int(got[name]) == C.sizeof(st), name
        for field, _ in st._fields_:
            assert int(got["%s.%s" % (name, field)]) == getattr(st, field).offset, (name, field)


def test_rust_ffi_structs_list_the_header_s_fields_in_order(ws):
    """bindings/rust cannot be compiled here; at least its #[repr(C)] structs must name the same fields in the same order."""
    txt = open(os.path.join(ROOT, "bindings", "rust", "src", "ffi.rs")).read()
    for name, st in (("ws_aabb", ws.ws_aabb), ("ws_quantization4", ws.ws_quantization4), ("ws_pointcloud_desc", ws.ws_pointcloud_desc),
                     ("ws_splatting_args", ws.ws_splatting_args), ("ws_frame_stats", ws.ws_frame_stats)):
        m = re.search(r"pub struct %s\s*\{(.*?)\}" % name, txt, re.S)
        assert m, name
        rust_fields = re.findall(r"pub (\w+)\s*:", m.group(1))
        assert rust_fields == [f for f, _ in st._fields_], name
    # every function the crate declares exists in the library
    declared = re.findall(r"pub fn (ws_\w+)\(", txt)
    assert declared and set(declared) <= set(ws.EXPORTED_SYMBOLS)
