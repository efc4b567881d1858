"""The bench.py contract that can be checked without a GPU: the reference arm (CPU oracle) prints ONE JSON line with the
keys the driver reads, and the GPU arm refuses to run without a CUDA device (no CPU fallback)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(*argv, env=None):
    return subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + list(argv), capture_output=True, text=True,
                          timeout=600, env=dict(os.environ, **(env or {})))


def test_reference_arm_prints_one_json_line():
    p = _run("--impl", "reference", "--workload", "cfg1", "--steps", "2", "--warmup", "1")
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [ln for ln in p.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["metric"] == "frames/sec" and d["unit"] == "frames/s" and d["higher_is_better"] is True
    assert d["steps"] == 2 and d["warmup"] == 1 and d["config"]["steps_requested"] == 2 and d["value"] > 0 and abs(d["ms_per_step"] * d["value"] - 1000.0) < 1.0
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "frames/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["config"]["workload"].startswith("cfg1: 100000 synthetic Gaussians")
    assert d["gpu_launches"] == 0


def test_reference_arm_under_torchrun_only_rank0_works():
    p = _run("--impl", "reference", "--workload", "cfg1", "--steps", "1", "--warmup", "0", env={"RANK": "3", "WORLD_SIZE": "4"})
    assert p.returncode == 0 and p.stdout.strip() == ""


def test_gpu_arm_fails_loudly_without_a_gpu():
    try:
        import torch
        if torch.cuda.is_available():
            import pytest
            pytest.skip("a GPU is present")
    except ImportError:
        pass
    p = _run("--workload", "cfg1", "--steps", "1")
    assert p.returncode != 0 and "no CUDA device" in (p.stderr + p.stdout)


def test_reference_arm_sets_its_own_thread_count():
    """torchrun exports OMP_NUM_THREADS=1 to every rank; the reference arm (and the GPU arm's cpu_baseline) must not inherit
    it -- round 1's N >= 2 reference lines ran on one core (VERDICT r01, weak 10)."""
    p = _run("--impl", "reference", "--workload", "cfg1", "--steps", "1", "--warmup", "0", env={"OMP_NUM_THREADS": "1", "RANK": "0", "WORLD_SIZE": "2"})
    assert p.returncode == 0, p.stderr[-2000:]
    d = json.loads(p.stdout.strip().splitlines()[-1])
    try:
        want = len(os.sched_getaffinity(0))
    except AttributeError:
        want = os.cpu_count()
    assert d["cpu_baseline"]["cores"] == want


def test_frame_crc_is_a_full_frame_hash():
    """the parity evidence carried by the bench lines: every byte of the downloaded frame enters the checksum"""
    import numpy as np
    sys.path.insert(0, ROOT)
    import bench
    a = np.zeros((64, 48, 4), np.float16)
    c0 = bench.frame_crc(a)
    for y, x, ch in ((0, 0, 0), (63, 47, 3), (31, 7, 2)):
        b = a.copy(); b[y, x, ch] = np.float16(6.1e-5)
        assert bench.frame_crc(b) != c0
    assert bench.frame_crc(a.copy()) == c0 and len(c0) == 8


def test_reference_arm_times_exactly_the_requested_steps():
    """--steps is the number of timed frames and --warmup the number of untimed ones, on the reference arm too"""
    p = _run("--impl", "reference", "--workload", "cfg1", "--steps", "7", "--warmup", "5")
    assert p.returncode == 0, p.stderr[-2000:]
    d = json.loads(p.stdout.strip().splitlines()[-1])
    assert d["steps"] == 7 and d["warmup"] == 5 and d["config"]["steps_requested"] == 7
    assert abs(d["ms_per_step"] * d["value"] - 1000.0) < 1.0 and "7 full frames" in d["cpu_baseline"]["sample"]


def test_steps_below_one_are_rejected():
    for argv in (("--steps", "0"), ("--impl", "reference", "--steps", "0"), ("--steps", "2", "--warmup", "-1")):
        p = _run(*argv)
        assert p.returncode == 2 and "--steps must be at least 1" in p.stderr, (argv, p.stderr[-500:])


def test_dump_outputs_writes_the_frame_or_a_fixed_sample_under_64_mb(tmp_path):
    """--dump-outputs: the cfg3 frame (33 MB as float32) is written whole; the cfg4 frame (133 MB) as a seeded pixel sample
    with its row-major indices; float dtypes only, at most 64 MB, and the same bytes every time"""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    g = torch.Generator().manual_seed(3)
    for (H, W), names in (((1080, 1920), ["frame.npy"]), ((2160, 3840), ["frame_sample.npy", "frame_sample_index.npy"])):
        frame = torch.rand((H, W, 4), generator=g).to(torch.float16)
        outs = []
        for run in range(2):
            d = tmp_path / ("%dx%d_%d" % (W, H, run))
            bench.dump_outputs(str(d), frame)
            assert sorted(os.listdir(d)) == sorted(names)
            assert sum(os.path.getsize(d / n) for n in names) <= 64 << 20
            outs.append({n: (d / n).read_bytes() for n in names})
        assert outs[0] == outs[1]
        full = frame.float().numpy()
        if names == ["frame.npy"]:
            a = np.load(tmp_path / ("%dx%d_0" % (W, H)) / "frame.npy")
            assert a.dtype == np.float32 and np.array_equal(a, full)
        else:
            d = tmp_path / ("%dx%d_0" % (W, H))
            px, idx = np.load(d / "frame_sample.npy"), np.load(d / "frame_sample_index.npy")
            assert px.dtype == np.float32 and idx.dtype == np.float64 and px.shape == (len(idx), 4)
            assert len(idx) == bench.DUMP_SAMPLE_PIXELS and (np.diff(idx) > 0).all()
            assert np.array_equal(px, full.reshape(-1, 4)[idx.astype(np.int64)])
