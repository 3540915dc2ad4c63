"""The per-series kernel choice of filo_query (scan_path, scan_wp_layout.h), through the host program tests/cpp/scan_path.cpp: the C2 shape
(480 rows in chunks of 400 + 80, T = 481, rate()[5m] step 15s on a gauge) runs on scan_wp_batch_kernel with O on V, 15 series per batch
in two batch buffers, one CTA per SM."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_scan_path(out_dir):
    exe = os.path.join(str(out_dir), "scan_path")
    subprocess.run(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "filodb_b200", "csrc"),
                    os.path.join(ROOT, "tests", "cpp", "scan_path.cpp"), "-o", exe], check=True)
    return exe


def scan_path(exe, **kw):
    """The choice for one table shape, as a dict of ints (and the kernel's name)."""
    r = subprocess.run([exe] + ["%s=%s" % (k, v) for k, v in kw.items()], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    out = dict(line.split("=", 1) for line in r.stdout.split())
    return {k: (v if k == "kernel" else int(v)) for k, v in out.items()}


def test_c2_shape_selects_the_batch_kernel_with_o_on_v(tmp_path):
    exe = build_scan_path(tmp_path)
    # C2's records: 16-byte header, two chunk entries, a const-DDV timestamp vector and an XOR value vector per chunk, ~3.8 KB
    for rec in (3712, 3808, 3904):
        p = scan_path(exe, rec=rec, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, cls="sum", sms=132)
        assert p["kernel"] == "batch" and p["alias"] == 1, p
        assert p["B"] == 15 and p["warps"] == 15 and p["rec_bufs"] == 2 and p["grid"] == 132, p
        assert p["smem"] <= 227 * 1024, p
    # depth: 5 * 15 * 132 series give every consumer warp five series, the last in round u = 4 // 2 = 2; one series fewer leaves the
    # last CTA's batch 4 empty
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132)["series_per_warp"] == 5
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132)["rounds"] == 2
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5 * 15 * 132 - 1)["rounds"] == 1
    # rate on a counter schema runs on the counter kernel; without the v2 kernel no per-series kernel runs in front of it
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, cls="counter")["kernel"] == "ctr"
    assert scan_path(exe, rec=3808, rows=480, chunks=2, T=481, wrows=21, n=5_000_000, v2=0)["kernel"] == "v2"
