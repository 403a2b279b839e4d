"""CPU: the byte counts bench_expert_gemm.py divides its times by.  They follow the grouped GEMM's A-load rule (csrc
gemm_common.cuh, tile_a_rows): the rows of an m-tile that the group owns, rounded up to 16, against a whole 128-row box."""
import importlib.util
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mod():
    spec = importlib.util.spec_from_file_location("bench_expert_gemm_under_test", os.path.join(ROOT, "bench_expert_gemm.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tile_rows_follow_the_cover_rule():
    b = _mod()
    want = {1: 16, 3: 16, 15: 16, 16: 16, 17: 32, 63: 64, 64: 64, 65: 80, 72: 80, 112: 112, 113: 128, 127: 128, 128: 128}
    for count, rows in want.items():
        assert b.tile_a_rows(count, 0) == rows, count
        assert b.tile_a_rows(count, 0, "box128") == 128
    # second m-tile of a group of 200 rows: 72 rows left -> 64 + 16; the first is a whole box
    assert b.tile_a_rows(200, 0) == 128 and b.tile_a_rows(200, 1) == 80
    assert b.tile_a_rows(129, 1) == 16


def test_kernel_rule_in_the_source_is_the_one_modelled():
    """The constants the model shares with the kernel."""
    src = open(os.path.join(ROOT, "aria_b200", "csrc", "gemm_common.cuh")).read()
    b = _mod()
    assert f"constexpr int BM = {b.BM};" in src and f"constexpr int A_BOX_MIN = {b.A_BOX_MIN};" in src
    assert "min(BM, (rows - m_idx * BM + A_BOX_MIN - 1) & ~(A_BOX_MIN - 1))" in src


def test_l2_bytes_of_one_expert():
    b = _mod()
    # bf16 fc1 + SwiGLU, one expert of 72 rows: 26 n-tiles x 40 k-blocks x (80 rows x 128 B of A + 16 KB of B)
    assert b.l2_smem_bytes([72], "fc1", "bf16") == 26 * 40 * (80 * 128 + 16384)
    assert b.l2_smem_bytes([72], "fc1", "bf16", "box128") == 26 * 40 * (16384 + 16384)
    # 3 rows: a single 16-row box; fc2 has 20 n-tiles and 26 k-blocks
    assert b.l2_smem_bytes([3], "fc2", "bf16") == 20 * 26 * (16 * 128 + 16384)
    # W8A16: the B stage is 128 x 64 e4m3; W8A8: 128-deep k-blocks, A rows stay 128 bytes
    assert b.l2_smem_bytes([3], "fc2", "w8a16") == 20 * 26 * (16 * 128 + 8192)
    assert b.l2_smem_bytes([3], "fc2", "w8a8") == 20 * 13 * (16 * 128 + 16384)
    assert b.l2_smem_bytes([72], "fc1", "w8a8") == 26 * 20 * (80 * 128 + 16384)
    # groups add up; empty groups have no tile; 200 rows = one whole tile + one of 80 rows
    assert b.l2_smem_bytes([0, 72, 0, 3], "fc2", "bf16") == b.l2_smem_bytes([72], "fc2", "bf16") + b.l2_smem_bytes([3], "fc2", "bf16")
    assert b.l2_smem_bytes([200], "fc2", "bf16") == 20 * 26 * ((128 + 80) * 128 + 2 * 16384)


def test_cfg2_traffic_is_twice_the_weights_with_whole_boxes():
    """At 72 rows per expert every tile pulled as much A as B; the cover brings A down to 80 / 128 of that."""
    b = _mod()
    counts = [72] * 64
    w = b.weight_bytes(counts, "fc1", "bf16")
    assert w == 64 * 2560 * 3328 * 2
    assert b.l2_smem_bytes(counts, "fc1", "bf16", "box128") == 2 * w
    assert b.l2_smem_bytes(counts, "fc1", "bf16") * 128 == w * (128 + 80)
    assert b.weight_bytes([0, 5, 0, 1], "fc2", "w8a16") == 2 * 1664 * 2560


def test_row_counts_are_seeded_and_complete():
    b = _mod()
    for rows in (6, 192, 4608):
        c = b.row_counts(rows)
        assert len(c) == b.E and sum(c) == rows and c == b.row_counts(rows)


def test_help_runs_without_a_gpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench_expert_gemm.py"), "--help"], capture_output=True, text=True)
    assert r.returncode == 0 and "--rows" in r.stdout
