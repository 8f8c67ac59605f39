"""CPU: the per-token attention work split of the persistent decode kernel (controlar_b200/csrc/pk_plan.h, plain integer code shared
by host and device) against a brute-force tiling check (tests/native/pk_plan_check.cpp): the parts of all CTAs / warps tile
the flattened (pair, key) space exactly once and every per-segment record describes exactly those parts."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("pkplan") / "pk_plan_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "native", "pk_plan_check.cpp")], check=True)
    return exe


@pytest.mark.parametrize("grid,b_eff,H,n_lo,n_hi", [
    (132, 16, 20, 1, 1144),      # config 2 on an H100 (132 SMs): GPT-XL, B = 8 + CFG, every context length of a 512 x 512 image
    (132, 8, 20, 1, 1656),       # config 4 on an H100: 768 x 512, B = 4 + CFG
    (148, 16, 20, 1, 1144),      # the same shapes at a larger grid
    (148, 8, 20, 1, 1656),
    (148, 16, 12, 1, 400),       # GPT-B heads
    (148, 2, 20, 1, 300),        # fewer pairs than CTAs: a pair spans several CTAs
    (148, 4, 4, 1, 80),          # the small test models
    (132, 16, 20, 100, 300),     # another grid size
    (148, 1, 4, 1, 40),          # tot < grid for short contexts: idle CTAs
])
def test_plan_tiles_the_key_space(checker, grid, b_eff, H, n_lo, n_hi):
    r = subprocess.run([checker, str(grid), str(b_eff), str(H), str(n_lo), str(n_hi)], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.startswith("ok"), r.stdout + r.stderr
