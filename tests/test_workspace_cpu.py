"""CPU: the offset arithmetic of a forward's workspace (controlar_b200/csrc/carve.h, plain host code) against a host check
(tests/native/carve_check.cpp): the measuring pass's total is the assigning pass's end offset, every buffer is 256-byte aligned,
the buffers are disjoint and in order, a zero-count take is null and takes no space, and a sized buffer accepts a write of exactly
its capacity and refuses one element more."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("carve") / "carve_check")
    subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "native", "carve_check.cpp")], check=True)
    return exe


def _dino(B, H, W, C=384, kpad=608, ad=1):
    hw = (H // 16) * (W // 16)
    rows, Tp = B * (hw + 1), (hw + 1 + 31) & ~31
    return [(2, n) for n in (B * hw * kpad, B * hw * C, hw * C, rows * C, rows * C, rows * 2 * C, B * C * Tp, rows * C, rows * 4 * C,
                             B * hw * C, B * hw * ad)]


def _vq_decode(B, h, w, ch=128, cmax=512, chunks=16):
    act, hw = B * 16 * h * 16 * w * ch, h * w
    hwp = (hw + 31) & ~31
    return [(2, act)] * 5 + [(4, B * 32 * 2 * (1 + chunks)), (4, B * hw * hwp), (2, B * hw * hwp), (2, B * cmax * hwp), (2, B * h * w * 32)]


@pytest.mark.parametrize("takes", [
    _dino(8, 512, 512),                                  # the control encoder of a 512 x 512 batch of 8
    _dino(1, 16, 16),                                    # its smallest input: every buffer shorter than one 256-byte slot or barely longer
    _vq_decode(2, 32, 32),                               # the tokenizer's decoder: bf16 and fp32 buffers mixed
    [(1, 1), (2, 1), (4, 1), (1, 255), (1, 256), (1, 257), (2, 128), (2, 129), (4, 64), (4, 65)],   # around the rounding boundary
    [(4, 0), (2, 100), (1, 0), (4, 7), (2, 0)],          # zero-count takes first, between and last
    [(4, 0)],
    [],
], ids=["dino-512", "dino-16", "vq-decode", "rounding", "zero-count", "only-zero", "empty"])
def test_carve_offsets(checker, takes):
    r = subprocess.run([checker] + ["%d:%d" % t for t in takes], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout == "ok %d\n" % len(takes), r.stdout + r.stderr
