"""The object boundary mask (dynosam_b200/frontend_csrc/boundary.cuh) on the host: its ellipse rows and thickness formula against
cv2 and the reference's expression, the host build of its sequential statement against the literal cv2 composition of
tests/boundary_oracle.py, bit for bit, and mutations of the statement that must each fail a case."""
import ctypes as C
import os
import shutil
import subprocess

import cv2
import numpy as np
import pytest

import boundary_cases as BC
import boundary_oracle as BO
import frame_cases as FC

ROOT = BC.ROOT
FE = os.path.join(ROOT, "dynosam_b200", "frontend_csrc")


def build_shim(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [FE]
    if patch is not None:                      # a mutated copy of boundary.cuh, seen only by this build
        src = open(BC.CUH).read()
        assert src.count(patch[0]) == 1, patch[0]
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "boundary.cuh"), "w").write(src.replace(patch[0], patch[1]))
        inc = [d]
    so = str(tmp_path / ("boundary_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "boundary_host.cu"), "-o", so], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    return build_shim(tmp_path_factory.mktemp("boundary"))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def host(lib, M, t, capacity=255):
    M = np.ascontiguousarray(M, np.int32); H, W = M.shape
    objs = np.zeros(max(capacity, 1), np.int32); bb = np.zeros((max(capacity, 1), 4), np.int32); ib = np.zeros_like(bb)
    mask = np.zeros((H, W), np.uint8)
    n = lib.host_boundary(_p(M), W, H, int(t), int(capacity), _p(objs), _p(bb), _p(ib), _p(mask))
    s = min(n, capacity)
    return objs[:s], bb[:s], ib[:s], mask


def differs(a, b):
    """the parts of two (objects, bb, inner_bb, mask) results that differ"""
    return [k for k, x, y in zip(("objects", "bb", "inner_bb", "mask"), a, b) if x.shape != y.shape or not np.array_equal(x, y)]


CASES = BC.cases()


def test_ellipse_rows_match_cv2(shim):
    for r in range(BC.CAP + 1):
        hw = np.zeros(r + 1, np.int32)
        shim.host_boundary_ellipse(r, _p(hw))
        el = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (2*r + 1, 2*r + 1))
        want = np.zeros_like(el)
        for dy in range(-r, r + 1):
            want[dy + r, r - hw[abs(dy)]:r + hw[abs(dy)] + 1] = 1
        assert np.array_equal(el, want), r


def test_thickness_formula(shim):
    sizes = [(c.w, c.h) for c in FC.CASES.values()] + [(640, 480), (1920, 1080), (2560, 1440)]
    for w, h in sizes:
        assert shim.host_boundary_thickness(w, h) == BO.thickness(w, h), (w, h)
    assert BO.thickness(1242, 375) == 15 and BO.thickness(640, 480) == 10 and BO.thickness(1920, 1080) == 68
    assert BO.thickness(2560, 1440) <= BC.CAP


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_statement_matches_oracle(shim, name):
    M, t = CASES[name]
    ref = BO.object_boundary(M, t)
    got = host(shim, M, t)
    assert not differs(ref, got), (name, differs(ref, got))


def test_cases_reach_their_rules():
    """the cases hit what they are named for: an erased object, all labels, an empty mask"""
    o, bb, ib, _ = BO.object_boundary(*CASES["inner_erased"])
    assert (ib[list(o).index(3)] == 0).all() and (ib[list(o).index(9)] != 0).all()
    assert len(BO.object_boundary(*CASES["all_255_labels"])[0]) == 255
    assert len(BO.object_boundary(*CASES["empty"])[0]) == 0


def test_capacity_writes_first_rows(shim):
    M, t = CASES["all_255_labels"]
    full = host(shim, M, t)
    part = host(shim, M, t, capacity=17)
    assert np.array_equal(part[0], full[0][:17]) and np.array_equal(part[1], full[1][:17]) and np.array_equal(part[2], full[2][:17])


MUTATIONS = {
    "rectangle_element": ("  return dx < r ? dx : r;", "  return r;"),
    "column_1x10": ("for (int d = -BOUNDARY_PAD; d <= BOUNDARY_PAD; d++)", "for (int d = -BOUNDARY_PAD; d < BOUNDARY_PAD; d++)"),
    "erosion_border_zero": ("continue;     // outside the image: never the minimum", "{ ero = 0; continue; }"),
    "first_writer": ("if (v > best) best = v;", "if (v > 0 && (best == 0 || v < best)) best = v;"),
    "inner_bb_no_pad": ("boundary_rect(inner_ext + 4*j, W, H, BOUNDARY_PAD, inner_bb + 4*n);",
                        "boundary_rect(inner_ext + 4*j, W, H, 0, inner_bb + 4*n);"),
}


@pytest.mark.parametrize("mutation", sorted(MUTATIONS))
def test_mutation_fails_a_case(tmp_path, mutation):
    lib = build_shim(tmp_path, MUTATIONS[mutation])
    failed = [name for name, (M, t) in BC.cases(dataset=False).items()
              if t <= 15 and differs(BO.object_boundary(M, t), host(lib, M, t))]
    assert failed, mutation
