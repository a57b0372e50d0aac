"""The variable layout (csrc/var_layout.cuh), built for the host, against a numpy statement of the layouts include/dynoba.h
documents: the pose-like elimination order, the SoA value images, the delta of dynoba_solve / dynoba_retract, the reduced
system of dynoba_get_reduced_system, and the prior and navigation tables.  Mutations of a copy of the header each fail
at least one check."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dynosam_b200", "csrc")

POSE6, POINT3, FLOW2, VEL3, BIAS6 = range(5)           # dynoba_var_kind
WIDTH = [12, 3, 2, 3, 6]                                # doubles of a value in the caller's arrays
TDIM = [6, 3, 2, 3, 6]                                  # tangent dimension
ROWS = [12, 3, 2, 12, 12]                               # rows of the SoA image: velocities and biases in the pose image
POSELIKE = (POSE6, VEL3, BIAS6)
DELTA_ORDER = (POSE6, POINT3, FLOW2, VEL3, BIAS6)       # dynoba_solve: [poses 6 | points 3 | flows 2 | velocities 3 | biases 6]
REDUCED_ORDER = (POSE6, VEL3, BIAS6)                    # dynoba_get_reduced_system: [poses 6 | velocities 3 | biases 6]

# (np, npt, nfl, nv, nb): pose-only, visual-inertial, no landmarks of a kind, strides past one and two 32-column tiles
CASES = [(5, 7, 0, 0, 0), (40, 70, 33, 40, 40), (3, 0, 5, 3, 3), (0, 4, 0, 6, 6), (33, 1, 1, 0, 2), (12, 65, 31, 12, 0)]


def _build(tmp_path, patch=None):
    nvcc = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
    if nvcc is None:
        pytest.skip("nvcc not available")
    inc = [CSRC]
    if patch is not None:                      # a mutated copy of var_layout.cuh, seen only by this build
        src = open(os.path.join(CSRC, "var_layout.cuh")).read()
        assert src.count(patch[0]) == 1, patch
        d = str(tmp_path / "mut"); os.makedirs(d, exist_ok=True)
        open(os.path.join(d, "var_layout.cuh"), "w").write(src.replace(patch[0], patch[1]))
        inc = [d, CSRC]
    so = str(tmp_path / ("var_layout_host%s.so" % ("" if patch is None else "_mut")))
    cmd = [nvcc, "-x", "cu", "--shared", "-Xcompiler", "-fPIC,-fopenmp", "-O2", "-std=c++17", "-Wno-deprecated-gpu-targets"]
    for i in inc:
        cmd += ["-I", i]
    r = subprocess.run(cmd + [os.path.join(ROOT, "tests", "capi", "var_layout_host.cu"), "-o", so, "-lgomp"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(so)
    lib.host_column_checked.restype = C.c_int32
    lib.host_column_checked.argtypes = [C.c_int, C.c_int64]
    lib.host_reduced_map.restype = C.c_int64
    return lib


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return _build(tmp_path_factory.mktemp("var_layout"))


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _pad32(n):
    return -(-n//32)*32


# ------------------------------------------------------------------------------------------------------------ mirror
class Layout:
    """The documented layout of counts n = [np, npt, nfl, nv, nb] and the maps finalize builds"""

    def __init__(self, n, pos, pt_new, fl_new):
        self.n, self.pos, self.pt_new, self.fl_new = list(n), pos, pt_new, fl_new
        self.NP = n[POSE6] + n[VEL3] + n[BIAS6]

    def index(self, kind, i):
        """index of a pose-like variable in [poses | velocities | biases]"""
        return {POSE6: 0, VEL3: self.n[POSE6], BIAS6: self.n[POSE6] + self.n[VEL3]}[kind] + i

    def column(self, kind, i):
        if kind == POINT3:
            return int(self.pt_new[i])
        if kind == FLOW2:
            return int(self.fl_new[i])
        return int(self.pos[self.index(kind, i)])

    def stride(self, kind):
        return _pad32(self.NP if kind in POSELIKE else self.n[kind])

    def image(self, kind, vals_of):
        """the SoA image holding `kind` after every kind that shares it is scattered: identity in the rotation rows of an
        unused pose-image column, every row of a variable's column written (0 past its width)"""
        img = np.zeros((ROWS[kind], self.stride(kind)))
        if ROWS[kind] == 12:
            img[[0, 4, 8], :] = 1.0
        for k in (POSELIKE if kind in POSELIKE else (kind,)):
            for i in range(self.n[k]):
                img[:, self.column(k, i)] = np.r_[vals_of[k][i], np.zeros(ROWS[kind] - WIDTH[k])]
        return img

    def delta_slots(self):
        """(array name, flat index) of every scalar of the public delta, in order"""
        out = []
        for kind in DELTA_ORDER:
            for i in range(self.n[kind]):
                p = self.column(kind, i)
                for c in range(TDIM[kind]):
                    if kind == POINT3:
                        out.append(("pt", c*self.stride(POINT3) + p))
                    elif kind == FLOW2:
                        out.append(("fl", c*self.stride(FLOW2) + p))
                    else:
                        out.append(("r", 6*p + c))
        return out

    def reduced_map(self):
        m = np.full(6*self.NP, -1, np.int32)
        u = 0
        for kind in REDUCED_ORDER:
            for i in range(self.n[kind]):
                for c in range(TDIM[kind]):
                    m[6*self.column(kind, i) + c] = u; u += 1
        return m, u


def mirror_positions(n, hints):
    """dynoba_set_variable_order: pose-like variables ordered by (rank, kind: pose < velocity < bias, index); a kind
    without a hint ranks by index"""
    keys = [(int(hints[k][i]) if hints.get(k) is not None else i, k, i) for k in POSELIKE for i in range(n[k])]
    order = sorted(range(len(keys)), key=lambda v: keys[v])
    pos = np.empty(len(keys), np.int32)
    pos[order] = np.arange(len(keys), dtype=np.int32)
    return pos


def _random_layout(rng, n):
    NP = n[POSE6] + n[VEL3] + n[BIAS6]
    return Layout(n, rng.permutation(NP).astype(np.int32), rng.permutation(n[POINT3]).astype(np.int32),
                  rng.permutation(n[FLOW2]).astype(np.int32))


def _set(lib, L):
    strides = np.zeros(5, np.int32)
    lib.host_set_layout(_ptr(np.array(L.n, np.int64)), _ptr(L.pos), _ptr(L.pt_new), _ptr(L.fl_new), _ptr(strides))
    return strides


# ------------------------------------------------------------------------------------------------------------ checks
def check_kinds(lib, rng):
    t = np.zeros((5, 4), np.int32)
    lib.host_kinds(_ptr(t))
    return t.tolist() == [[WIDTH[k], TDIM[k], ROWS[k], int(k in POSELIKE)] for k in range(5)]


def _hint_sets(rng, n):
    """None, frame ids, ties across and inside kinds, a permutation"""
    F = max(n[POSE6], n[VEL3], n[BIAS6], 1)
    yield {}
    yield {k: np.arange(n[k], dtype=np.int32) for k in POSELIKE}
    yield {POSE6: rng.integers(0, 3, n[POSE6]).astype(np.int32)}
    yield {k: rng.integers(-2, 2, n[k]).astype(np.int32) for k in POSELIKE}
    yield {VEL3: rng.permutation(n[VEL3]).astype(np.int32), BIAS6: np.full(n[BIAS6], F//2, np.int32)}
    yield {k: rng.permutation(n[k]).astype(np.int32) for k in (POSE6, BIAS6)}


def check_order(lib, rng):
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        for hints in _hint_sets(rng, n):
            got = np.full(L.NP, -7, np.int32)
            lib.host_poselike_positions(_ptr(hints.get(POSE6)), _ptr(hints.get(VEL3)), _ptr(hints.get(BIAS6)), _ptr(got))
            if not np.array_equal(got, mirror_positions(n, hints)):
                return False
    return True


def check_strides_and_columns(lib, rng):
    for n in CASES:
        L = _random_layout(rng, n)
        if _set(lib, L).tolist() != [L.stride(k) for k in range(5)]:
            return False
        for k in range(5):
            if [lib.host_column_checked(k, i) for i in range(n[k])] != [L.column(k, i) for i in range(n[k])]:
                return False
            if lib.host_column_checked(k, -1) != -1 or lib.host_column_checked(k, n[k]) != -1:
                return False
        if lib.host_column_checked(5, 0) != -1 or lib.host_column_checked(-1, 0) != -1:
            return False
    return True


def check_values(lib, rng):
    """blank image, scatter of every kind that shares it, against the mirror image; gather round trip"""
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        vals = {k: rng.normal(size=(n[k], WIDTH[k])) for k in range(5)}
        for kind in (POSE6, POINT3, FLOW2):
            img = np.full((ROWS[kind], L.stride(kind)), np.nan)
            lib.host_blank_image(kind, _ptr(img))
            for k in (POSELIKE if kind == POSE6 else (kind,)):
                lib.host_scatter_values(k, _ptr(np.ascontiguousarray(vals[k])), _ptr(img))
            if not np.array_equal(img, L.image(kind, vals)):
                return False
            for k in (POSELIKE if kind == POSE6 else (kind,)):
                back = np.full((n[k], WIDTH[k]), np.nan)
                lib.host_gather_values(k, _ptr(img), _ptr(back))
                if not np.array_equal(back, vals[k]):
                    return False
    return True


def check_value_refresh(lib, rng):
    """one kind scattered over an image that holds the others: only its columns change, every row of them"""
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        vals = {k: rng.normal(size=(n[k], WIDTH[k])) for k in range(5)}
        for k in POSELIKE:
            img = L.image(POSE6, vals)
            new = dict(vals); new[k] = rng.normal(size=(n[k], WIDTH[k]))
            img[WIDTH[k]:, [L.column(k, i) for i in range(n[k])]] = 7.0     # stale rows past the width
            lib.host_scatter_values(k, _ptr(np.ascontiguousarray(new[k])), _ptr(img))
            if not np.array_equal(img, L.image(POSE6, new)):
                return False
    return True


def _delta_arrays(L, fill):
    return {"r": np.full(6*L.NP + 32, fill), "pt": np.full(3*L.stride(POINT3), fill), "fl": np.full(2*L.stride(FLOW2), fill)}


def check_delta(lib, rng):
    """retract direction (scatter) and solve direction (gather), untouched scalars left as they were"""
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        slots = L.delta_slots()
        dim = sum(n[k]*TDIM[k] for k in range(5))
        if len(slots) != dim:
            return False
        delta = rng.normal(size=dim)
        got, want = _delta_arrays(L, np.nan), _delta_arrays(L, np.nan)
        for u, (a, j) in enumerate(slots):
            want[a][j] = delta[u]
        lib.host_scatter_delta(_ptr(delta), _ptr(got["r"]), _ptr(got["pt"]), _ptr(got["fl"]))
        if not all(np.array_equal(got[a], want[a], equal_nan=True) for a in want):
            return False
        src = {a: rng.normal(size=v.size) for a, v in _delta_arrays(L, 0.0).items()}
        out = np.full(dim, np.nan)
        lib.host_gather_delta(_ptr(src["r"]), _ptr(src["pt"]), _ptr(src["fl"]), _ptr(out))
        if not np.array_equal(out, np.array([src[a][j] for a, j in slots])):
            return False
    return True


def check_reduced_map(lib, rng):
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        m = np.full(6*L.NP, -7, np.int32)
        dim = lib.host_reduced_map(_ptr(m))
        want, wdim = L.reduced_map()
        if dim != wdim or dim != 6*n[POSE6] + 3*n[VEL3] + 6*n[BIAS6] or not np.array_equal(m, want):
            return False
        if n[VEL3] and (m == -1).sum() != 3*n[VEL3]:      # the inert scalars of the velocities, and only those
            return False
    return True


def check_prior_table(lib, rng):
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        pool = [(k, i) for k in POSELIKE for i in range(n[k])]
        sel = [pool[j] for j in rng.permutation(len(pool))[:min(7, len(pool))]]
        kind = np.array([k for k, _ in sel], np.int32); idx = np.array([i for _, i in sel], np.int32)
        slot = np.full((len(sel), 4), -7, np.int32); sidx = np.full(sum(TDIM[k] for k in kind), -7, np.int32)
        lib.host_prior_table(C.c_int(len(sel)), _ptr(kind), _ptr(idx), _ptr(slot), _ptr(sidx))
        lo, want_slot, want_sidx = 0, [], []
        for k, i in sel:
            p = L.column(k, i)
            want_slot.append([k, p, lo, len(want_sidx)])
            lo += WIDTH[k]
            want_sidx += [6*p + c for c in range(TDIM[k])]
        if slot.tolist() != want_slot or sidx.tolist() != want_sidx:
            return False
    return True


def check_nav_table(lib, rng):
    for n in CASES:
        L = _random_layout(rng, n); _set(lib, L)
        nav = np.full((n[VEL3] + n[BIAS6], 2), -7, np.int32)
        lib.host_nav_table(_ptr(nav))
        want = [[L.column(k, i), TDIM[k]] for k in (VEL3, BIAS6) for i in range(n[k])]
        if nav.tolist() != want:
            return False
    return True


CHECKS = {f.__name__[6:]: f for f in (check_kinds, check_order, check_strides_and_columns, check_values, check_value_refresh,
                                      check_delta, check_reduced_map, check_prior_table, check_nav_table)}


def _failures(lib):
    return [name for name, f in CHECKS.items() if not f(lib, np.random.default_rng(11))]


@pytest.mark.parametrize("check", list(CHECKS))
def test_layout_equals_the_mirror(lib, check):
    assert CHECKS[check](lib, np.random.default_rng(11)), check


MUTATIONS = {
    "velocity and bias blocks of the pose-like index swapped":
        ("kind == DYNOBA_BIAS6 ? np + nv : (kind == DYNOBA_VEL3 ? np : 0)", "kind == DYNOBA_BIAS6 ? np : (kind == DYNOBA_VEL3 ? np + nb : 0)"),
    "kind tiebreak of the order dropped":
        ("std::make_tuple(hints[kind].empty() ? i : hints[kind][i], kind, i)", "std::make_tuple(hints[kind].empty() ? i : hints[kind][i], 0, i)"),
    "pose-image padding not a rotation":
        ("img[p] = img[(size_t)4*st + p] = img[(size_t)8*st + p] = 1.0", "img[p] = img[(size_t)4*st + p] = 1.0"),
    "rows past the width left stale": ("for (int k = 0; k < K.rows; k++)", "for (int k = 0; k < K.width; k++)"),
    "flows before points in the delta":
        ("{DYNOBA_POSE6, DYNOBA_POINT3, DYNOBA_FLOW2, DYNOBA_VEL3, DYNOBA_BIAS6}", "{DYNOBA_POSE6, DYNOBA_FLOW2, DYNOBA_POINT3, DYNOBA_VEL3, DYNOBA_BIAS6}"),
    "prior lin offset by tangent dimension": ("lo += KINDS[kind[i]].width", "lo += KINDS[kind[i]].tdim"),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutation_of_the_layout_fails(tmp_path, mutation):
    bad = _failures(_build(tmp_path, MUTATIONS[mutation]))
    print(f"variable layout mutation '{mutation}' caught by: {bad}")
    assert bad, mutation
