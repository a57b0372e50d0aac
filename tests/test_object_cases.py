"""The object axis of the front end on the CPU: the oracles draw the tracking mask as cv::circle saturates a label into CV_8U,
the std::sort restatement of propagate_mask's vote equals libstdc++'s std::sort (a C++ program compiled here), the oracle's vote
follows it where it departs from the first maximum in label order, and the case lists of tests/object_cases.py reach every
boundary they name."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import dynamic_klt_oracle as KO
import object_cases as OC
from oracle import frontend_oracle as FO

SATURATION_LABELS = [255, 256, 300, 2**31 - 1, -1]


def _cv2_disc(label, shape, xy, r):
    """what the reference draws: cv::circle(CV_8U image, xy, r, cv::Scalar(label), FILLED)"""
    import cv2
    img = np.zeros(shape, np.uint8)
    cv2.circle(img, xy, r, (float(label), 0.0, 0.0, 0.0), cv2.FILLED)
    return img


@pytest.mark.parametrize("label", SATURATION_LABELS)
def test_dense_flow_oracle_tracking_mask_saturates(label):
    mask = np.full((40, 60), label, np.int32)
    flow = np.zeros((40, 60, 2), np.float32); flow[..., 0] = 1.5; flow[..., 1] = 0.5
    r = FO.track_dynamic(np.array([[20.3, 15.6]]), [label], [1], [7], flow, mask, None, FO.TrackParams(), 100)
    assert r[0][0] == 1
    assert np.array_equal(r[8], _cv2_disc(label, (40, 60), (20, 15), 2))


@pytest.mark.parametrize("label", SATURATION_LABELS)
def test_dynamic_klt_oracle_tracking_mask_saturates(label):
    mask = np.full((40, 60), label, np.int32)
    kp = np.array([[20.0, 15.0]], np.float32); lk = np.array([[22.3, 16.6]], np.float32)
    r = KO.track_dynamic_klt(np.zeros((40, 60), np.uint8), mask, None, kp, [label], [1], [7], lk, [1], [], np.zeros((0, 4), np.int32),
                             KO.Params(), 100)
    assert r["state"][0] == KO.TRACKED
    assert np.array_equal(r["tracking_mask"], _cv2_disc(label, (40, 60), (22, 16), 2))


CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dynosam_b200", "frontend_csrc", "frontend.cu")
_SORT_CC = r"""
#include <algorithm>
#include <cstdio>
#include <utility>
#include <vector>
#define __device__
static inline int __clz(int x) { return __builtin_clz((unsigned)x); }
// the vote's sort restatement of frontend.cu (PmPair .. pm_introsort_loop), pasted in by the test
@DEVICE_CODE@
// reads vectors of (label, count) pairs, one per line as "n l0 c0 l1 c1 ...", and prints the labels after std::sort with the
// comparator of FeatureTracker::propogateMask, then "|" and the labels after pm_introsort_loop and a stable sort by the same
// comparator (what libstdc++'s final insertion sort does); pm_vote_kernel takes the first of them as sorted[0]
int main() {
  int n;
  while (std::scanf("%d", &n) == 1) {
    std::vector<std::pair<int, int>> v(n);
    std::vector<PmPair> d(n);
    for (int i = 0; i < n; i++) {
      if (std::scanf("%d %d", &v[i].first, &v[i].second) != 2) return 1;
      d[i] = PmPair{v[i].first, v[i].second};
    }
    std::sort(v.begin(), v.end(), [](const std::pair<int, int>& a, const std::pair<int, int>& b) { return a.second > b.second; });
    for (const auto& p : v) std::printf("%d ", p.first);
    pm_introsort_loop(d.data(), n);
    std::stable_sort(d.begin(), d.end(), [](const PmPair& a, const PmPair& b) { return a.c > b.c; });
    std::printf("|");
    for (const auto& p : d) std::printf(" %d", p.l);
    std::printf("\n");
  }
  return 0;
}
"""


def _device_sort_code():
    with open(CSRC) as f:
        src = f.read()
    return src[src.index("struct PmPair"):src.index("// one CTA: the votes")]


def _tie_heavy_vectors(count=1000, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        n = int(rng.integers(1, 41))
        c = rng.integers(0, int(rng.integers(1, 5)), n)                 # 1 to 4 distinct counts: many ties
        out.append([(int(i), int(x)) for i, x in enumerate(c)])
    return out


def _median_of_three_killer(n):
    """counts that drive libstdc++'s introsort to its depth limit: McIlroy's adversary ("A killer adversary for quicksort",
    1999) answers the restated sort's comparisons, fixing values lazily, and the values it fixed are the input"""
    gas = n; val = [gas]*n; st = {"solid": 0, "cand": 0}

    def cmp(x, y):
        if val[x] == gas and val[y] == gas:
            z = x if x == st["cand"] else y
            val[z] = st["solid"]; st["solid"] += 1
        if val[x] == gas:
            st["cand"] = x
        elif val[y] == gas:
            st["cand"] = y
        return val[x] - val[y]
    FO.libstdcxx_sort(list(range(n)), lambda a, b: cmp(a, b) < 0)
    return [(i, n - v) for i, v in enumerate(val)]                   # larger count first = ascending value


def test_sort_restatement_equals_libstdcxx(tmp_path):
    """libstdcxx_sort and the device's restatement (followed by the stable final insertion sort) against std::sort compiled with
    g++, full order: 1000 tie-heavy vectors of 1-40 pairs, and median-of-three killers of 40-3000 pairs that reach the depth
    limit, where introsort heap-sorts (with ties inside the heap-sorted ranges once the counts are divided by 2 and 3)"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ not available")
    src = tmp_path / "sort_pairs.cc"; exe = tmp_path / "sort_pairs"
    src.write_text(_SORT_CC.replace("@DEVICE_CODE@", _device_sort_code()))
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), str(src)], check=True, capture_output=True)
    killers = [[(i, c//q) for i, c in _median_of_three_killer(n)] for n in (40, 64, 200, 1000, 3000) for q in (1, 2, 3)]
    vecs = _tie_heavy_vectors() + killers
    text = "".join(f"{len(v)} " + " ".join(f"{a} {b}" for a, b in v) + "\n" for v in vecs)
    out = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(out) == len(vecs)
    departs = heap_sorted = tied_heap = 0
    for v, line in zip(vecs, out):
        order, dev = line.split("|")
        ranges = []
        got_pairs = FO.libstdcxx_sort(v, lambda a, b: a[1] > b[1], ranges)
        got = [a for a, _ in got_pairs]
        assert got == [int(x) for x in order.split()], v
        assert [int(x) for x in dev.split()] == got, v
        mx = max(c for _, c in v)
        departs += got[0] != next(a for a, c in v if c == mx)
        heap_sorted += bool(ranges)
        tied_heap += any(len({c for _, c in got_pairs[f:l]}) < l - f for f, l in ranges)      # equal counts in a heap-sorted range
    assert departs > 100, departs                          # the first maximum in label order is not what std::sort gives
    assert heap_sorted >= 5 and tied_heap >= 2, (heap_sorted, tied_heap)
    assert os.path.exists(exe)


def test_oracle_vote_without_votes():
    """an object whose key-points all fall outside the image has no vote: with min_votes = 0 it is skipped, not propagated"""
    prev = np.zeros((40, 60), np.int32); prev[5:15, 5:20] = 3
    flow = np.zeros((40, 60, 2), np.float32); flow[..., 0] = 2.5; flow[..., 1] = 1.5
    cur = np.zeros((40, 60), np.int32)
    out = FO.propagate_mask(np.array([[0.5, 10.5], [70.0, 10.0]]), [3, 3], prev, flow, cur, FO.TrackParams(), 0)
    assert np.array_equal(out, cur)


def _propagated(v: OC.VoteCase):
    kp, lab, prev, flow, cur = OC.vote_frame(v)
    out = FO.propagate_mask(kp, lab, prev, flow, cur, FO.TrackParams(), v.min_votes)
    return {obj: bool((out == obj).sum() > (cur == obj).sum()) for obj, _, _ in v.votes}


@pytest.mark.parametrize("name,expected", [("labels17_tie0_a", {8: True}), ("labels17_tie0_b", {8: False}),
                                           ("labels17_tie0_c", {8: False}), ("labels16_tie0", {7: True}),
                                           ("mode300_minority0", {300: False}), ("mode0_majority", {300: True}), ("negative_mode", {5: False}),
                                           ("below_min", {4: False}), ("at_min", {4: True}), ("above_min", {4: True}),
                                           ("sequential", {3: True, 4: False})])
def test_oracle_vote_follows_std_sort(name, expected):
    """the oracle propagates an object exactly when sorted[0] of the restated std::sort is label 0; at 17 labels that is not the
    first maximum in label order (A: 0 after -40, B: 7 after 0, C: 1 after 0)"""
    v = OC.VOTES[name]
    assert _propagated(v) == expected
    for obj, vs, _ in v.votes:
        if len(vs) == 17:
            first = next(l for l, c in vs if c == max(c for _, c in vs))
            assert (first == 0) != expected[obj]


def test_object_cases_reach_every_boundary():
    seen = set()
    for c in OC.CASES.values():
        b = OC.boundaries(c)
        assert set(c.hits) <= b, (c.name, set(c.hits) - b)
        assert len(set(c.listed)) == len(c.listed) and all(o > 0 for o in c.listed) and len(c.listed) <= 64, c.name
        seen |= set(c.hits)
    missing = set(OC.REQUIRED) - seen
    assert not missing, missing
    assert all(h in OC.REQUIRED for c in OC.CASES.values() for h in c.hits)
    seen = set()
    for v in OC.VOTES.values():
        b = OC.vote_boundaries(v)
        assert set(v.hits) <= b, (v.name, set(v.hits) - b)
        seen |= set(v.hits)
    missing = set(OC.VOTE_REQUIRED) - seen
    assert not missing, missing


@pytest.mark.parametrize("name", [n for n, c in OC.CASES.items() if c.layout == "grid"])
def test_grid_layout_shows_every_object(name):
    """every object of a grid case is visible with its own label, in both frames, and moves with its flow"""
    c = OC.CASES[name]
    (g0, m0, f0), (g1, m1, _) = OC.frames(c)
    for m in (m0, m1):
        assert set(np.unique(m).tolist()) == {0} | set(c.labels)
    for lab in c.labels[:3]:
        ys, xs = np.nonzero(m0 == lab)
        dx, dy = f0[ys[0], xs[0]]
        assert np.array_equal(g1[ys + int(round(float(dy))), xs + int(dx)], g0[ys, xs])


def test_vote_frames_make_the_votes():
    """the current-mask labels under each object's key-points are the votes the case names"""
    for v in OC.VOTES.values():
        kp, lab, prev, flow, cur = OC.vote_frame(v)
        for obj, vs, by in v.votes:
            sel = lab == obj
            got = cur[kp[sel, 1].astype(int), kp[sel, 0].astype(int)]
            want = {l: c for l, c in vs}
            if by is not None:                                  # before `by` paints, its votes land on the background
                want[0] = want.get(0, 0) + want.pop(by)
            assert dict(zip(*np.unique(got, return_counts=True))) == want, v.name
