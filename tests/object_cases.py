"""Object lists and labels for the front end's per-object kernels (TEST INFRASTRUCTURE): named cases along the object axis, each
naming the boundaries it hits, in the style of frame_cases.Case; the frames for them (masks relabelled through a lookup table);
the hand-built votes of propagate_mask.

The boundaries of an object case:
  n0 n1 n2 n31 n32 n33 n63 n64   objects in the list of a call (ST_MAXOBJ = 64: warp ballots of 32 in the sampling scan, a
                                 6-bit object rank in trackDynamicKLT's candidate keys)
  contiguous        the labels are 1..n
  l255 l256 l257    labels around the 8-bit tracking mask and the old 256-bin vote
  l1000 l65535 l65536
  l2p24m1 l2p24 l2p24p1   2^24 - 1, 2^24, 2^24 + 1: (float)(size_t)id in Color::uniqueId stops being exact
  l2p31m1           the largest int32 id
  noncontiguous     labels with gaps
  ascending descending shuffled   the order of the object list
  absent_listed     a listed object has no pixels
  present_unlisted  a label of the mask is not in the list
  grid              every object visible (an 8 x 8 grid of textured rectangles with flows of their own)
  stream            SyntheticStream's overlapping layout, some of its objects hidden or outside the frame
The boundaries of a vote case (propagate_mask):
  mode_ge256_minority0   the mode of the votes is a label >= 256, a minority votes 0
  negative               votes on negative labels
  labels16_tie0 labels17_tie0   exactly 16 / 17 distinct vote labels, 0 tied for the maximum (libstdc++'s std::sort is an
                         insertion sort up to 16 elements, introsort partitions from 17)
  below_min at_min above_min    vote totals of min_votes - 1, min_votes, min_votes + 1
  sequential             two objects in turn, the second voting on pixels the first painted
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from dynosam_b200.synth_frames import SyntheticStream

W, H = 1242, 375
COUNT_BOUNDS = (0, 1, 2, 31, 32, 33, 63, 64)
LABEL_BOUNDS = {"l255": 255, "l256": 256, "l257": 257, "l1000": 1000, "l65535": 65535, "l65536": 65536, "l2p24m1": 2**24 - 1,
                "l2p24": 2**24, "l2p24p1": 2**24 + 1, "l2p31m1": 2**31 - 1}
REQUIRED = tuple(f"n{c}" for c in COUNT_BOUNDS) + ("contiguous",) + tuple(LABEL_BOUNDS) + (
    "noncontiguous", "ascending", "descending", "shuffled", "absent_listed", "present_unlisted", "grid", "stream")
VOTE_REQUIRED = ("mode_ge256_minority0", "negative", "labels16_tie0", "labels17_tie0", "below_min", "at_min", "above_min", "sequential")
ABSENT = 999_999                                          # listed, never in a mask


def _labels(n, special=(), seed=0):
    """n distinct positive labels: the special ones, then seeded gaps above 2000"""
    rng = np.random.default_rng(seed)
    out = list(special)
    while len(out) < n:
        c = int(rng.integers(2001, 2**30))
        if c not in out:
            out.append(c)
    return tuple(out[:n])


@dataclass(frozen=True)
class Case:
    name: str
    layout: str                 # "grid" or "stream"
    labels: tuple               # the label of layout object j (the raw mask's j + 1)
    listed: tuple               # the object list, in call order
    hits: tuple

    @property
    def n(self):
        return len(self.labels)


def boundaries(c: Case):
    """the boundaries of the module docstring that case c reaches"""
    b = {f"n{len(c.listed)}"} if len(c.listed) in COUNT_BOUNDS else set()
    b.add(c.layout)
    labs = set(c.labels)
    if labs == set(range(1, c.n + 1)):
        b.add("contiguous")
    elif c.n > 1:
        b.add("noncontiguous")
    b |= {k for k, v in LABEL_BOUNDS.items() if v in labs}
    lst = list(c.listed)
    if len(lst) > 1:
        if lst == sorted(lst):
            b.add("ascending")
        elif lst == sorted(lst, reverse=True):
            b.add("descending")
        else:
            b.add("shuffled")
    shown = set(np.unique(frames(c, (0,))[0][1]).tolist())
    if any(o not in shown for o in lst):
        b.add("absent_listed")
    if (shown - {0}) - set(lst):
        b.add("present_unlisted")
    return b


def _shuffled(labels, seed):
    out = list(labels)
    np.random.default_rng(seed).shuffle(out)
    return tuple(out)


_L64 = _labels(64, tuple(LABEL_BOUNDS.values()), 7)
CASES = {c.name: c for c in (
    Case("n0_contiguous", "grid", tuple(range(1, 9)), (), ("n0", "contiguous", "present_unlisted", "grid")),
    Case("n0_negative", "grid", (-1, -300, 2**31 - 1, 7, -2**31), (), ("n0", "l2p31m1", "noncontiguous", "present_unlisted", "grid")),
    Case("n1_l256", "grid", (256, 5, 9), (256,), ("n1", "l256", "noncontiguous", "present_unlisted", "grid")),
    Case("n2_l255_l257_desc", "grid", (255, 257, 4), (257, 255), ("n2", "l255", "l257", "descending", "present_unlisted", "grid")),
    Case("n31_l1000_shuffled", "grid", _labels(31, (1000, 65535), 1), _shuffled(_labels(31, (1000, 65535), 1), 1),
         ("n31", "l1000", "l65535", "noncontiguous", "shuffled", "grid")),
    Case("n32_l65536_asc", "grid", _labels(32, (65536, 2**24 - 1), 2), tuple(sorted(_labels(32, (65536, 2**24 - 1), 2))),
         ("n32", "l65536", "l2p24m1", "ascending", "grid")),
    Case("n33_l2p24_absent", "grid", _labels(32, (2**24, 2**24 + 1), 3), _shuffled(_labels(32, (2**24, 2**24 + 1), 3) + (ABSENT,), 3),
         ("n33", "l2p24", "l2p24p1", "absent_listed", "shuffled", "grid")),
    Case("n63_l2p31m1_desc", "grid", _labels(64, (2**31 - 1,), 4), tuple(sorted(_labels(64, (2**31 - 1,), 4)[:63], reverse=True)),
         ("n63", "l2p31m1", "descending", "present_unlisted", "grid")),
    Case("n64_contiguous_shuffled", "grid", tuple(range(1, 65)), _shuffled(range(1, 65), 5), ("n64", "contiguous", "shuffled", "grid")),
    Case("n64_edges_asc", "grid", _L64, tuple(sorted(_L64)), ("n64",) + tuple(LABEL_BOUNDS) + ("noncontiguous", "ascending", "grid")),
    Case("stream_l300", "stream", (300, 301, 256, 2**31 - 1, 65536, 7, 1000, 2**24 + 1, 255, 12), _shuffled((300, 301, 256, 2**31 - 1, 65536, 7, 1000, 2**24 + 1, 255, 12), 6),
         ("stream", "l256", "l2p31m1", "shuffled", "absent_listed")),
)}


# ------------------------------------------------------------------------------------------------ frames
def _texture(rng, h, w):
    import cv2
    return cv2.GaussianBlur(rng.integers(0, 256, (h, w)).astype(np.uint8), (0, 0), 1.2).astype(np.float64)


class GridStream:
    """n textured rectangles (n <= 64) on an 8 x 8 grid of 155 x 46 px cells at 1242 x 375, each moving by a whole-pixel velocity
    of its own inside its cell for the first frames; the background is a fixed texture with flow (-0.5, 0.25).  frame(k) is
    (gray uint8, raw mask int32 with object j as j + 1, flow float32[H][W][2]), the flow from frame k to k + 1."""

    def __init__(self, n, seed=11):
        rng = np.random.default_rng(seed)
        self.bg = _texture(rng, H, W)
        self.obj = []
        for j in range(n):
            cx, cy = 155*(j % 8), 46*(j//8)
            vx = int(rng.integers(-2, 3)) or 1; vy = int(rng.integers(-1, 2))
            self.obj.append(dict(x=cx + 8, y=cy + 5, w=139, h=36, vx=vx, vy=vy, tex=_texture(rng, 36, 139)))

    def frame(self, k):
        gray = self.bg.copy(); mask = np.zeros((H, W), np.int32)
        flow = np.zeros((H, W, 2), np.float32); flow[..., 0] = -0.5; flow[..., 1] = 0.25
        for j, o in enumerate(self.obj):
            x, y = o["x"] + o["vx"]*k, o["y"] + o["vy"]*k
            gray[y:y + o["h"], x:x + o["w"]] = o["tex"]
            mask[y:y + o["h"], x:x + o["w"]] = j + 1
            flow[y:y + o["h"], x:x + o["w"]] = (o["vx"], o["vy"] if o["vy"] else 1e-3)
        return np.clip(gray, 0, 255).astype(np.uint8), mask, flow


def relabel(raw_mask, labels):
    """the raw mask (0 background, j + 1 for layout object j) through the lookup table [0] + labels"""
    lut = np.array((0,) + tuple(labels), np.int64)
    return np.ascontiguousarray(lut[raw_mask].astype(np.int32))


def frames(c: Case, ks=(0, 1)):
    """[(gray, motion mask with the case's labels, flow)] of frames ks, C-contiguous"""
    src = GridStream(c.n) if c.layout == "grid" else SyntheticStream(n_objects=c.n, seed=4)      # seed 4: object 2 hidden in frames 0, 1
    out = []
    for k in ks:
        g, m, f = src.frame(k)
        out.append((np.ascontiguousarray(g, np.uint8), relabel(m, c.labels), np.ascontiguousarray(f, np.float32)))
    return out


# ------------------------------------------------------------------------------------------------ propagate_mask votes
@dataclass(frozen=True)
class VoteCase:
    """objects in ascending label order, each with its votes {current-mask label: count}; painted_by: the label whose warped
    pixels carry this object's votes (None: votes on pixels of their own)"""
    name: str
    votes: tuple                # ((object label, ((vote label, count), ...), painted_by), ...)
    min_votes: int
    hits: tuple


def vote_boundaries(v: VoteCase):
    b = set()
    for obj, vs, by in v.votes:
        d = dict(vs); tot = sum(d.values()); mx = max(d.values()) if d else 0
        mode_first = min(k for k, c in d.items() if c == mx) if d else None
        if d and mode_first >= 256 and 0 in d and d[0] < mx:
            b.add("mode_ge256_minority0")
        if any(k < 0 for k in d):
            b.add("negative")
        if len(d) in (16, 17) and d.get(0) == mx and sum(c == mx for c in d.values()) > 1:
            b.add(f"labels{len(d)}_tie0")
        b |= {{-1: "below_min", 0: "at_min", 1: "above_min"}[tot - v.min_votes]} if abs(tot - v.min_votes) <= 1 else set()
        if by is not None:
            b.add("sequential")
    return b


# 17 vote labels with 0 tied for the maximum, where libstdc++'s introsort and the first maximum in label order disagree: in A
# std::sort puts 0 first (the first maximum is -40), so the object is propagated; in B it puts 7 first (the first maximum is 0)
_T17_A = ((-40, 9), (0, 9), (1, 1), (2, 3), (3, 3), (4, 3), (5, 1), (6, 1), (7, 3), (8, 1), (9, 2), (10, 1), (11, 1), (12, 2), (13, 2),
          (14, 2), (300, 1))
_T17_B = ((-40, 3), (0, 9), (1, 2), (2, 1), (3, 1), (4, 9), (5, 2), (6, 3), (7, 9), (8, 2), (9, 9), (10, 2), (11, 1), (12, 1), (13, 2),
          (14, 1), (300, 9))
# C: every label in [0, 256) (all pairs from the vote kernel's histogram); std::sort puts 1 first, the first maximum is 0
_T17_C = ((0, 9), (1, 9), (2, 1), (3, 3), (4, 3), (5, 3), (6, 1), (7, 1), (8, 3), (9, 1), (10, 2), (11, 1), (12, 1), (13, 2), (14, 2),
          (15, 2), (16, 1))
VOTES = {v.name: v for v in (
    VoteCase("mode300_minority0", ((300, ((300, 190), (0, 10)), None),), 150, ("mode_ge256_minority0",)),
    VoteCase("mode0_majority", ((300, ((300, 10), (0, 190)), None),), 150, ()),
    VoteCase("negative_mode", ((5, ((-1, 120), (0, 60), (-300, 30)), None),), 150, ("negative",)),
    VoteCase("labels16_tie0", ((7, tuple((l, 6 if l in (0, 3, 9) else 2) for l in range(0, 16)), None),), 40, ("labels16_tie0",)),
    VoteCase("labels17_tie0_a", ((8, _T17_A, None),), 40, ("labels17_tie0", "negative")),
    VoteCase("labels17_tie0_b", ((8, _T17_B, None),), 40, ("labels17_tie0", "negative")),
    VoteCase("labels17_tie0_c", ((8, _T17_C, None),), 40, ("labels17_tie0",)),
    VoteCase("below_min", ((4, ((0, 19),), None),), 20, ("below_min",)),
    VoteCase("at_min", ((4, ((0, 20),), None),), 20, ("at_min",)),
    VoteCase("above_min", ((4, ((0, 15), (4, 6)), None),), 20, ("above_min",)),
    VoteCase("sequential", ((3, ((0, 40),), None), (4, ((0, 5), (3, 35)), 3)), 20, ("sequential",)),
)}


def vote_frame(v: VoteCase, w=320, h=160):
    """(prev_kp [n][2], prev_label [n], prev_mask, prev_flow, current_mask) that make the votes of v.  Every object j has a 30 x 20
    block of the previous mask in row band 0 that its flow (+2.5, +1.5) warps into the current frame; a vote on label L lands on a
    3 x 3 patch of L in the current mask (row band 1), a vote on 0 on the background, and a vote painted_by P on the pixels P's
    block warps onto (background in the current mask before P paints)."""
    prev = np.zeros((h, w), np.int32); flow = np.zeros((h, w, 2), np.float32); flow[..., 0] = 2.5; flow[..., 1] = 1.5
    cur = np.zeros((h, w), np.int32)
    block = {}
    for j, (obj, _, _) in enumerate(v.votes):
        x0, y0 = 10 + 50*j, 10
        prev[y0:y0 + 20, x0:x0 + 30] = obj; block[obj] = (x0 + 3, y0 + 2)      # a pixel its warp certainly paints
    patch = {}
    labs = sorted({l for _, vs, _ in v.votes for l, _ in vs if l != 0})
    for i, l in enumerate(labs):
        x0, y0 = 10 + 12*(i % 25), 60 + 12*(i//25)
        cur[y0:y0 + 3, x0:x0 + 3] = l; patch[l] = (x0 + 1, y0 + 1)
    kp, lab = [], []
    for obj, vs, by in v.votes:
        for l, cnt in vs:
            if by is not None and l == by:
                px, py = block[by][0] + 2, block[by][1] + 1        # painted by `by`, background before
            elif l == 0:
                px, py = 300, 150
            else:
                px, py = patch[l]
            kp += [(px + 0.25, py + 0.5)]*cnt; lab += [obj]*cnt
    return np.array(kp, np.float64).reshape(-1, 2), np.array(lab, np.int32), prev, flow, cur
