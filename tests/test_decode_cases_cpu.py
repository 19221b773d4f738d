"""CPU checks of the constructed decode cases (tests/decode_cases.py): every branch of the kernel the table names is
claimed by a case, and each case's maps reach what it claims when the kernel's strip, warp-segment and bucket-select
arithmetic is replayed on them."""
import os
import re

import numpy as np
import pytest

from oracle import decode_ref
from tests.decode_cases import (BND, BRANCHES, CAP, CASE, CASES, MAXJ, MAXK, SEG, TPB, Inputs, candidates,
                                owners, reached, select_rounds)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_every_branch_has_a_case():
    claimed = set().union(*(c.branches for c in CASES))
    assert claimed == set(BRANCHES), sorted(set(BRANCHES) ^ claimed)


@pytest.mark.parametrize("name", list(CASE))
def test_case_reaches_its_branches(name):
    case = CASE[name]
    assert case.reason and case.branches
    inp = case.build()
    assert isinstance(inp, Inputs)
    B, H, W, J = inp.shape
    assert set(inp.maps) == {"heat", "wh", "kps", "reg", "hm_hp", "hp_offset"}
    assert all(v.dtype == np.float32 and v.shape[0] == B and v.shape[2:] == (H, W) for v in inp.maps.values())
    assert 1 <= inp.K <= min(MAXK, H * W) and 1 <= J <= MAXJ
    missing = case.branches - reached(case, inp)
    assert not missing, sorted(missing)


def test_constants_match_the_kernel():
    src = open(os.path.join(ROOT, "centerpose_b200", "csrc", "decode.cu")).read()
    hdr = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    consts = dict(re.findall(r"constexpr int (\w+) = (\d+);", src))
    assert (int(consts["TPB"]), int(consts["CAP"]), int(consts["BND"])) == (TPB, CAP, BND)
    assert CAP // (TPB // 32) == SEG
    assert int(re.search(r"CPB200_DECODE_MAX_K (\d+)", hdr).group(1)) == MAXK
    assert int(re.search(r"CPB200_DECODE_MAX_J (\d+)", hdr).group(1)) == MAXJ


def test_strip_arithmetic():
    """scan_vec's (S, RS) split on the shapes of the scan cases, and the compaction order of one strip"""
    o = owners(12, 128, "vec")                  # XG 32, S 8, RS 2: strips 0..5 hold rows, warps 6 and 7 none
    assert o["strip"].max() == 5 and set(np.unique(o["warp"])) == set(range(6))
    o = owners(40, 40, "vec")                   # XG 10, S 25, RS 2: warp 0 = strips 0..3 (u 0..31)
    assert o["strip"][7, 0] == 3 and o["warp"][7, 4] == 0 and o["warp"][7, 8] == 1
    o = owners(8, 1100, "vec")                  # XG 275: one strip, column groups 256.. in the second pass
    assert o["strip"].max() == 0 and o["pas"][0, 4 * 256] == 1 and o["warp"][0, 4 * 256] == 0
    m = np.zeros((16, 128), np.float32)
    m[0, 5], m[1, 0], m[0, 7] = 0.5, 0.6, 0.4   # same warp (strip 0 of 8 rows x 2): row 0 before row 1
    vals, idx, counts = candidates(m, np.float32(0), "w128")
    assert idx.tolist() == [5, 7, 128] and counts[0] == 3


def test_select_rounds_outcomes():
    f = np.float32
    assert select_rounds(np.arange(1, 11, dtype=f), 10)[0] == "all"
    assert select_rounds(np.array([0.9, 0.5, 0.5, 0.1], f), 2)[:2] == ("resolve", 1)
    assert select_rounds(np.full(100, f(0.5)), 10)[0] == "give_up"


def test_sqrt_tie_case_is_the_references_choice():
    """joint 0 of 'sqrttie' goes to B (second in flat order, first in score order, larger squared distance)"""
    inp = CASE["sqrttie"].build()
    det = decode_ref.multi_pose_decode(**inp.maps, K=inp.K)
    assert det[0, 0, 5:7].tolist() == [np.float32(17.816463), np.float32(20.631685)]
    assert det[0, 0, 5 + 2 * 17] == np.float32(0.6)
    inp = CASE["sqrttie_swap"].build()
    det = decode_ref.multi_pose_decode(**inp.maps, K=inp.K)
    assert det[0, 0, 5:7].tolist() == [np.float32(22.783405), np.float32(20.632195)]
