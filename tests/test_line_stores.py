"""The shared-memory layout of the LineStores column (serve_device.cuh), the staging of the wide slot instance's fast path.

A flush round has lane group g = lane >> 3 load the eight 16-byte windows of one lane's 128-byte line, lane t = lane & 7
window t, as four 32-bit loads (word j of the window in load j).  Those loads must not conflict within a quarter-warp,
and the appends (every lane of a warp storing its word k) must not conflict at all.  The bank of a 32-bit word is its
index mod 32; the word indices come from the device address function, LineStores::window_word, compiled on the host."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ROWS, T = 39, 128  # GOFR_LINE_WORDS rows; threads per CTA

_PROG = r"""
#include <stdio.h>
#include "serve_device.cuh"
int main() {
    printf("%u %u\n", GOFR_LINE_WORDS, gofr::LineStores::kRowWords);
    for (unsigned s = 0; s < @T@; s++)
        for (unsigned w = 0; w < 10; w++)
            for (unsigned j = 0; j < 4; j++) printf("%u\n", gofr::LineStores::window_word(s, w, j));
    return 0;
}
"""


@pytest.fixture(scope="module")
def word(tmp_path_factory):
    d = tmp_path_factory.mktemp("line_stores")
    src, exe = d / "words.cpp", d / "words"
    src.write_text(_PROG.replace("@T@", str(T)))
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-w", "-I", os.path.join(ROOT, "gofr_b200", "csrc"), "-o", str(exe), str(src)])
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    rows, row_words = map(int, out[0].split())
    assert (rows, row_words) == (ROWS, T + 1)
    vals = [int(x) for x in out[1:] if x]
    return lambda s, w, j: vals[(s * 10 + w) * 4 + j]


def test_window_loads_conflict_free_per_quarter_warp(word):
    for s in range(T):  # the lane whose line a group stores, in any warp of the CTA
        for j in range(4):
            banks = [word(s, t, j) % 32 for t in range(8)]
            assert len(set(banks)) == 8, (s, j, banks)


def test_round_of_consecutive_lanes_conflict_free(word):
    # when four neighbouring lanes have a line (every lane does in a one-shape warp) one load touches 32 banks
    for warp0 in range(0, T, 32):
        for first in range(0, 32, 4):
            for j in range(4):
                banks = [word(warp0 + first + g, t, j) % 32 for g in range(4) for t in range(8)]
                assert len(set(banks)) == 32, (warp0, first, j)


def test_appends_conflict_free_and_inside_the_ring(word):
    for warp0 in range(0, T, 32):
        for k in range(ROWS):
            words = [word(warp0 + lane, k >> 2, k & 3) for lane in range(32)]
            assert len({x % 32 for x in words}) == 32, (warp0, k)
            assert max(words) < ROWS * (T + 1)
