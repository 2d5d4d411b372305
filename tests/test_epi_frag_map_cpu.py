"""CPU: the staging addresses of the fragment-native GEMM epilogue (wgmma.cuh stg_stmatrix_offset, option "tc_epi_frag"; 16-bit outputs).

The helper is compiled for the host from wgmma.cuh itself.  For every element of a 128 x BN tile (both consumer warpgroups, four warps
each, 32 lanes, every accumulator index) the byte stmatrix writes it to (lane l points matrix l / 8; register i of lane l holds row l / 4,
columns 2 (l & 3) and + 1 of matrix i) must be the byte stage_store16 writes for that (row, column), and the map must be a bijection onto
the staging tile."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

PROG = r"""
#include <cstdio>
#include "wgmma.cuh"
// per line: bn wg warp lane i offset - the byte the fragment path writes accumulator value d[i] of (wg, warp, lane) to
int main() {
  for (int bn = 64; bn <= 128; bn += 64)
    for (int wg = 0; wg < 2; ++wg)
      for (int w = 0; w < 4; ++w)
        for (int l = 0; l < 32; ++l)
          for (int i = 0; i < bn / 2; ++i) {
            // d[i] is in register m = (i & 7) / 2 of the stmatrix of block k = i / 8: matrix m, row l / 4, half i & 1 of the pair at 2 (l & 3)
            const int k = i / 8, m = (i & 7) / 2, src = 8 * m + l / 4;     // the lane that points matrix m's row l / 4
            printf("%d %d %d %d %d %u\n", bn, wg, w, l, i, stg_stmatrix_offset(64 * wg, w, src, k) + 4 * (l & 3) + 2 * (i & 1));
          }
  return 0;
}
"""


def _stage_store16_offset(row, col):
    """byte offset stage_store16 (gemm_tc.cu) writes 16-bit element (row, col) to: 16 consecutive columns of a row from a 16-aligned
    column c, two 16-byte chunks"""
    c, i = col - col % 16, col % 16
    sub = (c >> 6) * 16384 + row * 128
    ch = ((c & 63) >> 3) + (i >> 3)
    return sub + ((ch ^ (row & 7)) << 4) + 2 * (i & 7)


@pytest.fixture(scope="module")
def frag_map():
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not found")
    td = tempfile.mkdtemp()
    try:
        src, exe = os.path.join(td, "m.cu"), os.path.join(td, "m")
        open(src, "w").write(PROG)
        subprocess.check_call([NVCC, "-std=c++17", "-I", os.path.join(ROOT, "cosyvoice_b200", "csrc"), src, "-o", exe])
        out = subprocess.run([exe], check=True, stdout=subprocess.PIPE, text=True).stdout
    finally:
        shutil.rmtree(td, ignore_errors=True)
    return np.array([list(map(int, l.split())) for l in out.splitlines()], dtype=np.int64)


@pytest.mark.parametrize("bn", [64, 128])
def test_fragment_staging_matches_stage_store16(frag_map, bn):
    m = frag_map[frag_map[:, 0] == bn]
    wg, w, l, i, off = m[:, 1], m[:, 2], m[:, 3], m[:, 4], m[:, 5]
    # the accumulator layout (wgmma.cuh): d[i] of (warp w, lane l) is row 16 w + l / 4 + 8 ((i >> 1) & 1), column 8 (i >> 2) + 2 (l & 3) + (i & 1)
    row = 64 * wg + 16 * w + l // 4 + 8 * ((i >> 1) & 1)
    col = 8 * (i >> 2) + 2 * (l & 3) + (i & 1)
    assert len(m) == 128 * bn
    assert len(set(zip(row.tolist(), col.tolist()))) == 128 * bn                  # every element of the tile exactly once
    ref = np.array([_stage_store16_offset(r, c) for r, c in zip(row.tolist(), col.tolist())])
    bad = np.nonzero(off != ref)[0]
    assert bad.size == 0, [(int(row[k]), int(col[k]), int(off[k]), int(ref[k])) for k in bad[:5]]
    # a bijection onto the staging bytes: distinct element slots, together covering the tile's sub-tiles of 128-byte rows
    assert len(np.unique(off)) == len(off)
    assert np.array_equal(np.sort(off), 2 * np.arange(128 * bn))
