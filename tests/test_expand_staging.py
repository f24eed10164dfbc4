"""CPU check of the record-path dynamics expansion's staging (csrc/rollout.cu k_expand_lie_rec): a NumPy restatement of which thread writes
which slot of a knot's shared-memory image of the [A_e B_e] block, and of the line-store loop that copies the images into the records.
The index functions are the compiled ones (frag_layout.cuh ab_index / stage_swz through g++); the CTA shape and the seed tables are read
from rollout.cu."""
import os
import re
import subprocess
import tempfile

import numpy as np

import frag_emulator as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "trajectoryoptimization.jl_b200", "csrc")
REC_LEN, AB_LEN = 240, 192                 # doubles per record; the [A_e B_e] block is its first 192 (1536 bytes)


def _rollout_constants():
    src = open(os.path.join(CSRC, "rollout.cu")).read()
    kpb = int(re.search(r"#define EXPB_KPB (\d+)", src).group(1))
    t = int(re.search(r"#define EXPB_T (\d+)", src).group(1))
    seed = int(re.search(r"lie_seed\(int s\) \{ return \(int\)\(\((0x[0-9A-F]+)ULL", src).group(1), 16)
    triv = int(re.search(r"lie_trivial\(int s\) \{ return \(int\)\(\((0x[0-9A-F]+)ULL", src).group(1), 16)
    return kpb, t, [(seed >> (4 * s)) & 15 for s in range(10)], [(triv >> (4 * s)) & 15 for s in range(6)]


def _compiled_tables(kpb):
    src = r'''
#include <cstdio>
#define __host__
#define __device__
#include "frag_layout.cuh"
int main() {
    for (int e = 0; e < 12; e++) for (int j = 0; j < 16; j++) printf("%d ", fraglayout::ab_index(e, j));
    printf("\n");
    for (int kk = 0; kk < KPB; kk++) for (int d = 0; d < 192; d++) printf("%d ", fraglayout::stage_swz(d, kk));
    printf("\n");
    return 0;
}
'''
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.cpp"), "w").write(src)
        subprocess.check_call(["g++", "-std=c++17", f"-DKPB={kpb}", "-x", "c++", "-I", CSRC, os.path.join(d, "t.cpp"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")], text=True).splitlines()
    ab = np.array([int(v) for v in out[0].split()]).reshape(12, 16)
    swz = np.array([int(v) for v in out[1].split()]).reshape(kpb, AB_LEN)
    return ab, swz


KPB, T, SEEDS, TRIVIAL = _rollout_constants()
AB, SWZ = _compiled_tables(KPB)


def test_seed_tables_and_cta_shape():
    assert SEEDS == [3, 4, 5, 9, 10, 11, 12, 13, 14, 15] and TRIVIAL == [0, 1, 2, 6, 7, 8]
    assert sorted(SEEDS + TRIVIAL) == list(range(16))
    assert KPB * 10 <= T and T % 32 == 0
    # at N = 101 (100 knots per instance) no more than about a tenth of the lanes idles
    nkb = -(-100 // KPB)
    assert 1 - 1000 / (nkb * T) <= 0.10


def test_swizzle_is_a_permutation_inside_each_line():
    for kk in range(KPB):
        s = SWZ[kk]
        d = np.arange(AB_LEN)
        assert np.array_equal(s, d ^ ((((d >> 4) & 3) | ((kk & 1) << 2)) << 1))     # restated
        assert sorted(s) == list(range(AB_LEN))
        assert np.array_equal(s >> 4, d >> 4)                                        # stays in its 128-byte line
        assert np.array_equal(s & 1, d & 1)                                          # and in its half of a 16-byte chunk


def _stage(nk):
    """the image the CTA's threads write: image[kk][slot] = (e, j) of the element, and how often each slot is written"""
    img = np.full((KPB, AB_LEN, 2), -1)
    count = np.zeros((KPB, AB_LEN), dtype=int)
    for tid in range(T):
        kk, sd = tid // 10, tid % 10
        if kk >= nk:
            continue
        cols = [SEEDS[sd]] + ([TRIVIAL[sd]] if sd < 6 else [])
        for jj in cols:
            c = FE.PHYS[jj]
            cb = 8 * (c & 7) + (c >> 3)
            for e in range(12):
                assert (AB[e, 12] | cb) == AB[e, jj] and (AB[e, 12] & cb) == 0         # the kernel's OR of disjoint bits = ab_index(e, jj)
                slot = SWZ[kk][AB[e, 12] | cb]
                img[kk, slot] = (e, jj)
                count[kk, slot] += 1
    return img, count


def test_every_slot_of_the_image_is_written_exactly_once():
    for nk in range(1, KPB + 1):
        img, count = _stage(nk)
        assert np.all(count[:nk] == 1) and np.all(count[nk:] == 0)
        for kk in range(nk):                                                     # every (row, column) once, seed and closed-form columns
            assert sorted(map(tuple, img[kk])) == [(e, j) for e in range(12) for j in range(16)]


def test_line_stores_write_bytes_0_to_1536_of_each_record_in_record_order():
    for N in (2, 3, 7, 8, 13, 101, 102):
        nkb = -(-(N - 1) // KPB)
        B = 2
        for b in range(B):
            written = np.zeros(B * N * REC_LEN * 8, dtype=int)                   # bytes of the record array
            rec = np.full((B * N * REC_LEN, 2), -1)
            for kb in range(nkb):
                k0 = kb * KPB
                nk = min(KPB, N - 1 - k0)
                img, _ = _stage(nk)
                base = (b * N + k0) * REC_LEN
                for warp in range(T // 32):
                    for q in range(warp, nk, T // 32):
                        for lane in range(32):
                            for r in range(3):
                                w = lane + 32 * r
                                src = SWZ[q][2 * w] >> 1                         # the 16-byte chunk of the image
                                dst = base + q * REC_LEN + 2 * w                 # double index of the store
                                assert (dst * 8) % 16 == 0
                                written[dst * 8:dst * 8 + 16] += 1
                                rec[dst] = img[q, 2 * src]; rec[dst + 1] = img[q, 2 * src + 1]
            w = written.reshape(B * N, REC_LEN * 8)
            for bb in range(B):
                for k in range(N):
                    expect = 1 if (bb == b and k < N - 1) else 0                 # the terminal knot has no [A_e B_e] block
                    assert np.all(w[bb * N + k, :AB_LEN * 8] == expect), (N, bb, k)
                    assert np.all(w[bb * N + k, AB_LEN * 8:] == 0)               # the expansion part [192, 240) is never touched
            for k in range(N - 1):
                r = rec[(b * N + k) * REC_LEN:(b * N + k) * REC_LEN + AB_LEN]
                for e in range(12):
                    for j in range(16):
                        assert tuple(r[AB[e, j]]) == (e, j)                      # element (e, j) lands on ab_index(e, j)
