// frag_layout.cuh -- the per-knot RECORD consumed by the register-resident Riccati kernel (riccati_frag.cu) and written by the
// error-state expansion kernels (rollout.cu k_expand_lie_rec / k_expansion_rec16b, riccati_frag.cu k_expansion_rec).
//
// The backward pass of the error-state Quadrotor (n_e = 12, m = 4, z = [x_e; u] of 16 entries) keeps its whole recursion state in
// the fragment registers of mma.sync.m8n8k4.f64 (lane L = 4 fr + fc holds A[fr][fc], B[fc][fr], D[fr][2fc], D[fr][2fc+1]).  For
// the outputs of one product to be the operands of the next without any data movement, z is held in a PHYSICAL order p = 0..15:
//      u_a            <->  p = 2a                       (class (tile 0, reg 0) of a D fragment: columns 0,2,4,6)
//      x_e, 12 of them <-> the other three classes      k-step 0: p = 2fc+1   k-step 1: p = 8+2fc   k-step 2: p = 9+2fc
// with the attitude error (e = 3,4,5) on p = 8,10,12 so that the only non-diagonal block of the compact cost/AL expansion is the
// even-even 4 x 4 sub-block of tile (1,1).  tests/frag_emulator.py restates the lane algebra in NumPy; tests/test_frag_layout.py
// checks it against the dense recursion.
//
// Record of knot k (TO_REC_LEN = 240 doubles = 1920 B, one 1-D bulk TMA copy):
//   [  0,192)  [A_e B_e]_k as MMA fragments: element (ks, lane, mi) at (ks*32 + lane)*2 + mi  =  AB_e[e(q(ks,fc))][col(p = 8mi+fr)]
//   [192,208)  g~[p]   error-state gradient of cost + AL terms, physical order
//   [208,224)  hd[p]   diagonal of the error-state Hessian
//   [224,240)  Hb[a][b] = H~[8+2a][8+2b]   (attitude block + the diagonal entries it overlaps)
// The terminal knot uses only [192,240).
#pragma once

#define TO_REC_LEN 240
#define TO_REC_G 192
#define TO_REC_HD 208
#define TO_REC_HB 224

namespace fraglayout {
// logical error-state index e = 0..11 (r, phi, v, omega) -> physical index ; logical control a -> 2a
__host__ __device__ constexpr int phys_x(int e) {
    return e == 0 ? 1 : e == 1 ? 3 : e == 2 ? 5 : e == 3 ? 8 : e == 4 ? 10 : e == 5 ? 12 : e == 6 ? 7 : e == 7 ? 14 : e == 8 ? 9 : e == 9 ? 11 : e == 10 ? 13 : 15;
}
__host__ __device__ constexpr int phys_z(int j) { return j < 12 ? phys_x(j) : 2 * (j - 12); }   // logical z index (x_e then u_a)
// physical index -> logical error-state index, -1 for the control slots
__host__ __device__ constexpr int e_of_p(int p) {
    return p == 1 ? 0 : p == 3 ? 1 : p == 5 ? 2 : p == 8 ? 3 : p == 10 ? 4 : p == 12 ? 5 : p == 7 ? 6 : p == 14 ? 7 : p == 9 ? 8 : p == 11 ? 9 : p == 13 ? 10 : p == 15 ? 11 : -1;
}
// position inside the fragment block of the record of AB_e[row e][logical column j]
__host__ __device__ constexpr int ab_index(int e, int j) {
    const int q = phys_x(e);
    const int ks = (q < 8) ? 0 : ((q & 1) ? 2 : 1);
    const int fc = (q < 8) ? (q - 1) / 2 : ((q & 1) ? (q - 9) / 2 : (q - 8) / 2);
    const int c = phys_z(j);
    return (ks * 32 + 4 * (c & 7) + fc) * 2 + (c >> 3);
}
// place of double d of a knot's [A_e B_e] block in the shared-memory image of knot kk of rollout.cu k_expand_lie_rec: bits 1..3 (the 16-byte
// chunk within the 128-byte line) XOR the line index mod 4 (bits 4..5) and the knot's parity -- a permutation inside each line, so that the
// column stores of a warp spread over the shared-memory banks while the line stores still read every bank once
__host__ __device__ constexpr int stage_swz(int d, int kk) { return d ^ ((((d >> 4) & 3) | ((kk & 1) << 2)) << 1); }
}  // namespace fraglayout
