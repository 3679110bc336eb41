// verify_core.cuh — the per-signature decision procedure (one thread = one signature).
//
// Implements, for the reference's crypto crate:
//   Signature::verify       (crypto/src/lib.rs:200-204)  -> flag HS_F_STRICT  (dalek verify_strict)
//   Signature::verify_batch (crypto/src/lib.rs:206-219)  -> AND over votes of flag HS_F_EQ (deterministic restatement of
//                                                            the per-signature equation; SURVEY App. A.3)
// Decision procedure (SURVEY App. A):
//   parse_ok = (S < l) and A decompresses                       [Signature::from_bytes / PublicKey::from_bytes]
//   k        = SHA-512(R || A || M) mod l
//   R'       = [S]B + [k](-A)
//   eq       = parse_ok and R decompresses and R' == R as points (no cofactor)
//   small    = R or A is one of the 8 torsion points
//   strict   = eq and not small
//
// Scalar multiplication layout (table gathers instead of doublings, not dalek's vartime NAF — see DESIGN.md):
//   [S]B      : signed radix-2^w comb over a precomputed table of j * 2^(w i) * B, affine-Niels entries (96 B); no
//               doublings.  w is chosen per context: 24 by default (11 windows, 8.9 GB of the H100's 80 GB of HBM).
//   [k](-A)   : committee key -> the same comb over that validator's own table (w = 17 .. 8 by committee size);
//               generic key   -> radix-2^4 signed fixed window, 8-entry per-thread table, 252 doublings + 64 additions.
//   Every lane executes the same operation sequence (identity entry for digit 0), so warps never diverge.
#pragma once
#include <cstdint>
#include "../../include/hs_crypto.h"  // HS_WHY_*: the per-check bits of explain_record are the C ABI's
#include "fe.cuh"
#include "ge.cuh"
#include "sc.cuh"
#include "sha512.cuh"

#define HS_F_PARSE_OK 1u
#define HS_F_EQ 4u
#define HS_F_SMALL 8u
#define HS_F_STRICT 16u

// Comb window widths are runtime parameters: wider windows trade HBM capacity and gather traffic for fewer field
// multiplications — the right trade on a part whose integer-multiply pipe, not its memory system, is the binding resource
// (DESIGN.md §roofline).  Entries per window = 2^(w-1) (signed digits), windows = sc_ndigits_rt(w).
struct comb_params {
  int wa, na;  // committee-key tables: window width, number of windows
  int wb, nb;  // base-point table
  uint32_t bias_a[9], bias_b[9];
};
// Table layout: window i occupies entries [i * (H + 1), (i + 1) * (H + 1)), H = 2^(w-1); entry 0 of a window is the
// identity (1, 1, 0) and entry m is m * 2^(w i) * P, so a digit of magnitude 0 .. H indexes the table directly — no
// "digit == 0" branch or select in the hot loop (one extra 96-byte entry per window).
HS_HD size_t comb_window_stride(int w) { return ((size_t)1 << (w - 1)) + 1; }
HS_HD size_t comb_table_entries(int w) { return (size_t)sc_ndigits_rt(w) * comb_window_stride(w); }
#define HS_MAX_DIGITS 64  // >= na + nb for every supported (wa, wb) pair (wa, wb >= 8)

// most-significant-digit-first stream over a radix-16 recoding (generic-key window method); W * ndigits must be 256
template <int W>
struct digits_msb {
  uint32_t u[8];
  HS_HD void init(const uint32_t (&s)[8]) {
    static_assert(W * sc_ndigits<W>() == 256, "msb stream needs W | 256");
    sc_recoded<W> r;
    sc_recode<W>(r, s);
    for (int i = 0; i < 8; i++) u[i] = r.u[i];
  }
  HS_HD int next() {
    int d = (int)(u[7] >> (32 - W)) - (1 << (W - 1));
    for (int i = 7; i > 0; i--) u[i] = (u[i] << W) | (u[i - 1] >> (32 - W));
    u[0] <<= W;
    return d;
  }
};

// ---- table-entry loads: 96 B, 32 B-aligned -> six 16-byte loads (three full sectors)
#if defined(__CUDA_ARCH__)
#define HS_NIELS_UNPACK(q, a, b, c, d, e, f)                                                        \
  q.ypx.v[0] = a.x; q.ypx.v[1] = a.y; q.ypx.v[2] = a.z; q.ypx.v[3] = a.w;                           \
  q.ypx.v[4] = b.x; q.ypx.v[5] = b.y; q.ypx.v[6] = b.z; q.ypx.v[7] = b.w;                           \
  q.ymx.v[0] = c.x; q.ymx.v[1] = c.y; q.ymx.v[2] = c.z; q.ymx.v[3] = c.w;                           \
  q.ymx.v[4] = d.x; q.ymx.v[5] = d.y; q.ymx.v[6] = d.z; q.ymx.v[7] = d.w;                           \
  q.xy2d.v[0] = e.x; q.xy2d.v[1] = e.y; q.xy2d.v[2] = e.z; q.xy2d.v[3] = e.w;                       \
  q.xy2d.v[4] = f.x; q.xy2d.v[5] = f.y; q.xy2d.v[6] = f.z; q.xy2d.v[7] = f.w;
#endif
HS_HD void niels_load(ge_niels &q, const ge_niels *p) {
#if defined(__CUDA_ARCH__)
  const uint4 *s = reinterpret_cast<const uint4 *>(p);
  uint4 a = __ldg(s + 0), b = __ldg(s + 1), c = __ldg(s + 2), d = __ldg(s + 3), e = __ldg(s + 4), f = __ldg(s + 5);
  HS_NIELS_UNPACK(q, a, b, c, d, e, f)
#else
  q = *p;
#endif
}
// streaming (evict-first) variant for the per-key tables: tens of GB of committee tables stream through L2
HS_HD void niels_load_stream(ge_niels &q, const ge_niels *p) {
#if defined(__CUDA_ARCH__)
  const uint4 *s = reinterpret_cast<const uint4 *>(p);
  uint4 a = __ldcs(s + 0), b = __ldcs(s + 1), c = __ldcs(s + 2), d = __ldcs(s + 3), e = __ldcs(s + 4), f = __ldcs(s + 5);
  HS_NIELS_UNPACK(q, a, b, c, d, e, f)
#else
  q = *p;
#endif
}

// acc += sum_i dig[i] * 2^(w i) * P using P's comb table; dig[] holds the signed digits (stride between digits)
HS_HD void ge_comb_accumulate_rt(ge_ext &acc, const ge_niels *table, const int32_t *dig, int stride, int w, int n) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < n; i++) {
    int d = dig[i * stride];
    uint32_t neg = (uint32_t)(d < 0);
    int mag = d < 0 ? -d : d;
    ge_niels q;
    niels_load(q, table + (size_t)i * comb_window_stride(w) + mag);
    ge_madd_signed(acc, acc, q, neg);
  }
}

// acc = sum over the A windows of digit * 2^(wa i) * (-A)  +  sum over the B windows of digit * 2^(wb i) * B.
// dig[0 .. na) are k's digits, dig[na .. na+nb) are S's.  ONE loop body (one copy of the mixed addition in the
// instruction cache).  Shape of an iteration (VERDICT r1 #4: keep non-multiply work off the integer-multiply pipe):
//   * the sign of the digit is applied AT LOAD TIME: -q = (ymx, ypx, -xy2d), so the two halves of the entry are simply
//     fetched into each other's registers (pointer selection, no fe_select), and the sign of xy2d is absorbed by choosing
//     which of F / G feeds X3 and Y3 (Z3 = F G is symmetric);
//   * the entry of iteration i+1 is fetched into the SAME registers right after the three multiplications that consume
//     entry i — the remaining four multiplications cover the latency, and there is no q = q_next register copy;
//   * digit 0 indexes the window's identity entry: no branch, no select.
struct niels_signed {  // table entry with the digit's sign applied to the first two coordinates
  fe m0, m1, xy2d;     // m0 multiplies (Y - X), m1 multiplies (Y + X)
};
HS_HD void niels_load_signed(niels_signed &q, const ge_niels *entry, uint32_t neg, bool stream) {
#if defined(__CUDA_ARCH__)
  const uint4 *s = reinterpret_cast<const uint4 *>(entry);
  const uint4 *p0 = s + (neg ? 0 : 2), *p1 = s + (neg ? 2 : 0);  // ypx at +0, ymx at +32 bytes
  uint4 a, b, c, d, e, f;
  if (stream) {
    a = __ldcs(p0); b = __ldcs(p0 + 1); c = __ldcs(p1); d = __ldcs(p1 + 1); e = __ldcs(s + 4); f = __ldcs(s + 5);
  } else {
    a = __ldg(p0); b = __ldg(p0 + 1); c = __ldg(p1); d = __ldg(p1 + 1); e = __ldg(s + 4); f = __ldg(s + 5);
  }
  q.m0.v[0] = a.x; q.m0.v[1] = a.y; q.m0.v[2] = a.z; q.m0.v[3] = a.w; q.m0.v[4] = b.x; q.m0.v[5] = b.y; q.m0.v[6] = b.z; q.m0.v[7] = b.w;
  q.m1.v[0] = c.x; q.m1.v[1] = c.y; q.m1.v[2] = c.z; q.m1.v[3] = c.w; q.m1.v[4] = d.x; q.m1.v[5] = d.y; q.m1.v[6] = d.z; q.m1.v[7] = d.w;
  q.xy2d.v[0] = e.x; q.xy2d.v[1] = e.y; q.xy2d.v[2] = e.z; q.xy2d.v[3] = e.w; q.xy2d.v[4] = f.x; q.xy2d.v[5] = f.y; q.xy2d.v[6] = f.z; q.xy2d.v[7] = f.w;
#else
  (void)stream;
  q.m0 = neg ? entry->ypx : entry->ymx;
  q.m1 = neg ? entry->ymx : entry->ypx;
  q.xy2d = entry->xy2d;
#endif
}
HS_HD const ge_niels *comb_entry(const ge_niels *atab, const ge_niels *btab, const int32_t *dig, int stride, int j, const comb_params &cp,
                                 uint32_t &neg, bool &is_a) {
  const int d = dig[j * stride];
  neg = (uint32_t)(d < 0);
  const int mag = d < 0 ? -d : d;
  is_a = j < cp.na;
  return is_a ? atab + (size_t)j * comb_window_stride(cp.wa) + mag : btab + (size_t)(j - cp.na) * comb_window_stride(cp.wb) + mag;
}
HS_HD void ge_comb_ab(ge_ext &acc, const ge_niels *atab, const ge_niels *btab, const int32_t *dig, int stride, const comb_params &cp) {
  const int NT = cp.na + cp.nb;
  niels_signed q;
  uint32_t neg, negn = 0;
  bool is_a;
  {
    // the first entry IS the accumulator's first value: identity + q costs one multiplication (affine Niels -> extended, scaled by 4:
    // X = 2(m1 - m0), Y = 2(m1 + m0), Z = 4, T = (m1 - m0)(m1 + m0)) instead of a 7-multiplication mixed addition
    const ge_niels *e = comb_entry(atab, btab, dig, stride, 0, cp, neg, is_a);
    niels_load_signed(q, e, neg, is_a);
    fe x2, y2;
    fe_sub(x2, q.m1, q.m0);
    fe_add(y2, q.m1, q.m0);
    fe_mul(acc.T, x2, y2);
    fe_add(acc.X, x2, x2);
    fe_add(acc.Y, y2, y2);
    fe_set0(acc.Z);
    acc.Z.v[0] = 4;
    if (NT > 1) {
      e = comb_entry(atab, btab, dig, stride, 1, cp, neg, is_a);
      niels_load_signed(q, e, neg, is_a);
    }
  }
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 1; i < NT; i++) {
    fe a, b, t, dd;
    fe_sub(t, acc.Y, acc.X);
    fe_mul(a, t, q.m0);
    fe_add(t, acc.Y, acc.X);
    fe_mul(b, t, q.m1);
    fe_mul(t, acc.T, q.xy2d);
    if (i + 1 < NT) {  // entry i is consumed: fetch entry i+1 into the same registers
      const ge_niels *e = comb_entry(atab, btab, dig, stride, i + 1, cp, negn, is_a);
      if (is_a) niels_load_signed(q, e, negn, true);   // per-key tables stream through L2 (evict-first)
      else niels_load_signed(q, e, negn, false);
    }
    fe_add(dd, acc.Z, acc.Z);
    fe E, H, F, G, P, Q;
    fe_sub(E, b, a);
    fe_add(H, b, a);
    fe_sub(F, dd, t);
    fe_add(G, dd, t);
    fe_select(P, F, G, neg);  // -q negates t, i.e. swaps F and G
    fe_select(Q, G, F, neg);
    fe_mul(acc.X, E, P);
    fe_mul(acc.Y, Q, H);
    fe_mul(acc.Z, F, G);
    if (i + 1 < NT) fe_mul(acc.T, E, H);  // nobody reads T after the last addition
    neg = negn;
  }
}

// ---- latency path (one WARP per signature): the na + nb table entries are summed as a binary tree across lanes instead of
// serially in one thread — 5 levels of point additions instead of 28 — and R is decompressed by a second warp meanwhile,
// so a single Signature::verify is bounded by one square-root chain, not by 28 mixed additions + an inversion.
// Entry of (signed) digit d as an extended point.  q holds the entry with its first two coordinates ordered by the sign
// (niels_load_signed): m1 = y'+x', m0 = y'-x' of the signed point, so X2 = m1 - m0 = 2x', Y2 = m1 + m0 = 2y' and
// (X : Y : Z : T) = (2 X2 : 2 Y2 : 4 : X2 Y2) is that point scaled by 4 — one multiplication, xy2d not needed.
HS_HD void ge_from_signed_niels(ge_ext &p, const fe &m0, const fe &m1) {
  fe x2, y2;
  fe_sub(x2, m1, m0);
  fe_add(y2, m1, m0);
  fe_mul(p.T, x2, y2);
  fe_add(p.X, x2, x2);
  fe_add(p.Y, y2, y2);
  fe_set0(p.Z);
  p.Z.v[0] = 4;
}
// r = p + q, both extended (9M; complete)
HS_HD void ge_add_ext(ge_ext &r, const ge_ext &p, const ge_ext &q) {
  ge_cached c;
  ge_to_cached(c, q);
  ge_add_cached(r, p, c);
}
// Projective equality with an affine point: (X : Y : Z) == (x, y)  <=>  X == x Z and Y == y Z   (Z != 0 on the curve)
HS_HD uint32_t ge_proj_equals_affine(const fe &X, const fe &Y, const fe &Z, const fe &x, const fe &y) {
  fe t;
  fe_mul(t, x, Z);
  uint32_t ex = fe_eq(t, X);
  fe_mul(t, y, Z);
  return ex & fe_eq(t, Y);
}

// acc = [k]P for an arbitrary point P (already negated by the caller when -A is wanted): radix-16 signed fixed window.
// tab: 9 cached entries of thread-private scratch (tab[j] = j*P, tab[0] = identity).
HS_HD void ge_scalarmult_window4(ge_ext &acc, const ge_ext &P, const uint32_t (&k)[8], ge_cached *tab) {
  ge_cached_identity(tab[0]);
  ge_to_cached(tab[1], P);
  ge_ext m;
  m = P;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int j = 2; j <= 8; j++) {
    ge_add_cached(m, m, tab[1]);  // complete formula: also correct for m == P (doubling) and torsion points
    ge_to_cached(tab[j], m);
  }
  digits_msb<4> ds;
  ds.init(k);
  ge_identity(acc);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < 64; i++) {
    if (i != 0) {
      // ONE copy of the doubling in the instruction stream (the 4x unrolled form made this loop body 5.2 k instructions and the
      // kernel's top stall "no instruction"); T is only needed after the last of the four
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
      for (int d = 0; d < 4; d++) {
        ge_p1p1 c;
        ge_dbl_p1p1(c, acc);
        ge_p1p1_to_proj(acc, c);
        if (d == 3) fe_mul(acc.T, c.E, c.H);
      }
    }
    int d = ds.next();
    uint32_t neg = (uint32_t)(d < 0);
    int mag = d < 0 ? -d : d;
    ge_cached q = tab[mag];
    ge_cached_cneg(q, neg);
    ge_add_cached(acc, acc, q);
  }
}

// ---- phase 1 ("main"): everything up to the projective result R' = [S]B + [k](-A) = (X : Y : Z).
// meta bit0 = parse_ok (S canonical, A decompresses), bit1 = small (R or A is a torsion point).
#define HS_META_PARSE_OK 1u
#define HS_META_SMALL 2u
#define HS_META_MISS 0x80u  // committee lookup miss: record is re-run through the generic path

// dig: thread-private digit slots (shared memory on the GPU: dig[i * dig_stride]), at least nb (generic) / na + nb entries
HS_HD uint32_t verify_generic_main(ge_ext &acc, const uint32_t (&R)[8], const uint32_t (&S)[8], const uint32_t (&A)[8],
                                   const uint32_t (&h)[16], const ge_niels *btable, ge_cached *tab, int32_t *dig, int dig_stride,
                                   const comb_params &cp) {
  uint32_t k[8];
  sc_reduce512(k, h);
  uint32_t s_ok = sc_is_canonical(S);
  ge_ext Apt, negA;
  uint32_t a_ok = ge_decompress(Apt, A);
  uint32_t small = ge_enc_is_small_order(R) | ge_enc_is_small_order(A);
  ge_neg(negA, Apt);
  ge_scalarmult_window4(acc, negA, k, tab);
  sc_digits_rt(dig, dig_stride, S, cp.bias_b, cp.wb, cp.nb);
  ge_comb_accumulate_rt(acc, btable, dig, dig_stride, cp.wb, cp.nb);
  return ((s_ok & a_ok) ? HS_META_PARSE_OK : 0u) | (small ? HS_META_SMALL : 0u);
}
// Committee key: -A's comb table was built at registration; a_flags bit0 = A decompressed, bit1 = A is small order.
HS_HD uint32_t verify_committee_main(ge_ext &acc, const uint32_t (&R)[8], const uint32_t (&S)[8], const uint32_t (&h)[16],
                                     const ge_niels *btable, const ge_niels *neg_a_table, uint32_t a_flags, int32_t *dig, int dig_stride,
                                     const comb_params &cp) {
  uint32_t s_ok, small;
  {
    uint32_t k[8];
    sc_reduce512(k, h);
    s_ok = sc_is_canonical(S);
    small = ge_enc_is_small_order(R) | ((a_flags >> 1) & 1u);
    sc_digits_rt(dig, dig_stride, k, cp.bias_a, cp.wa, cp.na);
    sc_digits_rt(dig + cp.na * dig_stride, dig_stride, S, cp.bias_b, cp.wb, cp.nb);
  }
  ge_comb_ab(acc, neg_a_table, btable, dig, dig_stride, cp);
  return ((s_ok & a_flags & 1u) ? HS_META_PARSE_OK : 0u) | (small ? HS_META_SMALL : 0u);
}

// ---- phase 2 ("finish"): affine comparison with R's encoding given 1/Z (the inversion is batched by the caller)
HS_HD uint32_t verify_flags_from(const fe &X, const fe &Y, const fe &zinv, const uint32_t (&R)[8], uint32_t meta) {
  uint32_t parse_ok = meta & HS_META_PARSE_OK, small = (meta & HS_META_SMALL) ? 1u : 0u;
  uint32_t eq = (ge_matches_encoding(X, Y, zinv, R) && parse_ok) ? 1u : 0u;
  uint32_t fl = 0;
  if (parse_ok) fl |= HS_F_PARSE_OK;
  if (eq) fl |= HS_F_EQ;
  if (small) fl |= HS_F_SMALL;
  if (eq && !small) fl |= HS_F_STRICT;
  return fl;
}

// ---- table construction (runs on the GPU at context creation / committee registration; also under host emu)
// Fills entries [first + 1, first + 1 + count) of window `win` of P's comb table: entry m = m * 2^(W win) * P as an
// affine Niels point (the call with first == 0 also writes the window's identity entry 0).  The forward pass parks (X, Y, Z) in the destination slots and the running product of the Z's in
// `prod` (count entries of scratch); one inversion then serves the whole block (Montgomery's trick).
HS_HD void comb_build_block(ge_niels *table, const ge_ext &P, int W, int win, int first, int count, fe *prod) {
  ge_ext base = P;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int i = 0; i < W * win; i++) ge_dbl(base, base);
  ge_cached cb;
  ge_to_cached(cb, base);
  // m = (first + 1) * base by double-and-add (first + 1 <= 2^(W-1))
  ge_ext m;
  ge_identity(m);
  const int mult = first + 1;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int b = W; b >= 0; b--) {
    ge_dbl(m, m);
    if ((mult >> b) & 1) ge_add_cached(m, m, cb);
  }
  ge_niels *slot = table + (size_t)win * comb_window_stride(W) + 1 + first;  // entry 0 of the window is the identity
  if (first == 0) ge_niels_identity(slot[-1]);
  fe run;
  fe_set1(run);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int c = 0; c < count; c++) {
    slot[c].ypx = m.X;
    slot[c].ymx = m.Y;
    slot[c].xy2d = m.Z;
    fe_mul(run, run, m.Z);
    prod[c] = run;
    if (c + 1 < count) ge_add_cached(m, m, cb);
  }
  fe u;
  fe_invert(u, run);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int c = count - 1; c >= 0; c--) {
    fe X = slot[c].ypx, Y = slot[c].ymx, Z = slot[c].xy2d, zinv, x, y;
    if (c > 0) fe_mul(zinv, u, prod[c - 1]);
    else zinv = u;
    fe_mul(u, u, Z);
    fe_mul(x, X, zinv);
    fe_mul(y, Y, zinv);
    ge_niels q;
    ge_affine_to_niels(q, x, y);
    fe_canon(q.ypx, q.ypx);  // canonical field elements: table bytes are representation-independent
    fe_canon(q.ymx, q.ymx);
    fe_canon(q.xy2d, q.xy2d);
    slot[c] = q;
  }
}

// ---- mend (hs_table_mend): the entries comb_build_block writes for (win, first, count), built into `stage` (count + 1 entries of
// scratch; stage[0] stands for entry `first`) and never into the table, then compared with the live entries of `window` (entry 0 of
// that window of the table): only an entry whose 96 bytes differ is stored, once, with its final affine bytes.  A correct entry is
// never written, so a gather that runs beside the mend reads a changed value only where the table was already wrong.  Returns the
// entries stored.
HS_HD uint32_t niels_store_if_differs(ge_niels *dst, const ge_niels &v) {
#if defined(__CUDA_ARCH__)
  uint4 *d = reinterpret_cast<uint4 *>(dst);
  const uint4 w[6] = {make_uint4(v.ypx.v[0], v.ypx.v[1], v.ypx.v[2], v.ypx.v[3]),     make_uint4(v.ypx.v[4], v.ypx.v[5], v.ypx.v[6], v.ypx.v[7]),
                      make_uint4(v.ymx.v[0], v.ymx.v[1], v.ymx.v[2], v.ymx.v[3]),     make_uint4(v.ymx.v[4], v.ymx.v[5], v.ymx.v[6], v.ymx.v[7]),
                      make_uint4(v.xy2d.v[0], v.xy2d.v[1], v.xy2d.v[2], v.xy2d.v[3]), make_uint4(v.xy2d.v[4], v.xy2d.v[5], v.xy2d.v[6], v.xy2d.v[7])};
  uint32_t diff = 0;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    const uint4 a = __ldcg(d + j);  // L2: the current bytes, never a stale L1 line
    diff |= (a.x ^ w[j].x) | (a.y ^ w[j].y) | (a.z ^ w[j].z) | (a.w ^ w[j].w);
  }
  if (!diff) return 0;
#pragma unroll
  for (int j = 0; j < 6; j++) d[j] = w[j];
  return 1;
#else
  if (!memcmp(dst, &v, sizeof(ge_niels))) return 0;
  memcpy(dst, &v, sizeof(ge_niels));
  return 1;
#endif
}
HS_HD uint32_t comb_mend_block(ge_niels *window, ge_niels *stage, const ge_ext &P, int W, int win, int first, int count, fe *prod) {
  // comb_build_block addresses the block from a table's start: given the stage's address less the block's offset in a table, it writes
  // entries first .. first + count to stage[0 ..], and k_build_comb keeps its code.
  comb_build_block(stage - (size_t)win * comb_window_stride(W) - first, P, W, win, first, count, prod);
  uint32_t stored = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int c = first ? 1 : 0; c <= count; c++) stored += niels_store_if_differs(window + first + c, stage[c]);
  return stored;
}

// ---- table audit (hs_table_audit): every entry of a built comb table checked against the layout above with the curve arithmetic the
// verify paths use, never with comb_build_block.  An entry passes when it is canonical, its third coordinate is 2dxy of the first two,
// and it is the previous entry of its window plus entry 1; entry 0 must be the identity, entry 1 of window 0 the table's point, and entry
// 1 of window i + 1 twice entry 2^(w-1) of window i.  By induction every entry is then m * 2^(w i) * P.
// An affine Niels entry as an extended point scaled by 4 (its X = 4x, Y = 4y, Z = 4, T = 4xy): 1 multiplication.
HS_HD void audit_niels_to_ext(ge_ext &p, const ge_niels &e) { ge_from_signed_niels(p, e.ymx, e.ypx); }
// (X : Y : Z) equals the point of entry e: with e's 2x = ypx - ymx and 2y = ypx + ymx, compare (2X : 2Y : Z) with (2x, 2y).
HS_HD uint32_t audit_proj_is_entry(const fe &X, const fe &Y, const fe &Z, const ge_niels &e) {
  fe x2, y2, X2, Y2;
  fe_sub(x2, e.ypx, e.ymx);
  fe_add(y2, e.ypx, e.ymx);
  fe_add(X2, X, X);
  fe_add(Y2, Y, Y);
  return ge_proj_equals_affine(X2, Y2, Z, x2, y2);
}
HS_HD uint32_t audit_fe_is_canonical(const fe &a) {
  fe t;
  fe_canon(t, a);
  uint32_t d = 0;
  for (int i = 0; i < 8; i++) d |= t.v[i] ^ a.v[i];
  return d == 0;
}
// The checks of entry m (> 0: m - 1 is prev) that need no other window: identity for m = 0; otherwise canonical coordinates,
// 2 xy2d == d (ypx^2 - ymx^2), and for m >= 2 e == prev + one (one = entry 1 of the same window).  1 = pass.
HS_HD uint32_t audit_entry_local(const ge_niels &e, const ge_niels &prev, const ge_niels &one, uint32_t m) {
  if (m == 0) {
    uint32_t d = (e.ypx.v[0] ^ 1u) | (e.ymx.v[0] ^ 1u) | e.xy2d.v[0];
    for (int i = 1; i < 8; i++) d |= e.ypx.v[i] | e.ymx.v[i] | e.xy2d.v[i];
    return d == 0;
  }
  uint32_t ok = audit_fe_is_canonical(e.ypx) & audit_fe_is_canonical(e.ymx) & audit_fe_is_canonical(e.xy2d);
  {
    fe a, b, d;
    fe_sqr(a, e.ypx);
    fe_sqr(b, e.ymx);
    fe_sub(a, a, b);
    fe_const(d, HS_CONST(HS_D));
    fe_mul(a, a, d);
    fe_add(b, e.xy2d, e.xy2d);
    ok &= fe_eq(a, b);
  }
  if (m >= 2) {
    ge_ext p;
    audit_niels_to_ext(p, prev);
    ge_p1p1 c;
    ge_madd_signed_p1p1(c, p, one, 0);
    fe X, Y, Z;
    fe_mul(X, c.E, c.F);
    fe_mul(Y, c.G, c.H);
    fe_mul(Z, c.F, c.G);
    ok &= audit_proj_is_entry(X, Y, Z, e);
  }
  return ok;
}
// Window link: entry 1 of window i + 1 (one) == 2 * entry 2^(w-1) of window i (last).
HS_HD uint32_t audit_link(const ge_niels &one, const ge_niels &last) {
  ge_ext p;
  audit_niels_to_ext(p, last);
  ge_p1p1 c;
  ge_dbl_p1p1(c, p);
  fe X, Y, Z;
  fe_mul(X, c.E, c.F);
  fe_mul(Y, c.G, c.H);
  fe_mul(Z, c.F, c.G);
  return audit_proj_is_entry(X, Y, Z, one);
}
// The point entry 1 of window 0 must hold: -A for the 32-byte key enc (returns 0 when it does not decompress), B for enc == nullptr.
HS_HD uint32_t audit_anchor_point(ge_ext &P, const uint32_t *enc) {
  if (!enc) {
    ge_basepoint(P);
    return 1;
  }
  uint32_t w[8];
  for (int i = 0; i < 8; i++) w[i] = enc[i];
  ge_ext A;
  const uint32_t ok = ge_decompress(A, w);
  ge_neg(P, A);
  return ok;
}
HS_HD uint32_t audit_anchor(const ge_niels &one, const ge_ext &P) { return audit_proj_is_entry(P.X, P.Y, P.Z, one); }
// The first finding of an audit, as one 64-bit key whose minimum is the first in (slot, window, entry) order: code 0 = the base table,
// s + 1 = key slot s; window field 0 = a finding about the slot itself (key bytes, flag, lookup), i + 1 = window i of its table.
HS_HD uint64_t audit_key(uint64_t code, uint32_t wfield, uint32_t entry) { return (code << 32) | ((uint64_t)wfield << 26) | entry; }
// The windows a finding at entry m of window win puts up for the mend (hs_table_mend), from its local checks (audit_entry_local) and
// its edge check (the anchor for window 0, the link otherwise; 1 for m != 1).  Bit 0: its own window, which holds every entry whose
// local check can fail.  Bit 1: the window before, as well, for a failed link: its entry 2^(w-1) may be the wrong one.  Bit 2: the
// anchor failed (window 0 is flagged too): the slot's key bytes may have changed instead, so only a map that confirms them lets it be
// mended.  A flagged window that is correct costs its recomputation and nothing else: the mend writes no correct entry.
HS_HD uint32_t audit_mend_flags(uint32_t win, uint32_t m, uint32_t local_ok, uint32_t edge_ok) {
  uint32_t f = (local_ok && edge_ok) ? 0u : 1u;
  if (m == 1 && !edge_ok) f |= win ? 2u : 4u;
  return f;
}

// ---- explanation of a verdict (hs_explain_rec128): every check of the decision procedure above as its own HS_WHY_* bit, evaluated
// independently (no "first failure"), with no table of any kind and without the fast paths' shortcuts: [S]B and [k](-A) both by the
// radix-16 window with B as an ordinary variable point (never btable or a comb), the equation as a projective compare with R
// decompressed (never ge_matches_encoding), and small order by three doublings of the decompressed point (never
// ge_enc_is_small_order, the encoding list the fast paths use), so the two small-order methods check each other.
//   strict verdict   <=> why == 0
//   batch-eq verdict <=> (why & ~(HS_WHY_A_SMALL | HS_WHY_R_SMALL)) == 0
// [8]P == identity, for a decompressed (affine) P: (X : Y : Z) == (0 : 1 : 1).
HS_HD uint32_t explain_is_small_order(const ge_ext &P) {
  ge_ext t;
  ge_dbl(t, P);
  ge_dbl(t, t);
  ge_dbl(t, t);
  return fe_is_zero(t.X) & fe_eq(t.Y, t.Z);
}
// h = SHA-512(R || A || M) as 16 words (k = h mod l).  tab: 9 cached entries of thread-private scratch, as ge_scalarmult_window4 takes.
HS_HD uint32_t explain_record(const uint32_t (&R)[8], const uint32_t (&S)[8], const uint32_t (&A)[8], const uint32_t (&h)[16], ge_cached *tab) {
  uint32_t why = sc_is_canonical(S) ? 0u : HS_WHY_S_NONCANONICAL;
  ge_ext Apt, Rpt;
  if (!ge_decompress(Apt, A)) why |= HS_WHY_A_INVALID;
  else if (explain_is_small_order(Apt)) why |= HS_WHY_A_SMALL;
  if (!ge_decompress(Rpt, R)) why |= HS_WHY_R_INVALID;
  else if (explain_is_small_order(Rpt)) why |= HS_WHY_R_SMALL;
  if (why & (HS_WHY_S_NONCANONICAL | HS_WHY_A_INVALID | HS_WHY_R_INVALID)) return why;
  uint32_t k[8];
  sc_reduce512(k, h);
  ge_ext negA, B, kA, sB, Rp;
  ge_neg(negA, Apt);
  ge_scalarmult_window4(kA, negA, k, tab);
  ge_basepoint(B);
  ge_scalarmult_window4(sB, B, S, tab);
  ge_add_ext(Rp, sB, kA);
  if (!ge_proj_equals_affine(Rp.X, Rp.Y, Rp.Z, Rpt.X, Rpt.Y)) why |= HS_WHY_EQUATION;
  return why;
}
// The flag byte verify_flags_from writes for the same record, from its explain_record mask: the signature cache's audit
// (hs_queue_sig_audit) re-derives a stored entry's flags with it, table-free.
HS_HD uint32_t flags_from_why(uint32_t why) {
  uint32_t fl = 0;
  if (!(why & (HS_WHY_S_NONCANONICAL | HS_WHY_A_INVALID))) fl |= HS_F_PARSE_OK;
  if (!(why & ~(HS_WHY_A_SMALL | HS_WHY_R_SMALL))) fl |= HS_F_EQ;
  if (why & (HS_WHY_A_SMALL | HS_WHY_R_SMALL)) fl |= HS_F_SMALL;
  if (!why) fl |= HS_F_STRICT;
  return fl;
}

// ---- signing (load generation only: SURVEY §8f.4 — the reference node signs on the CPU, one signature per request,
// crypto/src/lib.rs:185-191; this exists to synthesise 2^20-scale benchmark / test inputs in milliseconds).  RFC 8032 §5.1.6:
//   (a, prefix) = clamp / split of SHA-512(seed);  r = SHA-512(prefix || M) mod l;  R = [r]B;  k = SHA-512(R || A || M) mod l;
//   S = (r + k a) mod l.   M is a 32-byte Digest.  Deterministic: byte-identical to dalek / OpenSSL / the oracle.
HS_HD void ge_compress_words(uint32_t (&out)[8], const ge_ext &p) {
  fe zinv, x, y;
  fe_invert(zinv, p.Z);
  fe_mul(x, p.X, zinv);
  fe_mul(y, p.Y, zinv);
  fe_canon(x, x);
  fe_canon(y, y);
  for (int i = 0; i < 8; i++) out[i] = y.v[i];
  out[7] |= (x.v[0] & 1u) << 31;
}
// r (8 limbs) + k (8 limbs) * a (8 limbs), reduced mod l.  a < 2^255, k < l, r < l: the 512-bit intermediate cannot overflow.
HS_HD void sc_muladd(uint32_t (&out)[8], const uint32_t (&k)[8], const uint32_t (&a)[8], const uint32_t (&r)[8]) {
  uint32_t t[16];
  for (int i = 0; i < 16; i++) t[i] = (i < 8) ? r[i] : 0u;
  for (int i = 0; i < 8; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < 8; j++) {
      uint64_t v = (uint64_t)k[i] * a[j] + t[i + j] + carry;
      t[i + j] = (uint32_t)v;
      carry = v >> 32;
    }
    for (int j = i + 8; j < 16 && carry; j++) {
      uint64_t v = (uint64_t)t[j] + carry;
      t[j] = (uint32_t)v;
      carry = v >> 32;
    }
  }
  sc_reduce512(out, t);
}
HS_HD void sha512_two_words32(uint32_t (&out)[16], const uint32_t (&p)[8], const uint32_t (&q)[8]) {  // SHA-512(p[32] || q[32])
  uint64_t w[16];
  for (int i = 0; i < 4; i++) {
    w[i] = be64_from_le32(p[2 * i], p[2 * i + 1]);
    w[4 + i] = be64_from_le32(q[2 * i], q[2 * i + 1]);
  }
  w[8] = 0x8000000000000000ULL;
  for (int i = 9; i < 15; i++) w[i] = 0;
  w[15] = 64 * 8;
  sha512_state s;
  sha512_init(s);
  sha512_compress(s, w);
  sha512_output_words(s, out);
}
// dig: na/nb scratch digit slots as in the verify paths.  sig_r / sig_s receive the two halves of the signature.
HS_HD void sign_digest_core(uint32_t (&sig_r)[8], uint32_t (&sig_s)[8], const uint32_t (&seed)[8], const uint32_t (&A)[8], const uint32_t (&M)[8],
                            const ge_niels *btable, int32_t *dig, int dig_stride, const comb_params &cp) {
  uint32_t h[16], a[8], prefix[8], r[8], k[8];
  {  // SHA-512(seed): one block of 32 bytes
    uint64_t w[16];
    for (int i = 0; i < 4; i++) w[i] = be64_from_le32(seed[2 * i], seed[2 * i + 1]);
    w[4] = 0x8000000000000000ULL;
    for (int i = 5; i < 15; i++) w[i] = 0;
    w[15] = 32 * 8;
    sha512_state s;
    sha512_init(s);
    sha512_compress(s, w);
    sha512_output_words(s, h);
  }
  for (int i = 0; i < 8; i++) {
    a[i] = h[i];
    prefix[i] = h[8 + i];
  }
  a[0] &= 0xfffffff8u;                  // clamp: clear the low 3 bits, clear bit 255, set bit 254
  a[7] = (a[7] & 0x7fffffffu) | 0x40000000u;
  sha512_two_words32(h, prefix, M);
  sc_reduce512(r, h);
  ge_ext Rp;
  ge_identity(Rp);
  sc_digits_rt(dig, dig_stride, r, cp.bias_b, cp.wb, cp.nb);
  ge_comb_accumulate_rt(Rp, btable, dig, dig_stride, cp.wb, cp.nb);
  ge_compress_words(sig_r, Rp);
  sha512_ram32(h, sig_r, A, M);
  sc_reduce512(k, h);
  sc_muladd(sig_s, k, a, r);
}
// public key of a seed: A = [a]B
HS_HD void keygen_core(uint32_t (&A)[8], const uint32_t (&seed)[8], const ge_niels *btable, int32_t *dig, int dig_stride, const comb_params &cp) {
  uint32_t h[16], a[8];
  uint64_t w[16];
  for (int i = 0; i < 4; i++) w[i] = be64_from_le32(seed[2 * i], seed[2 * i + 1]);
  w[4] = 0x8000000000000000ULL;
  for (int i = 5; i < 15; i++) w[i] = 0;
  w[15] = 32 * 8;
  sha512_state s;
  sha512_init(s);
  sha512_compress(s, w);
  sha512_output_words(s, h);
  for (int i = 0; i < 8; i++) a[i] = h[i];
  a[0] &= 0xfffffff8u;
  a[7] = (a[7] & 0x7fffffffu) | 0x40000000u;
  // the comb recoder takes scalars below 2^253: split a = a_lo + 2^252 * a_hi (a_hi in 4 .. 7) is avoided by reducing mod l first
  uint32_t t[16], ar[8];
  for (int i = 0; i < 16; i++) t[i] = (i < 8) ? a[i] : 0u;
  sc_reduce512(ar, t);                  // [a]B = [a mod l]B
  ge_ext P;
  ge_identity(P);
  sc_digits_rt(dig, dig_stride, ar, cp.bias_b, cp.wb, cp.nb);
  ge_comb_accumulate_rt(P, btable, dig, dig_stride, cp.wb, cp.nb);
  ge_compress_words(A, P);
}
