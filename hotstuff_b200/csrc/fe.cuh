// fe.cuh — GF(2^255-19) arithmetic for the sm_90a Ed25519 engine.
//
// Representation: 8 saturated 32-bit limbs, little-endian, value anywhere in [0, 2^256) and only
// meaningful mod p = 2^255-19 (2^256 = 38 mod p).  This is NOT dalek's 5x51 / 10x25.5 layout: one
// IMAD.WIDE.U32.X does a 32x32->64 multiply-accumulate with carry-in/out,
// so a saturated-limb schoolbook product costs 64 of them and no separate carry handling (fe_asm.cuh), versus
// 100 for the 10-limb layout.  Replaces the field arithmetic that the reference reaches through
// ed25519-dalek (crypto/Cargo.toml:10) on every Signature::verify (crypto/src/lib.rs:200-204).
//
// HS_HOST_EMU: when compiled by a host compiler (tests/hostemu) the PTX paths are replaced by portable C
// so the exact same curve / scalar / window logic can be unit-tested against the oracle without a GPU.
// That build is test-only; the product library is CUDA-only and has no CPU path.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define HS_HD __host__ __device__ __forceinline__
#else
#define HS_HD inline
#endif

#if defined(__CUDA_ARCH__)
#include "fe_asm.cuh"
#endif

struct fe {
  uint32_t v[8];
};

// ---------------------------------------------------------------- portable wide helpers (host emu + rarely-used paths)
HS_HD void fe_reduce16_c(uint32_t (&r)[8], const uint32_t (&c)[16]) {
  uint64_t acc = 0;
  uint32_t t[9];
  for (int i = 0; i < 8; i++) {
    acc += (uint64_t)c[i] + (uint64_t)c[8 + i] * 38u;
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  t[8] = (uint32_t)acc;
  acc = (uint64_t)t[8] * 38u;
  for (int i = 0; i < 8; i++) {
    acc += t[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  t[0] += (uint32_t)acc * 38u;
  for (int i = 0; i < 8; i++) r[i] = t[i];
}

HS_HD void fe_mul_c(uint32_t (&r)[8], const uint32_t (&a)[8], const uint32_t (&b)[8]) {
  uint32_t c[16];
  for (int i = 0; i < 16; i++) c[i] = 0;
  for (int i = 0; i < 8; i++) {
    uint64_t carry = 0;
    for (int j = 0; j < 8; j++) {
      uint64_t t = (uint64_t)a[i] * b[j] + c[i + j] + carry;
      c[i + j] = (uint32_t)t;
      carry = t >> 32;
    }
    c[i + 8] = (uint32_t)carry;
  }
  fe_reduce16_c(r, c);
}

// ---------------------------------------------------------------- mul / sqr
HS_HD void fe_mul(fe &r, const fe &a, const fe &b) {
#if defined(__CUDA_ARCH__)
  uint32_t t[8];
#if defined(HS_FE_KARATSUBA)
  fe_mul_karatsuba_asm(t, a.v, b.v);  // experiment: 56 wide multiplies + ~117 ALU ops instead of 72 + 37
#else
  fe_mul_asm(t, a.v, b.v);
#endif
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#else
  uint32_t t[8];
  fe_mul_c(t, a.v, b.v);
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#endif
}

HS_HD void fe_sqr(fe &r, const fe &a) {
#if defined(__CUDA_ARCH__)
  uint32_t t[8];
  fe_sqr_asm(t, a.v);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#else
  uint32_t t[8];
  fe_mul_c(t, a.v, a.v);
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#endif
}

// ---------------------------------------------------------------- add / sub (result in [0, 2^256))
HS_HD void fe_add(fe &r, const fe &a, const fe &b) {
#if defined(__CUDA_ARCH__)
  uint32_t t[8];
  fe_add_asm(t, a.v, b.v);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#else
  uint64_t acc = 0;
  uint32_t t[8];
  for (int i = 0; i < 8; i++) {
    acc += (uint64_t)a.v[i] + b.v[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  acc *= 38u;
  for (int i = 0; i < 8; i++) {
    acc += t[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  t[0] += (uint32_t)acc * 38u;
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#endif
}

HS_HD void fe_sub(fe &r, const fe &a, const fe &b) {
#if defined(__CUDA_ARCH__)
  uint32_t t[8];
  fe_sub_asm(t, a.v, b.v);
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#else
  int64_t acc = 0;
  uint32_t t[8];
  for (int i = 0; i < 8; i++) {
    acc += (int64_t)a.v[i] - (int64_t)b.v[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;  // arithmetic shift: -1 on borrow
  }
  acc *= 38;  // 0 or -38
  for (int i = 0; i < 8; i++) {
    acc += t[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  t[0] -= (uint32_t)(-acc) * 38u;
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
#endif
}

// ---------------------------------------------------------------- small helpers
HS_HD void fe_set0(fe &r) {
  for (int i = 0; i < 8; i++) r.v[i] = 0;
}
HS_HD void fe_set1(fe &r) {
  fe_set0(r);
  r.v[0] = 1;
}
HS_HD void fe_copy(fe &r, const fe &a) {
  for (int i = 0; i < 8; i++) r.v[i] = a.v[i];
}
HS_HD void fe_neg(fe &r, const fe &a) {
  fe z;
  fe_set0(z);
  fe_sub(r, z, a);
}
// r = c ? b : a   (c is 0/1; branch-free select)
HS_HD void fe_select(fe &r, const fe &a, const fe &b, uint32_t c) {
  uint32_t m = 0u - c;
  for (int i = 0; i < 8; i++) r.v[i] = (a.v[i] & ~m) | (b.v[i] & m);
}
HS_HD void fe_cswap(fe &a, fe &b, uint32_t c) {
  uint32_t m = 0u - c;
  for (int i = 0; i < 8; i++) {
    uint32_t t = (a.v[i] ^ b.v[i]) & m;
    a.v[i] ^= t;
    b.v[i] ^= t;
  }
}

// 32 little-endian bytes (as 8 u32 words) -> fe; bit 255 is dropped, the value is NOT required to be < p
// (dalek FieldElement::from_bytes semantics, SURVEY App. A.1).
HS_HD void fe_from_words(fe &r, const uint32_t (&w)[8]) {
  for (int i = 0; i < 8; i++) r.v[i] = w[i];
  r.v[7] &= 0x7fffffffu;
}

// Fully reduce to the canonical representative in [0, p).
HS_HD void fe_canon(fe &r, const fe &a) {
  // fold bit 255: v = (v mod 2^255) + 19*(v >> 255)  -> < 2^255 + 19
  uint32_t top = a.v[7] >> 31;
  uint64_t acc = (uint64_t)top * 19u;
  uint32_t t[8];
  for (int i = 0; i < 8; i++) {
    acc += (i == 7) ? (a.v[7] & 0x7fffffffu) : a.v[i];
    t[i] = (uint32_t)acc;
    acc >>= 32;
  }
  // if t >= p then t -= p  <=>  if (t + 19) has bit 255 set then t = t + 19 - 2^255 ; this can be needed twice
  // only when t >= 2^255 (t < 2^255+19 -> t-p < 38), so one more pass covers it.
  for (int pass = 0; pass < 2; pass++) {
    uint32_t u[8];
    uint64_t c = 19;
    for (int i = 0; i < 8; i++) {
      c += t[i];
      u[i] = (uint32_t)c;
      c >>= 32;
    }
    uint32_t ge = (u[7] >> 31) | (uint32_t)c;  // t + 19 >= 2^255
    uint32_t m = 0u - (ge & 1u);
    u[7] &= 0x7fffffffu;
    for (int i = 0; i < 8; i++) t[i] = (t[i] & ~m) | (u[i] & m);
  }
  for (int i = 0; i < 8; i++) r.v[i] = t[i];
}
HS_HD uint32_t fe_is_zero(const fe &a) {
  fe t;
  fe_canon(t, a);
  uint32_t acc = 0;
  for (int i = 0; i < 8; i++) acc |= t.v[i];
  return acc == 0;
}
HS_HD uint32_t fe_eq(const fe &a, const fe &b) {
  fe t;
  fe_sub(t, a, b);
  return fe_is_zero(t);
}
// "negative" = least significant bit of the canonical encoding (RFC 8032 §5.1.2)
HS_HD uint32_t fe_is_neg(const fe &a) {
  fe t;
  fe_canon(t, a);
  return t.v[0] & 1u;
}

HS_HD void fe_sqr_n(fe &r, const fe &a, int n) {
  fe_sqr(r, a);
#pragma unroll 1
  for (int i = 1; i < n; i++) fe_sqr(r, r);
}

// z^(2^250-1); also returns z^11.  (Standard 2,9,11,2^5-1,2^10-1,... ladder for 2^255-19.)
HS_HD void fe_pow2_250_1(fe &out, fe &z11, const fe &z) {
  fe z2, z9, t, a, b, c;
  fe_sqr(z2, z);
  fe_sqr_n(t, z2, 2);
  fe_mul(z9, t, z);
  fe_mul(z11, z9, z2);
  fe_sqr(t, z11);
  fe_mul(a, t, z9);  // 2^5-1
  fe_sqr_n(t, a, 5);
  fe_mul(b, t, a);  // 2^10-1
  fe_sqr_n(t, b, 10);
  fe_mul(c, t, b);  // 2^20-1
  fe_sqr_n(t, c, 20);
  fe_mul(t, t, c);  // 2^40-1
  fe_sqr_n(t, t, 10);
  fe_mul(b, t, b);  // 2^50-1
  fe_sqr_n(t, b, 50);
  fe_mul(c, t, b);  // 2^100-1
  fe_sqr_n(t, c, 100);
  fe_mul(t, t, c);  // 2^200-1
  fe_sqr_n(t, t, 50);
  fe_mul(out, t, b);  // 2^250-1
}
// z^(p-2)
HS_HD void fe_invert(fe &r, const fe &z) {
  fe t, z11;
  fe_pow2_250_1(t, z11, z);
  fe_sqr_n(t, t, 5);
  fe_mul(r, t, z11);
}
// z^((p-5)/8) = z^(2^252-3)
HS_HD void fe_pow_p58(fe &r, const fe &z) {
  fe t, z11;
  fe_pow2_250_1(t, z11, z);
  fe_sqr_n(t, t, 2);
  fe_mul(r, t, z);
}
