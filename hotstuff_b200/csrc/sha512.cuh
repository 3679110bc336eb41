// sha512.cuh — SHA-512 (FIPS 180-4) for the verify kernels and the Digest surface.
//
// Replaces: ed25519_dalek::Sha512 as used for k = H(R || A || M) inside Signature::verify / verify_batch
// (crypto/src/lib.rs:200-219) and for Digest = SHA-512(..)[..32] at consensus/src/messages.rs:81,151,203,270,308
// and mempool/src/processor.rs:30.
//
// One thread hashes one message (Merkle–Damgård is sequential within a message; parallelism is across
// signatures / messages).  The 80 rounds are fully unrolled over a rolling 16-word schedule so every index
// is a compile-time constant and the schedule lives in registers.
#pragma once
#include <cstdint>
#include "fe.cuh"
#include "hs_constants.cuh"

#if defined(__CUDACC__)
__device__ __constant__ uint64_t HS_SHA512_K_DEV[80] = {HS_SHA512_K_INIT};
__device__ __constant__ uint32_t HS_ONE_DEV = 1;
 // opaque multiplier: keeps ptxas from folding mad.wide(x, 1, y) back into ALU adds
#endif

HS_HD uint64_t sha_k(int i) {
#if defined(__CUDA_ARCH__)
  return HS_SHA512_K_DEV[i];
#else
  return HS_SHA512_K_HOST[i];
#endif
}

HS_HD uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
// SHA-512 on a 32-bit datapath is ALU-pipe bound (funnel shifts, LOP3 and add-with-carry all issue there).  The round is
// therefore written on explicit 32-bit halves: a 64-bit rotate is exactly two funnel shifts (SHF.R.W), each three-way xor /
// Ch / Maj one LOP3 per half, and the halves are packed with mov.b64 (free: a register pair) so that ptxas still sees 64-bit
// adds and merges them into three-input IADD3 / IADD3.X pairs.  Per round: 24 SHF + 12 LOP3 + 12 add = 48 instructions
// (r1 code, left to the compiler from uint64_t expressions: 67, with shifts split into IMAD.SHL + SHF + extra LOP3).
// Experiment HS_SHA_FMA_ADD moves half of every 64-bit add to the FMA pipe (x + y = mad.wide(x_lo, 1, y) + (x_hi << 32)).
// It and rotations on the FMA pipe (x * 2^(32-n) as IMAD.WIDE yields both shifted halves; 24 SHF -> 24 IMAD.WIDE + 8 LOP3 per round:
// ALU instructions 46 -> 36 per round) were slower where they were measured; the kernel stays on the ALU pipe.
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ uint64_t sha_pack(uint32_t lo, uint32_t hi) {
  uint64_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
  return r;
}
__device__ __forceinline__ void sha_unpack(uint32_t &lo, uint32_t &hi, uint64_t x) { asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(x)); }
template <int N>
__device__ __forceinline__ uint32_t sha_rot_lo(uint32_t lo, uint32_t hi) {
  return N < 32 ? __funnelshift_r(lo, hi, N) : (N == 32 ? hi : __funnelshift_r(hi, lo, N - 32));
}
template <int N>
__device__ __forceinline__ uint32_t sha_rot_hi(uint32_t lo, uint32_t hi) {
  return N < 32 ? __funnelshift_r(hi, lo, N) : (N == 32 ? lo : __funnelshift_r(lo, hi, N - 32));
}
template <int A, int B, int C>
__device__ __forceinline__ uint64_t sha_big_sigma(uint64_t x) {  // rotr A ^ rotr B ^ rotr C
  uint32_t l, h;
  sha_unpack(l, h, x);
  return sha_pack(sha_rot_lo<A>(l, h) ^ sha_rot_lo<B>(l, h) ^ sha_rot_lo<C>(l, h), sha_rot_hi<A>(l, h) ^ sha_rot_hi<B>(l, h) ^ sha_rot_hi<C>(l, h));
}
template <int A, int B, int C>
__device__ __forceinline__ uint64_t sha_small_sigma(uint64_t x) {  // rotr A ^ rotr B ^ shr C   (C < 32)
  uint32_t l, h;
  sha_unpack(l, h, x);
  return sha_pack(sha_rot_lo<A>(l, h) ^ sha_rot_lo<B>(l, h) ^ __funnelshift_r(l, h, C), sha_rot_hi<A>(l, h) ^ sha_rot_hi<B>(l, h) ^ (h >> C));
}
__device__ __forceinline__ uint64_t sha_ch(uint64_t e, uint64_t f, uint64_t g) {
  uint32_t el, eh, fl, fh, gl, gh;
  sha_unpack(el, eh, e);
  sha_unpack(fl, fh, f);
  sha_unpack(gl, gh, g);
  return sha_pack((el & fl) ^ (~el & gl), (eh & fh) ^ (~eh & gh));
}
__device__ __forceinline__ uint64_t sha_maj(uint64_t a, uint64_t b, uint64_t c) {
  uint32_t al, ah, bl, bh, cl, ch;
  sha_unpack(al, ah, a);
  sha_unpack(bl, bh, b);
  sha_unpack(cl, ch, c);
  return sha_pack((al & bl) ^ (al & cl) ^ (bl & cl), (ah & bh) ^ (ah & ch) ^ (bh & ch));
}
#define HS_SIG1(e) sha_big_sigma<14, 18, 41>(e)
#define HS_SIG0(a) sha_big_sigma<28, 34, 39>(a)
#define HS_SSIG0(w) sha_small_sigma<1, 8, 7>(w)
#define HS_SSIG1(w) sha_small_sigma<19, 61, 6>(w)
#define HS_CH(e, f, g) sha_ch(e, f, g)
#define HS_MAJ(a, b, c) sha_maj(a, b, c)
#else
#define HS_SIG1(e) (rotr64(e, 14) ^ rotr64(e, 18) ^ rotr64(e, 41))
#define HS_SIG0(a) (rotr64(a, 28) ^ rotr64(a, 34) ^ rotr64(a, 39))
#define HS_SSIG0(w) (rotr64(w, 1) ^ rotr64(w, 8) ^ ((w) >> 7))
#define HS_SSIG1(w) (rotr64(w, 19) ^ rotr64(w, 61) ^ ((w) >> 6))
#define HS_CH(e, f, g) (((e) & (f)) ^ (~(e) & (g)))
#define HS_MAJ(a, b, c) (((a) & (b)) ^ ((a) & (c)) ^ ((b) & (c)))
#endif
HS_HD uint64_t add64_fma(uint64_t x, uint64_t y) {
#if defined(__CUDA_ARCH__) && defined(HS_SHA_FMA_ADD)
  uint64_t t;
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(t) : "r"((uint32_t)x), "r"(HS_ONE_DEV), "l"(y));
  return t + (x & 0xffffffff00000000ULL);
#else
  return x + y;
#endif
}
HS_HD uint32_t bswap32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(x, 0, 0x0123);
#else
  return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24);
#endif
}
// big-endian 64-bit message word from two little-endian 32-bit memory words (lo = bytes 0..3, hi = bytes 4..7)
HS_HD uint64_t be64_from_le32(uint32_t lo, uint32_t hi) { return ((uint64_t)bswap32(lo) << 32) | bswap32(hi); }

struct sha512_state {
  uint64_t h[8];
};

HS_HD void sha512_init(sha512_state &s) {
  const uint64_t h0[8] = {HS_SHA512_H0_INIT};
  for (int i = 0; i < 8; i++) s.h[i] = h0[i];
}

// One compression; w[16] is consumed (used as the rolling schedule).
// Code shape: 16 fully unrolled rounds over the loaded block, then a 4-trip loop whose body is 16 unrolled rounds with
// the schedule update — every w[] / state index is a compile-time constant (registers), but the hot body is ~2.5 k
// instructions instead of the ~8.5 k of an 80-round unroll, which thrashed the instruction cache (ncu: 6 of every 10
// stall cycles of the digest kernel were "no instruction").
#define HS_SHA_ROUND(a, b, c, d, e, f, g, h, kw)                                 \
  {                                                                              \
    uint64_t t1_ = add64_fma(add64_fma(h, HS_SIG1(e)), add64_fma(HS_CH(e, f, g), (kw))); \
    uint64_t t2_ = add64_fma(HS_SIG0(a), HS_MAJ(a, b, c));                       \
    d = add64_fma(d, t1_);                                                       \
    h = add64_fma(t1_, t2_);                                                     \
  }
#define HS_SHA_SCHED(w, j)                                                                          \
  {                                                                                                 \
    uint64_t w15_ = w[((j) + 1) & 15], w2_ = w[((j) + 14) & 15];                                    \
    w[(j) & 15] = add64_fma(add64_fma(w[(j) & 15], HS_SSIG0(w15_)), add64_fma(w[((j) + 9) & 15], HS_SSIG1(w2_))); \
  }
#define HS_SHA_8ROUNDS(w, base, j0)                                   \
  HS_SHA_ROUND(a, b, c, d, e, f, g, h, sha_k((base) + (j0) + 0) + w[(j0) + 0]) \
  HS_SHA_ROUND(h, a, b, c, d, e, f, g, sha_k((base) + (j0) + 1) + w[(j0) + 1]) \
  HS_SHA_ROUND(g, h, a, b, c, d, e, f, sha_k((base) + (j0) + 2) + w[(j0) + 2]) \
  HS_SHA_ROUND(f, g, h, a, b, c, d, e, sha_k((base) + (j0) + 3) + w[(j0) + 3]) \
  HS_SHA_ROUND(e, f, g, h, a, b, c, d, sha_k((base) + (j0) + 4) + w[(j0) + 4]) \
  HS_SHA_ROUND(d, e, f, g, h, a, b, c, sha_k((base) + (j0) + 5) + w[(j0) + 5]) \
  HS_SHA_ROUND(c, d, e, f, g, h, a, b, sha_k((base) + (j0) + 6) + w[(j0) + 6]) \
  HS_SHA_ROUND(b, c, d, e, f, g, h, a, sha_k((base) + (j0) + 7) + w[(j0) + 7])

HS_HD void sha512_compress(sha512_state &s, uint64_t (&w)[16]) {
  uint64_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
  HS_SHA_8ROUNDS(w, 0, 0)
  HS_SHA_8ROUNDS(w, 0, 8)
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int base = 16; base < 80; base += 16) {
    HS_SHA_SCHED(w, 0) HS_SHA_SCHED(w, 1) HS_SHA_SCHED(w, 2) HS_SHA_SCHED(w, 3)
    HS_SHA_SCHED(w, 4) HS_SHA_SCHED(w, 5) HS_SHA_SCHED(w, 6) HS_SHA_SCHED(w, 7)
    HS_SHA_8ROUNDS(w, base, 0)
    HS_SHA_SCHED(w, 8) HS_SHA_SCHED(w, 9) HS_SHA_SCHED(w, 10) HS_SHA_SCHED(w, 11)
    HS_SHA_SCHED(w, 12) HS_SHA_SCHED(w, 13) HS_SHA_SCHED(w, 14) HS_SHA_SCHED(w, 15)
    HS_SHA_8ROUNDS(w, base, 8)
  }
  s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}

// Compression of a block whose K[t] + W[t] values are already known (80 words).  Used for the padding-only final block of
// messages whose length is a multiple of 128 bytes (e.g. the 512-byte transactions of BASELINE config[1]): that block is
// 0x80, zeros, bit length — its whole message schedule depends on the length alone, so the host expands it once per launch
// (sha512_pad_schedule) and the device runs the 80 rounds without the 64 schedule updates (~45 % of a compression).
struct sha512_kw {
  uint64_t kw[80];
};
HS_HD void sha512_compress_kw(sha512_state &s, const sha512_kw &t) {
  uint64_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int base = 0; base < 80; base += 8) {
    HS_SHA_ROUND(a, b, c, d, e, f, g, h, t.kw[base + 0])
    HS_SHA_ROUND(h, a, b, c, d, e, f, g, t.kw[base + 1])
    HS_SHA_ROUND(g, h, a, b, c, d, e, f, t.kw[base + 2])
    HS_SHA_ROUND(f, g, h, a, b, c, d, e, t.kw[base + 3])
    HS_SHA_ROUND(e, f, g, h, a, b, c, d, t.kw[base + 4])
    HS_SHA_ROUND(d, e, f, g, h, a, b, c, t.kw[base + 5])
    HS_SHA_ROUND(c, d, e, f, g, h, a, b, t.kw[base + 6])
    HS_SHA_ROUND(b, c, d, e, f, g, h, a, t.kw[base + 7])
  }
  s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}
// Same, the K[t] + W[t] words read with a stride (shared-memory table [80][stride] shared by a warp, k_digest32_long).
HS_HD void sha512_compress_kw_strided(sha512_state &s, const uint64_t *kw, int stride) {
  uint64_t a = s.h[0], b = s.h[1], c = s.h[2], d = s.h[3], e = s.h[4], f = s.h[5], g = s.h[6], h = s.h[7];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int base = 0; base < 80; base += 8) {
    const uint64_t *q = kw + (size_t)base * stride;
    HS_SHA_ROUND(a, b, c, d, e, f, g, h, q[0 * stride])
    HS_SHA_ROUND(h, a, b, c, d, e, f, g, q[1 * stride])
    HS_SHA_ROUND(g, h, a, b, c, d, e, f, q[2 * stride])
    HS_SHA_ROUND(f, g, h, a, b, c, d, e, q[3 * stride])
    HS_SHA_ROUND(e, f, g, h, a, b, c, d, q[4 * stride])
    HS_SHA_ROUND(d, e, f, g, h, a, b, c, q[5 * stride])
    HS_SHA_ROUND(c, d, e, f, g, h, a, b, q[6 * stride])
    HS_SHA_ROUND(b, c, d, e, f, g, h, a, q[7 * stride])
  }
  s.h[0] += a; s.h[1] += b; s.h[2] += c; s.h[3] += d; s.h[4] += e; s.h[5] += f; s.h[6] += g; s.h[7] += h;
}
// Expands one block's message schedule and parks K[t] + W[t] at kw[t * stride] (t = 0 .. 79); w[16] is consumed.
HS_HD void sha512_expand_kw(uint64_t *kw, int stride, uint64_t (&w)[16]) {
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int j = 0; j < 16; j++) kw[(size_t)j * stride] = sha_k(j) + w[j];
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (int base = 16; base < 80; base += 16) {
    HS_SHA_SCHED(w, 0) HS_SHA_SCHED(w, 1) HS_SHA_SCHED(w, 2) HS_SHA_SCHED(w, 3)
    HS_SHA_SCHED(w, 4) HS_SHA_SCHED(w, 5) HS_SHA_SCHED(w, 6) HS_SHA_SCHED(w, 7)
    HS_SHA_SCHED(w, 8) HS_SHA_SCHED(w, 9) HS_SHA_SCHED(w, 10) HS_SHA_SCHED(w, 11)
    HS_SHA_SCHED(w, 12) HS_SHA_SCHED(w, 13) HS_SHA_SCHED(w, 14) HS_SHA_SCHED(w, 15)
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < 16; j++) kw[(size_t)(base + j) * stride] = sha_k(base + j) + w[j];
  }
}
// Host side: K[t] + W[t] of the padding-only block that ends a message of `total_len` bytes (total_len % 128 == 0).
inline void sha512_pad_schedule(sha512_kw &t, uint64_t total_len) {
  uint64_t w[80];
  for (int i = 0; i < 16; i++) w[i] = 0;
  w[0] = 0x8000000000000000ULL;
  w[14] = total_len >> 61;
  w[15] = total_len << 3;
  for (int i = 16; i < 80; i++) {
    const uint64_t s0 = rotr64(w[i - 15], 1) ^ rotr64(w[i - 15], 8) ^ (w[i - 15] >> 7);
    const uint64_t s1 = rotr64(w[i - 2], 19) ^ rotr64(w[i - 2], 61) ^ (w[i - 2] >> 6);
    w[i] = w[i - 16] + s0 + w[i - 7] + s1;
  }
  for (int i = 0; i < 80; i++) t.kw[i] = w[i] + HS_SHA512_K_HOST[i];
}

// state -> 64 output bytes as 16 little-endian u32 words (word j = bytes 4j..4j+3 of the digest)
HS_HD void sha512_output_words(const sha512_state &s, uint32_t (&out)[16]) {
  for (int i = 0; i < 8; i++) {
    out[2 * i] = bswap32((uint32_t)(s.h[i] >> 32));
    out[2 * i + 1] = bswap32((uint32_t)s.h[i]);
  }
}

// k-hash fast path: SHA-512(R[32] || A[32] || M[32]) — exactly one block (every message the reference signs is a
// 32-byte Digest: crypto/src/lib.rs:185,200,206).  Inputs are little-endian u32 words as loaded from memory.
HS_HD void sha512_ram32(uint32_t (&out)[16], const uint32_t (&R)[8], const uint32_t (&A)[8], const uint32_t (&M)[8]) {
  uint64_t w[16];
  for (int i = 0; i < 4; i++) {
    w[i] = be64_from_le32(R[2 * i], R[2 * i + 1]);
    w[4 + i] = be64_from_le32(A[2 * i], A[2 * i + 1]);
    w[8 + i] = be64_from_le32(M[2 * i], M[2 * i + 1]);
  }
  w[12] = 0x8000000000000000ULL;
  w[13] = 0;
  w[14] = 0;
  w[15] = 96 * 8;
  sha512_state s;
  sha512_init(s);
  sha512_compress(s, w);
  sha512_output_words(s, out);
}

// Byte-granular reader for arbitrary-length / arbitrarily-aligned messages.
HS_HD uint64_t load_be64_bytes(const uint8_t *p) {
  uint64_t v = 0;
  for (int i = 0; i < 8; i++) v = (v << 8) | p[i];
  return v;
}

// One 64-bit big-endian message word at message offset m (multiple of 8): real bytes, then the 0x80 terminator,
// then zeros.  Keeps the schedule index static so w[] stays in registers.
HS_HD uint64_t sha512_msg_word(const uint8_t *msg, uint64_t len, uint64_t m, bool aligned8) {
  if (m + 8 <= len) {
    if (aligned8) {
      uint64_t le = *reinterpret_cast<const uint64_t *>(msg + m);
      return ((uint64_t)bswap32((uint32_t)le) << 32) | bswap32((uint32_t)(le >> 32));
    }
    return load_be64_bytes(msg + m);
  }
  if (m > len) return 0;
  uint64_t v = 0;
  int nb = (int)(len - m);
  for (int i = 0; i < nb; i++) v |= (uint64_t)msg[m + i] << (56 - 8 * i);
  return v | ((uint64_t)0x80 << (56 - 8 * nb));
}

// Absorbs blocks [b0, b1) of prefix || msg || padding into s.  The prefix is n_prefix_words (0 or 8) big-endian 64-bit
// words already in registers (R||A for the k-hash; none for Digest); message bytes stream from global memory.
HS_HD void sha512_absorb_blocks(sha512_state &s, const uint64_t (&prefix_words)[8], int n_prefix_words, const uint8_t *msg, uint64_t len,
                                uint64_t b0, uint64_t b1) {
  const uint64_t P = (uint64_t)n_prefix_words * 8;
  const uint64_t total = P + len;
  const uint64_t nblk = (total + 17 + 127) / 128;
  const bool aligned8 = ((reinterpret_cast<uintptr_t>(msg) & 7u) == 0);
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
  for (uint64_t b = b0; b < b1; b++) {
    uint64_t w[16];
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int j = 0; j < 16; j++) {
      uint64_t o = b * 128 + 8 * (uint64_t)j;
      uint64_t v;
      if (o < P) v = prefix_words[j & 7];  // only reachable for b == 0, j < 8
      else v = sha512_msg_word(msg, len, o - P, aligned8);
      if (b == nblk - 1 && j == 14) v = total >> 61;
      if (b == nblk - 1 && j == 15) v = total << 3;
      w[j] = v;
    }
    sha512_compress(s, w);
  }
}
HS_HD uint64_t sha512_nblocks(uint64_t total_len) { return (total_len + 17 + 127) / 128; }
// General hash of prefix || msg[0..len).
HS_HD void sha512_prefix_msg(uint32_t (&out)[16], const uint64_t (&prefix_words)[8], int n_prefix_words, const uint8_t *msg,
                             uint64_t len) {
  sha512_state s;
  sha512_init(s);
  sha512_absorb_blocks(s, prefix_words, n_prefix_words, msg, len, 0, sha512_nblocks((uint64_t)n_prefix_words * 8 + len));
  sha512_output_words(s, out);
}
// The 16 message words of block b of msg[0..len) || padding (no prefix).
HS_HD void sha512_block_words(uint64_t (&w)[16], const uint8_t *msg, uint64_t len, uint64_t b) {
  const uint64_t nblk = (len + 17 + 127) / 128;
  const bool aligned8 = ((reinterpret_cast<uintptr_t>(msg) & 7u) == 0);
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int j = 0; j < 16; j++) {
    uint64_t v = sha512_msg_word(msg, len, b * 128 + 8 * (uint64_t)j, aligned8);
    if (b == nblk - 1 && j == 14) v = len >> 61;
    if (b == nblk - 1 && j == 15) v = len << 3;
    w[j] = v;
  }
}
