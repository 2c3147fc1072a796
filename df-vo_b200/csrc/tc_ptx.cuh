// wgmma / TMA / mbarrier PTX wrappers, the fused conv epilogue and the MMA consumer shared by the tensor-core convolution
// kernels (conv_tc.cu: per-tap operand loads, stride 1|2;  conv_halo.cu / conv_chain.cu: halo-resident operand, stride 1).
#pragma once
#include "ops.h"
#ifndef DFVO_HOSTSIM
#include "wgmma.cuh"
#endif

namespace dfvo {

// what the epilogue needs to turn accumulator columns of one output pixel into stored channels
struct TcEpi {
  int Cout, zero_pad_to, act, out_f32;
  int round_tf32;          // fp32 output rounded to the tf32 grid (tf32 mode activations)
  int vec16;               // output and residual base and pixel strides are 16-byte aligned: whole 8-channel runs per store
  void* out;
  const void* res;
};

#ifndef DFVO_HOSTSIM
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"((uint64_t)tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"((uint64_t)tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"((uint64_t)tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// ---- wgmma (warpgroup MMA) ordering: fence before the first MMA that touches accumulator registers the warpgroup has read or
// written since its last MMA; commit closes a group of issued MMAs; wait<N> returns once at most N groups are still in flight
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// K-major, 128-byte-swizzle shared-memory matrix descriptor (sm_90 GMMA layout): start>>4 [0,14) | LBO>>4 [16,30) (unused for
// swizzled K-major, 1) | SBO>>4 [32,46) = distance of consecutive 8-row groups | base offset [49,52) = 0 | SWIZZLE_128B (1) [62,64).
// The swizzle XOR is a function of the absolute shared-memory address and the pattern starts at the 1024-B aligned stage base
// (base offset 0), so a start shifted by whole 128-B rows or by 32 B inside a row addresses exactly the bytes TMA wrote there.
__device__ __forceinline__ uint64_t desc_sw128(uint32_t saddr, uint32_t sbo_bytes) {
  const uint32_t lo = ((saddr >> 4) & 0x3FFFu) | (1u << 16);
  const uint32_t hi = ((sbo_bytes >> 4) & 0x3FFFu) | (1u << 30);
  return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ float tc_round_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}
// Programmatic dependent launch (PDL): a kernel launched with cudaLaunchAttributeProgrammaticStreamSerialization may start
// while its predecessor in the stream is still running; it must not touch data the predecessor produces (or overwrite
// data it reads) before pdl_wait(), which returns once the predecessor grid has completed and flushed.  pdl_trigger()
// lets the *next* kernel of the stream start its own prologue early.  The convolution kernels run their prologue
// (barrier init, tensor-map prefetch: nothing a predecessor writes) before the wait.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void prefetch_tmap(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)tmap) : "memory");
}
// one elected lane of a fully active warp (cute::elect_one_sync): ptxas keeps TMA issues under this
// predicate on the uniform datapath without the per-instruction ELECT loop it emits under `if (lane == 0)`
__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .b32 rx;\n\t.reg .pred px;\n\t"
      "elect.sync rx|px, 0xffffffff;\n\t"
      "@px mov.s32 %0, 1;\n\t}"
      : "+r"(pred));
  return pred != 0;
}
}  // namespace tc

// bias + optional residual + activation + store of the two adjacent output channels (c, c + 1) of one pixel (c even): the pair a
// thread holds in the wgmma accumulator fragment.  opix / rpix = element offsets of the pixel; channels in [Cout, zero_pad_to) are
// written as zeros, channels from zero_pad_to on are not written.
__device__ __forceinline__ void tc_store2(const TcEpi& p, const float* bias, float a, float b, int c, long long opix, long long rpix) {
  if (c >= p.zero_pad_to) return;
  const bool two = c + 1 < p.zero_pad_to;
  float v[2] = {a, b};
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (c + j < p.Cout) {
      float x = v[j] + bias[c + j];
      if (p.res) x += p.out_f32 ? reinterpret_cast<const float*>(p.res)[rpix + c + j]
                                : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.res)[rpix + c + j]);
      v[j] = apply_act(x, p.act);
    } else {
      v[j] = 0.f;
    }
  }
  if (p.out_f32) {
    if (p.round_tf32) { v[0] = tc::tc_round_tf32(v[0]); v[1] = tc::tc_round_tf32(v[1]); }
    float* o = reinterpret_cast<float*>(p.out) + opix + c;
    if (two && (reinterpret_cast<uintptr_t>(o) & 7u) == 0) {
      *reinterpret_cast<float2*>(o) = make_float2(v[0], v[1]);
    } else {
      o[0] = v[0];
      if (two) o[1] = v[1];
    }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + opix + c;
    if (two && (reinterpret_cast<uintptr_t>(o) & 3u) == 0) {
      *reinterpret_cast<__nv_bfloat162*>(o) = __floats2bfloat162_rn(v[0], v[1]);
    } else {
      o[0] = __float2bfloat16_rn(v[0]);
      if (two) o[1] = __float2bfloat16_rn(v[1]);
    }
  }
}

// 4 x 4 transpose of accumulator pairs across the quad of lanes that holds one fragment row pair: on entry lane q's v[2 r + e] is
// its pair slot r; on exit lane q's v[2 r + e] is what lane r held in slot q.  Two butterfly stages, each swapping one bit of the
// lane index with the same bit of the slot index, with every register index a compile-time constant.  All 32 lanes must take part.
__device__ __forceinline__ void tc_quad_transpose(float (&v)[8], int q) {
#pragma unroll
  for (int b = 0; b < 2; ++b) {
    const bool bq = (q >> b) & 1;
#pragma unroll
    for (int lo = 0; lo < 4; ++lo) {
      if (lo & (1 << b)) continue;
      const int hi = lo | (1 << b);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float r = __shfl_xor_sync(0xffffffffu, bq ? v[2 * lo + e] : v[2 * hi + e], 1 << b);
        if (bq) v[2 * lo + e] = r; else v[2 * hi + e] = r;
      }
    }
  }
}

// bias + optional residual + activation ACT + store of the 8 consecutive output channels c .. c + 7 of one pixel, all < Cout, with
// 16-byte loads and stores (the caller checked TcEpi::vec16; c is a multiple of 8).  Per element the same arithmetic as tc_store2.
template <int ACT>
__device__ __forceinline__ void tc_store8(const TcEpi& p, const float* bias, float (&v)[8], int c, long long opix, long long rpix) {
  uint4 rb16 = make_uint4(0u, 0u, 0u, 0u);
  if (p.res && !p.out_f32) rb16 = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + rpix + c);
#pragma unroll
  for (int k = 0; k < 2; ++k) {               // channels c + 4 k .. + 3: the fp32 residual in two 16-byte loads
    float r[4];
    if (p.res) {
      if (p.out_f32) {
        const float4 r4 = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + rpix + c)[k];
        r[0] = r4.x; r[1] = r4.y; r[2] = r4.z; r[3] = r4.w;
      } else {
        const uint32_t w0 = k ? rb16.z : rb16.x, w1 = k ? rb16.w : rb16.y;
        const __nv_bfloat162 b0 = *reinterpret_cast<const __nv_bfloat162*>(&w0), b1 = *reinterpret_cast<const __nv_bfloat162*>(&w1);
        r[0] = __low2float(b0); r[1] = __high2float(b0); r[2] = __low2float(b1); r[3] = __high2float(b1);
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float x = v[4 * k + e] + bias[c + 4 * k + e];
      if (p.res) x += r[e];
      v[4 * k + e] = apply_act(x, ACT);
    }
  }
  if (p.out_f32) {
    if (p.round_tf32) {
#pragma unroll
      for (int e = 0; e < 8; ++e) v[e] = tc::tc_round_tf32(v[e]);
    }
    float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + opix + c);
    o[0] = make_float4(v[0], v[1], v[2], v[3]);
    o[1] = make_float4(v[4], v[5], v[6], v[7]);
  } else {
    uint32_t w[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const __nv_bfloat162 b2 = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
      w[k] = *reinterpret_cast<const uint32_t*>(&b2);
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + opix + c) = make_uint4(w[0], w[1], w[2], w[3]);
  }
}

// One wgmma accumulator fragment row pair (M rows r and r + 8 of a warp: pair slot 2 j + h = acc[4 j + 2 h], acc[4 j + 2 h + 1]
// = row r + 8 h, channels 8 j + 2 (lane % 4) + {0, 1}) through tc_quad_transpose in groups of four pair slots: afterwards lane q
// of a quad holds row r + 8 (q & 1), channels 8 (2 g + (q >> 1)) .. + 7 of group g, stored with tc_store8.  A warp store then
// covers 16 rows x 32 contiguous bytes (bf16) instead of 8 rows x 4 B per 32-byte sector.  The warp takes this path as a whole
// (all rows inside the image, all BN channels < Cout, vec16); pix(h) is the element offset of the lane's pixel in row r + 8 h.
// The activation is a template parameter here: apply_act's run-time switch costs an indirect branch per element.
template <int BN, int ACT, typename Pix>
__device__ __forceinline__ void tc_store_frag16_act(const TcEpi& p, const float* bias, const float (&acc)[BN / 2], int cbase, int lane,
                                                    Pix pix) {
  const int q = lane & 3, h = q & 1;
  long long opix, rpix;
  pix(h, &opix, &rpix);
#pragma unroll
  for (int g = 0; g < BN / 16; ++g) {
    float v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = acc[8 * g + k];
    tc_quad_transpose(v, q);
    tc_store8<ACT>(p, bias, v, cbase + 8 * (2 * g + (q >> 1)), opix, rpix);
  }
}
template <int BN, typename Pix>
__device__ __forceinline__ void tc_store_frag16(const TcEpi& p, const float* bias, const float (&acc)[BN / 2], int cbase, int lane, Pix pix) {
  switch (p.act) {
    case ACT_LEAKY: tc_store_frag16_act<BN, ACT_LEAKY>(p, bias, acc, cbase, lane, pix); break;
    case ACT_RELU: tc_store_frag16_act<BN, ACT_RELU>(p, bias, acc, cbase, lane, pix); break;
    case ACT_ELU: tc_store_frag16_act<BN, ACT_ELU>(p, bias, acc, cbase, lane, pix); break;
    case ACT_SIGMOID: tc_store_frag16_act<BN, ACT_SIGMOID>(p, bias, acc, cbase, lane, pix); break;
    default: tc_store_frag16_act<BN, ACT_NONE>(p, bias, acc, cbase, lane, pix); break;
  }
}
// An mbarrier-guarded ring of shared-memory slots as one side walks it: slot i, its full / empty barriers, the phase bit.
struct TcRing {
  uint32_t base, slot_bytes, full0, empty0;
  int n, i;
  uint32_t ph;
  __device__ __forceinline__ uint32_t slot() const { return base + (uint32_t)i * slot_bytes; }
  __device__ __forceinline__ uint32_t full() const { return full0 + 8u * (uint32_t)i; }
  __device__ __forceinline__ uint32_t empty() const { return empty0 + 8u * (uint32_t)i; }
  __device__ __forceinline__ void next() { if (++i == n) { i = 0; ph ^= 1u; } }
};

// Development aid (scripts/halo_phases.py): compiled with DFVO_HALO_STAMPS, the leader thread of each consumer warpgroup of
// k_conv_halo records per-tile phase clocks (clock64, SM-local) into tc::g_halo_stamps; without it these macros compile to nothing
// and the product kernels are unchanged.  Row HALO_STAMP_TILES of a (CTA, warpgroup) is the tile in progress; DFVO_HALO_STAMP_TILE
// copies it to the row of the CTA's it-th tile.  Slots: 0 tile start, 1 first A slot full, 2 sum of A-full waits, 3 sum of
// B-full waits, 4 last MMA retired, 5 epilogue stored.
#ifdef DFVO_HALO_STAMPS
#define HALO_STAMP_CTAS 288
#define HALO_STAMP_TILES 128
#define HALO_STAMP_N 6
namespace tc {
static __device__ unsigned long long g_halo_stamps[HALO_STAMP_CTAS][2][HALO_STAMP_TILES + 1][HALO_STAMP_N];
__device__ __forceinline__ unsigned long long* halo_stamp_row(int row) {
  return g_halo_stamps[blockIdx.x % HALO_STAMP_CTAS][(threadIdx.x >> 7) & 1][row];
}
}  // namespace tc
#define DFVO_HALO_STAMP(k) \
  do { if ((threadIdx.x & 127) == 0) tc::halo_stamp_row(HALO_STAMP_TILES)[k] = clock64(); } while (0)
#define DFVO_HALO_TIMED(k, stmt)                                                                                  \
  do {                                                                                                            \
    const long long t0_ = clock64();                                                                              \
    stmt;                                                                                                         \
    if ((threadIdx.x & 127) == 0) tc::halo_stamp_row(HALO_STAMP_TILES)[k] += clock64() - t0_;                     \
  } while (0)
#define DFVO_HALO_STAMP_TILE(it)                                                                                  \
  do {                                                                                                            \
    if ((threadIdx.x & 127) == 0) {                                                                               \
      unsigned long long* cur_ = tc::halo_stamp_row(HALO_STAMP_TILES);                                            \
      if ((it) < HALO_STAMP_TILES)                                                                                \
        for (int k_ = 0; k_ < HALO_STAMP_N; ++k_) tc::halo_stamp_row(it)[k_] = cur_[k_];                          \
      cur_[2] = cur_[3] = 0;                                                                                      \
    }                                                                                                             \
  } while (0)
#else
#define DFVO_HALO_STAMP(k) do {} while (0)
#define DFVO_HALO_TIMED(k, stmt) do { stmt; } while (0)
#define DFVO_HALO_STAMP_TILE(it) do {} while (0)
#endif

// the MMAs of one tap: S sub-tiles (+8 pixels = +1024 B each) x NKS K steps (+32 B inside the 128-B swizzle atom)
template <int S, int BN, int TF32, int NKS>
__device__ __forceinline__ void halo_tap_mma(float (&acc)[S][BN / 2], uint32_t at, uint32_t bt, uint32_t a_sbo, uint32_t fresh) {
  using namespace tc;
#pragma unroll
  for (int sub = 0; sub < S; ++sub)
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks)
      Wgmma<BN, TF32>::mma(acc[sub], desc_sw128(at + (uint32_t)sub * 1024u + 32u * ks, a_sbo), desc_sw128(bt + 32u * ks, 1024u),
                           ks == 0 ? fresh : 1u);
}

// The taps of one (source, channel chunk) of a halo tile, NKS K steps each.  NKS is a template parameter and every tap's
// fence -> MMAs -> commit -> wait<1> is one basic block: a run-time branch between the fence and the commit makes ptxas close a
// wgmma group inside each branch and insert an empty one at the commit (C7519 "warpgroup.arrive is injected"), so wait<1>
// would keep only that empty group in flight and the tensor pipe would drain after every tap.  The chunk does not drain at its
// end either: its last tap's group stays in flight into the next chunk.  pend_b = empty barrier of the B slot whose group may
// still be in flight (0: none); the previous chunk's A slot (ring slot before ra.i) is released after this chunk's first
// wait<1> unless this is the tile's first chunk (fresh == 0); the tile's last slots after its final wait<0> (halo_tile_mma).
template <int S, int BN, int TF32, int NKS>
__device__ __forceinline__ void halo_chunk_mma(float (&acc)[S][BN / 2], const TcRing& ra, TcRing& rb, uint32_t a0, uint32_t a_sbo, int kh,
                                               int kw, int HW, uint32_t& fresh, uint32_t& pend_b, bool leader) {
  using namespace tc;
  const bool prev_a = fresh != 0u;
  for (int ky = 0; ky < kh; ++ky) {
    for (int kx = 0; kx < kw; ++kx) {
      DFVO_HALO_TIMED(3, mbar_wait(rb.full(), rb.ph));
      wgmma_fence();
      halo_tap_mma<S, BN, TF32, NKS>(acc, a0 + (uint32_t)(ky * HW + kx) * 128u, rb.slot(), a_sbo, fresh);
      wgmma_commit();
      wgmma_wait<1>();
      if (leader) {
        if (pend_b) mbar_arrive(pend_b);
        if (prev_a && ky == 0 && kx == 0) mbar_arrive(ra.empty0 + 8u * (uint32_t)(ra.i ? ra.i - 1 : ra.n - 1));
      }
      pend_b = rb.empty();
      rb.next();
      fresh = 1u;
    }
  }
}

// MMA main loop of one tile of the halo-resident kernels (conv_halo.cu, conv_chain.cu) for one consumer warpgroup: wg 0 / 1 owns
// pixel rows 0-7 / 8-15 of every 8 x 16 sub-tile (M = 64 each).  Per (source, channel chunk) one A slot holds the HW x HH pixel
// halo (128 B per pixel, SWIZZLE_128B); tap (ky, kx) reads it through a descriptor whose start is shifted by (ky * HW + kx) pixels
// and whose SBO is one halo row, so the 8-row groups of the K-major operand are the sub-tile's pixel rows.  One B slot per tap
// (BN x 128 B of weights) is shared by the S sub-tiles and released once the MMAs of the next tap are issued and its own have
// completed; an A slot likewise once the first tap of the next chunk is issued and its own last tap has completed, so the tensor
// pipe drains only before the epilogue.  Holding the previous chunk's A slot until then cannot stall the A producer with two A
// slots: the next chunk's slot was released when this chunk's first group retired, so the producer fills it while this chunk
// runs, and this chunk's slot is released (at the latest by the final wait<0>) before the consumer waits on any later A slot.
// `leader` = one thread of the warpgroup (the empty barriers count one arrival per consumer warpgroup).
template <int S, int BN, int TF32>
__device__ __forceinline__ void halo_tile_mma(float (&acc)[S][BN / 2], TcRing& ra, TcRing& rb, int nsrc, const int* srcC, int chunk,
                                              int esize, int kh, int kw, int HW, int wg, bool leader) {
  using namespace tc;
  const uint32_t a_sbo = (uint32_t)HW * 128u;
  uint32_t fresh = 0;                         // 0 for the first (chunk, tap) of the tile: its ks = 0 MMAs overwrite
  uint32_t pend_b = 0u;
  for (int s = 0; s < nsrc; ++s) {
    for (int c0 = 0; c0 < srcC[s]; c0 += chunk) {
      const int rem = srcC[s] - c0;
      const int nks = ((rem >= chunk ? chunk : rem) * esize) >> 5;        // 32-byte K steps (16 bf16 / 8 tf32) with real channels
      DFVO_HALO_TIMED(2, mbar_wait(ra.full(), ra.ph));
      if (s == 0 && c0 == 0) DFVO_HALO_STAMP(1);
      const uint32_t a0 = ra.slot() + (uint32_t)wg * 8u * a_sbo;
      switch (nks) {                                                       // compile-time K steps: no wgmma in a run-time loop
        case 4: halo_chunk_mma<S, BN, TF32, 4>(acc, ra, rb, a0, a_sbo, kh, kw, HW, fresh, pend_b, leader); break;
        case 3: halo_chunk_mma<S, BN, TF32, 3>(acc, ra, rb, a0, a_sbo, kh, kw, HW, fresh, pend_b, leader); break;
        case 2: halo_chunk_mma<S, BN, TF32, 2>(acc, ra, rb, a0, a_sbo, kh, kw, HW, fresh, pend_b, leader); break;
        default: halo_chunk_mma<S, BN, TF32, 1>(acc, ra, rb, a0, a_sbo, kh, kw, HW, fresh, pend_b, leader); break;
      }
      ra.next();
    }
  }
  wgmma_wait<0>();
  DFVO_HALO_STAMP(4);
  if (leader) {
    mbar_arrive(pend_b);
    mbar_arrive(ra.empty0 + 8u * (uint32_t)(ra.i ? ra.i - 1 : ra.n - 1));
  }
}

// Epilogue of one halo tile for one consumer warpgroup: the thread's accumulator pairs are pixels (x0 + 8 sub + lane / 4,
// y0 + 8 wg + 2 warp + h), channels cbase + 8 j + 2 (lane % 4) + {0, 1}.  A sub-tile whose two pixel rows of this warp lie inside
// the image, with all BN channels real and 16-byte aligned output / residual (TcEpi::vec16), is stored in 8-channel runs
// (tc_store_frag16); anything else pair by pair (tc_store2).  The condition is uniform across the warp.
template <int S, int BN>
__device__ __forceinline__ void halo_tile_store(const float (&acc)[S][BN / 2], const TcEpi& ep, const float* bias_s, int cbase, int n,
                                                int x0, int y0, int W, int H, long long oN, long long oH, long long oW, long long rN,
                                                long long rH, long long rW, int wg, int warp_in_wg, int lane) {
  const int yw = y0 + 8 * wg + 2 * warp_in_wg;
  const bool vec = ep.vec16 && cbase + BN <= ep.Cout && yw + 1 < H;
#pragma unroll
  for (int sub = 0; sub < S; ++sub) {
    const int x = x0 + 8 * sub + (lane >> 2);
    if (vec && x0 + 8 * sub + 8 <= W) {
      tc_store_frag16<BN>(ep, bias_s, acc[sub], cbase, lane, [&](int h, long long* opix, long long* rpix) {
        *opix = n * oN + (yw + h) * oH + x * oW; *rpix = n * rN + (yw + h) * rH + x * rW;
      });
      continue;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int y = yw + h;
      if (y >= H || x >= W) continue;
      const long long opix = n * oN + y * oH + x * oW, rpix = n * rN + y * rH + x * rW;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        tc_store2(ep, bias_s, acc[sub][4 * j + 2 * h], acc[sub][4 * j + 2 * h + 1], cbase + 8 * j + 2 * (lane & 3), opix, rpix);
    }
  }
}

#endif  // !DFVO_HOSTSIM

// internal: the halo-resident kernel (conv_halo.cu); conv_tc() dispatches to it for stride-1 rectangular tap sets
int conv_halo(const ConvTc& c, cudaStream_t s);
bool conv_halo_supported(const ConvTc& c);
// per-launch CUDA-event timing shared by both kernels (bench.py roofline; DFVO_TC_TRACE=1 prints every launch)
struct TcProf { cudaEvent_t e0, e1; };
bool tc_prof_begin(cudaStream_t s, TcProf* p);                       // false (and no events) when profiling is off
void tc_prof_end(cudaStream_t s, const TcProf& p, double flops, const char* desc);
int tc_encode_map(void* map, const void* ptr, int rank, const unsigned long long* dims, const unsigned long long* strides_bytes,
                  const unsigned* box, int esize = 2, int swizzle_bytes = 128);   // bf16 (esize 2) or fp32 (4); swizzle 128 / 64 / 32 B; zero OOB fill
int tc_num_sms();
bool tc_epi_vec16(const ConvTc& c);                                  // TcEpi::vec16 of a layer: 16-byte aligned output / residual
// launch config with the PDL attribute set unless DFVO_PDL=0 (attr must outlive the cudaLaunchKernelEx call)
#ifndef DFVO_HOSTSIM
void tc_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int grid, int block, size_t smem, cudaStream_t s);
#endif

}  // namespace dfvo
