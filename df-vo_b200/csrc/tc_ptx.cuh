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

// MMA main loop of one tile of the halo-resident kernels (conv_halo.cu, conv_chain.cu) for one consumer warpgroup: wg 0 / 1 owns
// pixel rows 0-7 / 8-15 of every 8 x 16 sub-tile (M = 64 each).  Per (source, channel chunk) one A slot holds the HW x HH pixel
// halo (128 B per pixel, SWIZZLE_128B); tap (ky, kx) reads it through a descriptor whose start is shifted by (ky * HW + kx) pixels
// and whose SBO is one halo row, so the 8-row groups of the K-major operand are the sub-tile's pixel rows.  One B slot per tap
// (BN x 128 B of weights) is shared by the S sub-tiles and released once the MMAs of the next tap are issued and its own have
// completed; the A slot is released at the end of its chunk.  `leader` = one thread of the warpgroup (the empty barriers count
// one arrival per consumer warpgroup).
template <int S, int BN, int TF32>
__device__ __forceinline__ void halo_tile_mma(float (&acc)[S][BN / 2], TcRing& ra, TcRing& rb, int nsrc, const int* srcC, int chunk,
                                              int esize, int kh, int kw, int HW, int wg, bool leader) {
  using namespace tc;
  const uint32_t a_sbo = (uint32_t)HW * 128u;
  uint32_t fresh = 0;                         // 0 for the first (chunk, tap) of the tile: its ks = 0 MMAs overwrite
  for (int s = 0; s < nsrc; ++s) {
    for (int c0 = 0; c0 < srcC[s]; c0 += chunk) {
      const int rem = srcC[s] - c0;
      const int nks = ((rem >= chunk ? chunk : rem) * esize) >> 5;        // 32-byte K steps (16 bf16 / 8 tf32) with real channels
      mbar_wait(ra.full(), ra.ph);
      const uint32_t a0 = ra.slot() + (uint32_t)wg * 8u * a_sbo;
      int pend = -1;
      for (int ky = 0; ky < kh; ++ky) {
        for (int kx = 0; kx < kw; ++kx) {
          mbar_wait(rb.full(), rb.ph);
          wgmma_fence();
          const uint32_t at = a0 + (uint32_t)(ky * HW + kx) * 128u, bt = rb.slot();
          switch (nks) {                                                   // compile-time K steps: no wgmma in a run-time loop
            case 4: halo_tap_mma<S, BN, TF32, 4>(acc, at, bt, a_sbo, fresh); break;
            case 3: halo_tap_mma<S, BN, TF32, 3>(acc, at, bt, a_sbo, fresh); break;
            case 2: halo_tap_mma<S, BN, TF32, 2>(acc, at, bt, a_sbo, fresh); break;
            default: halo_tap_mma<S, BN, TF32, 1>(acc, at, bt, a_sbo, fresh); break;
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (pend >= 0 && leader) mbar_arrive(rb.empty0 + 8u * (uint32_t)pend);
          pend = rb.i;
          rb.next();
          fresh = 1u;
        }
      }
      wgmma_wait<0>();
      if (leader) { mbar_arrive(rb.empty0 + 8u * (uint32_t)pend); mbar_arrive(ra.empty()); }
      ra.next();
    }
  }
}

// Epilogue of one halo tile for one consumer warpgroup: the thread's accumulator pairs are pixels (x0 + 8 sub + lane / 4,
// y0 + 8 wg + 2 warp + h), channels cbase + 8 j + 2 (lane % 4) + {0, 1}.
template <int S, int BN>
__device__ __forceinline__ void halo_tile_store(const float (&acc)[S][BN / 2], const TcEpi& ep, const float* bias_s, int cbase, int n,
                                                int x0, int y0, int W, int H, long long oN, long long oH, long long oW, long long rN,
                                                long long rH, long long rW, int wg, int warp_in_wg, int lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int y = y0 + 8 * wg + 2 * warp_in_wg + h;
    if (y >= H) continue;
#pragma unroll
    for (int sub = 0; sub < S; ++sub) {
      const int x = x0 + 8 * sub + (lane >> 2);
      if (x >= W) continue;
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
// launch config with the PDL attribute set unless DFVO_PDL=0 (attr must outlive the cudaLaunchKernelEx call)
#ifndef DFVO_HOSTSIM
void tc_launch_config(cudaLaunchConfig_t* cfg, cudaLaunchAttribute* attr, int grid, int block, size_t smem, cudaStream_t s);
#endif

}  // namespace dfvo
