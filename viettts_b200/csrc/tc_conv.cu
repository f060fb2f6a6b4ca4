// Tensor-core NWC conv1d for sm_90a: implicit GEMM on wgmma with fp32 accumulators in registers.
//
// Same operator as conv1d.cu (hk.Conv1D of vietTTS/hifigan/model.py:21-41 with the leaky_relu /
// 3-way-mean / bias / residual fusions), but the contraction runs on the Hopper tensor cores in
// "bf16x3" arithmetic:  every fp32 operand v is split into hi = bf16(v), lo = bf16(v - hi) and the
// product is accumulated in fp32 as  a_hi*w_hi + a_hi*w_lo + a_lo*w_hi  (the dropped a_lo*w_lo
// term and the split truncation are ~2^-17 relative -- see DESIGN.md).
// The generator's fast mode (VTTS_PRECISION_FP16, template flag F16) runs the same kernels with ONE fp16 operand plane:
// v -> fp16_rn(v) saturated to +-65504, one wgmma .f32.f16.f16 per (chunk, tap, 64-row block) instead of three bf16
// ones, fp32 accumulators and the same epilogues (waveform error ~1e-3 L-inf, see DESIGN.md §3).
//
// GEMM view per tap j:  D[time, cout] += A_j[time, cin] * W_j[cin, cout]
//   M = 64 time rows per wgmma (one warpgroup), N = Cout tile (32..256), K = 16 channels.
//   A operand: activations in shared memory, K-major, NO swizzle, rows 16 B apart:
//       [plane hi|lo][k-half (8 ch)][row][8 x bf16]     (fp16: plane 0 only)
//     so tap j / dilation d is just a start-address offset of j*d*16 bytes in the descriptor (no im2col).
//   B operand: weights pre-split and pre-packed at load time into the same canonical layout,
//     streamed with cp.async.bulk (TMA bulk copy) through an mbarrier ring, one tap per stage
//     (fp16: one plane, half the bytes per stage; the stage keeps its bf16 size).
//
// One persistent CTA per SM, 12 warps:
//   warps 0-7  two consumer warpgroups: each owns MW x 64 rows of the tile, issues the wgmmas of its rows and runs the
//              epilogue (+ bias (+ BN/act) (+ residual), fp32 NWC store; the plain one staged through shared memory)
//   warp  8    weight producer (one lane, cp.async.bulk + expect_tx)
//   warps 9-11 activation converters: fp32 global -> [mean3] -> leaky_relu -> hi/lo bf16 -> smem
// The ConvTranspose instantiation (SUB) walks a tile in row steps of NCWG x 64 rows instead: its ring stages hold a row
// step over several chunks (the row-block ring, SUB_* below), so each input row is read once per tile.
// A consumer keeps one wgmma group in flight: it releases a ring stage when the NEXT group has been issued and the
// previous one has retired (wgmma.wait_group 1), so issue and tensor-core execution overlap.
//
// The fused ResBlock pair (tc_pair_kernel, C = N <= 64) is the same machinery twice per tile:
//   conv1 (dilated) over R rows of the intermediate -> + b1, lrelu, zero outside [0, len) -> hi/lo split into a
//   shared-memory operand that never leaves the SM -> conv2 (dilation 1) -> + b2 + x.  Tiles overlap by
//   PAIR_OVERLAP rows so that conv2's halo comes from the tile's own intermediate.
#include <cuda_bf16.h>

#include <algorithm>

#include "tc_common.cuh"
#include "vtts_internal.cuh"

namespace {

using namespace tcx;

constexpr int NCWG = 2;                       // consumer warpgroups
constexpr int NCONS = NCWG * 128;             // consumer threads (warps 0-7)
constexpr int PROD_WARP = NCONS / 32;         // weight producer warp (8)
constexpr int NCONV = 96;                     // converter threads (warps 9-11)
constexpr int NTHREADS = NCONS + 32 + NCONV;  // 384
constexpr int NA = 4;                         // activation stages
constexpr int HALO = 64;                      // staged rows beyond the tile: dilation * (k - 1) <= 64
constexpr int PAIR_OVERLAP = 16;              // pair kernel: rows per tile that only feed conv2's halo (k - 1 <= 16)
constexpr int NQ = 2;                         // tile-id ring slots
constexpr int NREADERS = (NCONS + NCONV) / 32;  // warps that read the tile-id ring

// Row-block ring of the sub-row (ConvTranspose) instantiation.  Its input is the 3-way mean of three chain tensors, so a
// tile's live input is three times that of a ResBlock conv; converted chunk by chunk, every row of it would be revisited
// Cin/16 times and fall out of L2 in between.  Instead a ring stage holds one row step of the tile -- NCWG x 64 rows, one
// 64-row block per consumer warpgroup, plus the tap halo -- over SUB_CG 16-channel chunks, so each pass reads contiguous
// SUB_CG x 64 B row segments of x0 (x1, x2) and every input element is read once per tile.  Layout per chunk:
// [plane hi|lo][k-half][SUB_RS rows][16 B], chunks SUB_CSB bytes apart.  SUB_RS = 129 (k-half stride = 4 words mod 32)
// and SUB_CSB = 24 words mod 32 put the 16 float4 columns of a converted row on 32 distinct banks.
constexpr int SUB_CG = 4;                          // chunks per stage (64 channels)
constexpr int SUB_HALO = 1;                        // (k - 1) * dilation of the ConvTranspose's two taps
constexpr int SUB_RS = NCWG * 64 + SUB_HALO;       // rows per stage
constexpr int SUB_CSB = SUB_RS * 64 + 32;          // bytes per chunk
constexpr int SUB_STAGE = SUB_CG * SUB_CSB;
static_assert(SUB_RS * 4 % 32 == 4 && SUB_CSB / 4 % 32 == 24, "bank-conflict-free converter stores");

template <int N, int MW, int PAIRF, bool STAGED = false, bool SUB = false>
struct TcCfg {
  static constexpr int R = 64 * MW * NCWG;                  // rows computed per tile
  static constexpr int R_OUT = R - PAIR_OVERLAP;             // rows stored per tile of the pair kernel
  static constexpr int RA = R + HALO;                       // allocated activation rows per stage
  static constexpr int A_STAGE = RA * 64;                   // bytes: 2 planes x 2 k-halves x RA rows x 16 B
  static constexpr int NAS = SUB ? (N == 64 ? 4 : 2) : NA;  // activation stages (SUB: row-block stages, as many as fit)
  static constexpr int A_BYTES = SUB ? NAS * SUB_STAGE : NA * A_STAGE;
  static constexpr int W_STAGE = N * 64;                    // bytes of one packed (chunk, tap) weight block
  static constexpr int NW = N == 256 ? 4 : 8;               // weight stages
  static constexpr int NCH2 = PAIRF ? N / 16 : 0;           // 16-channel chunks of the on-chip intermediate
  // STAGED: tc_conv_kernel's plain-epilogue staging, per consumer warpgroup: one 64-row block of up to 128 columns
  // (EPI_NC), rows EPI_LD floats apart, then the N bias values.  EPI_LD = 8 (mod 32) words puts the 4 rows x 8 columns
  // of a half-warp's accumulator float2 accesses on 32 distinct banks.
  static constexpr int EPI_NC = N < 128 ? N : 128;
  static constexpr int EPI_LD = EPI_NC + 8;
  static constexpr int EPI_WG = 64 * EPI_LD + N;             // floats
  static constexpr int EPI_STAGE = STAGED ? NCWG * EPI_WG * 4 : 0;   // the register epilogue keeps the L1 it would take
  static constexpr int SMEM_BYTES =
      A_BYTES + NW * W_STAGE + NCH2 * A_STAGE + EPI_STAGE + (2 * NA + 2 * NW + 2 * NQ) * 8 + NQ * 4 + 1024;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory of one CTA");
};

struct Ring {
  uint32_t s = 0, p = 0;
  template <int NS>
  __device__ __forceinline__ void next() { if (++s == NS) { s = 0; p ^= 1; } }
};

// Tiles are handed out at run time.  A tile's cost depends on its problem (k taps, skipped rows past a row's length),
// so a fixed tile -> CTA map leaves SMs idle: with 132 CTAs and 3 problems, tile % 3 == blockIdx.x % 3 and each CTA
// would run one problem only.  The weight-producer lane of each CTA takes tickets from a launch-wide counter and passes
// every ticket on to the CTA's other roles through the NQ-slot tile-id ring (-1 ends the launch).
//
// Ticket order is (batch row, row tile) major, problem minor, with the problems sorted by k, descending: CTAs running at
// the same time work on the same rows, so an input several problems share (the first pair of a ResBlock stage, the
// column groups of a ConvTranspose) is read from DRAM once and served from L2 to the others.
struct Tile {
  int pi, b, tt;   // problem, batch row, row tile
};
__device__ __forceinline__ Tile decode_tile(int t, int nprob, int tiles_per_row) {
  Tile d;
  d.pi = t % nprob; t /= nprob;
  d.tt = t % tiles_per_row;
  d.b = t / tiles_per_row;
  return d;
}

// next ticket, or -1 once the launch's tiles are gone.  Tile blockIdx.x is every CTA's first (grid <= ntiles), so no
// CTA waits for the counter to start; the counter hands out tiles gridDim.x onwards.  The last CTA to run out zeroes
// both counters for the next launch (launches of a context are stream-ordered, and every CTA has taken its last ticket
// by then).
__device__ __forceinline__ int take_ticket(int* sched, int ntiles) {
  const int t = (int)gridDim.x + atomicAdd(&sched[0], 1);
  if (t < ntiles) return t;
  __threadfence();
  if (atomicAdd(&sched[1], 1) == (int)gridDim.x - 1) {
    atomicExch(&sched[0], 0);
    atomicExch(&sched[1], 0);
  }
  return -1;
}

struct TileQueue {
  int* id;
  uint64_t* full;    // producer lane arrives after writing id[s]
  uint64_t* empty;   // lane 0 of every reader warp arrives once it has read id[s]
  Ring r;
  // producer lane: publish ticket t (or -1)
  __device__ __forceinline__ void put(int t, int* err, long long& acc) {
    mbar_wait_t(&empty[r.s], r.p ^ 1, err, 6, acc);
    id[r.s] = t;
    mbar_arrive(&full[r.s]);
    r.next<NQ>();
  }
  // whole reader warp: the next tile id; the slot is released at once, so the ring only bounds how far the producer
  // runs ahead
  __device__ __forceinline__ int get(int* err, long long& acc) {
    int t = 0;
    if ((threadIdx.x & 31) == 0) {
      mbar_wait_t(&full[r.s], r.p, err, 6, acc);
      t = id[r.s];
      mbar_arrive(&empty[r.s]);
    }
    r.next<NQ>();
    return __shfl_sync(0xffffffffu, t, 0);
  }
};

// s / 3, rounded to nearest like the IEEE division s / 3.0f, without its branch to a slow path: q0 = s * RN(1/3), then one
// correction by the exact residual s - 3 q0 (Markstein).  Bit-equal to s / 3.0f for every float except +-0 and +-inf,
// where it would give +0 and NaN; for those s / 3 is s itself (scripts/check_div3.c checks all 2^32 inputs).
__device__ __forceinline__ float div3_rn(float s) {
  constexpr float y = 0x1.555556p-2f;   // RN(1/3)
  const float q0 = __fmul_rn(s, y);
  const float q1 = __fmaf_rn(__fmaf_rn(-q0, 3.0f, s), y, q0);
  return (s == 0.f || fabsf(s) == __int_as_float(0x7f800000)) ? s : q1;
}

// converters: fill A stage `stage` with rows [row_base, row_base + rows) of channels [ch0, ch0 + 4 * QN) of
// x0 (+x1+x2)/3, leaky_relu'd (pre_mode >= 1), zero outside [lo, valid); bf16 hi/lo planes, or one saturated fp16 plane
// (F16).  The stage holds QN / 4 chunks of [plane][k-half][RS rows][16 B], CSB bytes apart; thread ct converts float4
// column ct % QN of every (NCONV / QN)-th row.
// LOADS_FIRST: all 3 x U loads of a step are issued before the first mean, and the mean divides with div3_rn.  The IEEE
// division by 3 branches to a slow path; the compiler does not hoist later loads above that branch (in source order, row
// u + 1's loads would wait for row u's data, one memory round trip per row), and the 4 U branches serialize the step's
// arithmetic.
template <int QN, int RS, int CSB, bool F16, bool LOADS_FIRST = false>
__device__ __forceinline__ void convert_rows(uint8_t* stage, int ct, const float* x0, const float* x1, const float* x2, int ld, int ch0,
                                             int row_base, int rows, int lo, int valid, int pre_mode, float slope) {
  static_assert(NCONV % QN == 0, "whole rows per converter step");
  constexpr int RSTEP = NCONV / QN, RA = RS;
  const int q = ct % QN;                    // 4-channel group
  const int r0 = ct / QN;
  uint8_t* st = stage + (q >> 2) * CSB + (((q >> 1) & 1) * RA) * 16 + (q & 1) * 8;
  const int coff = ch0 + q * 4;
  constexpr int U = 8;                      // loads in flight per thread
  for (int rr0 = r0; rr0 < rows; rr0 += RSTEP * U) {
    float4 v[U];
    if constexpr (LOADS_FIRST) {
      float4 a[U], bb[U];
      bool in[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int rr = rr0 + u * RSTEP;
        const int t = row_base + rr;
        in[u] = rr < rows && t >= lo && t < valid;
        v[u] = a[u] = bb[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (in[u]) {
          const size_t off = (size_t)t * ld + coff;
          v[u] = ldg_pf256(x0 + off);
          if (pre_mode == 2) {
            a[u] = ldg_pf256(x1 + off);
            bb[u] = ldg_pf256(x2 + off);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (in[u] && pre_mode == 2) {
          v[u].x = div3_rn((v[u].x + a[u].x) + bb[u].x);
          v[u].y = div3_rn((v[u].y + a[u].y) + bb[u].y);
          v[u].z = div3_rn((v[u].z + a[u].z) + bb[u].z);
          v[u].w = div3_rn((v[u].w + a[u].w) + bb[u].w);
        }
      }
    } else {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int rr = rr0 + u * RSTEP;
        const int t = row_base + rr;
        v[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rr < rows && t >= lo && t < valid) {
          const size_t off = (size_t)t * ld + coff;
          v[u] = ldg_pf256(x0 + off);
          if (pre_mode == 2) {
            const float4 a = ldg_pf256(x1 + off);
            const float4 bb = ldg_pf256(x2 + off);
            v[u].x = ((v[u].x + a.x) + bb.x) / 3.0f;
            v[u].y = ((v[u].y + a.y) + bb.y) / 3.0f;
            v[u].z = ((v[u].z + a.z) + bb.z) / 3.0f;
            v[u].w = ((v[u].w + a.w) + bb.w) / 3.0f;
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int rr = rr0 + u * RSTEP;
      if (rr < rows) {
        float4 x = v[u];
        if (pre_mode >= 1) {
          x.x = lrelu(x.x, slope); x.y = lrelu(x.y, slope); x.z = lrelu(x.z, slope); x.w = lrelu(x.w, slope);
        }
        if constexpr (F16) {
          *reinterpret_cast<uint2*>(st + (size_t)rr * 16) = f16x4_sat(x);
        } else {
          uint2 hi, lo;
          split4(x, hi, lo);
          *reinterpret_cast<uint2*>(st + (size_t)rr * 16) = hi;
          *reinterpret_cast<uint2*>(st + (size_t)(2 * RA + rr) * 16) = lo;
        }
      }
    }
  }
}

// one 16-channel chunk c over RA-row stages
template <int RA, bool F16>
__device__ __forceinline__ void convert_chunk(uint8_t* stage, int ct, const float* x0, const float* x1, const float* x2, int ld, int c,
                                              int row_base, int rows, int lo, int valid, int pre_mode, float slope) {
  convert_rows<4, RA, 0, F16>(stage, ct, x0, x1, x2, ld, c * 16, row_base, rows, lo, valid, pre_mode, slope);
}

// weight producer: the k packed (chunk, tap) blocks of chunks [0, nch) of one conv, one ring stage each
// (a block is N * 64 bytes of bf16 hi/lo, or N * 32 bytes of fp16)
template <int N, int NW, bool F16>
__device__ __forceinline__ void produce_weights(uint8_t* w_st, uint64_t* w_full, uint64_t* w_empty, Ring& rw, const void* wpk, int nch,
                                                int k, int* err, long long& wait_acc) {
  constexpr int WB = F16 ? N * 32 : N * 64;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(wpk);
  for (int i = 0; i < nch * k; ++i) {
    mbar_wait_t(&w_empty[rw.s], rw.p ^ 1, err, 4, wait_acc);
    mbar_expect_tx(&w_full[rw.s], WB);
    bulk_g2s(w_st + rw.s * (N * 64), src + (size_t)i * WB, WB, &w_full[rw.s]);
    rw.next<NW>();
  }
}

// consumer warpgroup: acc[mt] (+)= sum over chunks c < nch and taps j < k of A(rows (wg*MW + mt)*64 + j*dil) . W(c, j).
// A_FROM_RING: the A operand of chunk c is the next stage of the activation ring (released after its last tap);
// otherwise it is chunk c of the fixed buffer at a_st_u32 (the pair kernel's intermediate).
// A_REGS (fixed buffer only): the A fragments are loaded into registers with ldmatrix and the wgmmas take A from
// registers, so the tensor core fetches only B from shared memory; each group then retires before the next one loads.
// F16: one fp16 product per (chunk, tap, 64-row block); the weight block is [k-half][n][8], so its k-halves are N rows
// apart.
template <int N, int MW, int RA, int NW, bool A_FROM_RING, bool A_REGS, bool F16>
__device__ __forceinline__ void consume(float (&acc)[MW][N / 2], int wg, uint32_t a_st_u32, uint64_t* a_full, uint64_t* a_empty, Ring& ra,
                                        uint32_t w_st_u32, uint64_t* w_full, uint64_t* w_empty, Ring& rw, int nch, int k, int dil,
                                        int* err, long long& w_a, long long& w_w) {
  const uint64_t a_tmpl = make_desc(0, RA * 16, 128);
  const uint64_t b_tmpl = make_desc(0, (F16 ? 1 : 2) * N * 16, 128);   // k-half blocks are 2N rows apart ([hi rows | lo rows]) or N (fp16)
  const bool lane0 = (threadIdx.x & 31) == 0;
  int pend_w = -1, pend_a = -1;
  for (int c = 0; c < nch; ++c) {
    uint32_t a_base;
    if constexpr (A_FROM_RING) {
      mbar_wait_t(&a_full[ra.s], ra.p, err, 2, w_a);
      a_base = a_st_u32 + ra.s * (RA * 64);
    } else {
      a_base = a_st_u32 + c * (RA * 64);
    }
    for (int j = 0; j < k; ++j) {
      mbar_wait_t(&w_full[rw.s], rw.p, err, 3, w_w);
      const uint32_t w_base = w_st_u32 + rw.s * (N * 64);
      const uint64_t b_hi = b_tmpl | (uint64_t)(w_base >> 4);
      const uint64_t b_lo = b_tmpl | (uint64_t)((w_base + N * 16) >> 4);
      const uint32_t first = (c | j) != 0 ? 1u : 0u;
      if constexpr (A_REGS) {
        static_assert(!A_FROM_RING && !F16, "register A operand: bf16 planes of the fixed buffer");
        const int lane = threadIdx.x & 31, wl = (threadIdx.x >> 5) & 3;
        uint32_t fa_hi[MW][4], fa_lo[MW][4];
#pragma unroll
        for (int mt = 0; mt < MW; ++mt) {
          // ldmatrix matrix q = lane / 8: rows (q & 1) * 8 .. +7 of the warp's 16, k-half q >> 1
          const int row = (wg * MW + mt) * 64 + wl * 16 + ((lane >> 3) & 1) * 8 + (lane & 7) + j * dil;
          const uint32_t addr = a_base + ((lane >> 4) * RA + row) * 16;
          ldmatrix_x4(fa_hi[mt], addr);
          ldmatrix_x4(fa_lo[mt], addr + 2 * RA * 16);
        }
        wgmma_fence();
#pragma unroll
        for (int mt = 0; mt < MW; ++mt) {
          wgmma_rs<N>(acc[mt], fa_hi[mt], b_hi, first);
          wgmma_rs<N>(acc[mt], fa_hi[mt], b_lo, 1u);
          wgmma_rs<N>(acc[mt], fa_lo[mt], b_hi, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();          // the fragments are rewritten by the next tap's loads
        if (lane == 0) mbar_arrive(&w_empty[rw.s]);
        rw.next<NW>();
        continue;
      }
      wgmma_fence();
#pragma unroll
      for (int mt = 0; mt < MW; ++mt) {
        const uint32_t row = a_base + ((wg * MW + mt) * 64 + j * dil) * 16;
        const uint64_t a_hi = a_tmpl | (uint64_t)(row >> 4);
        const uint64_t a_lo = a_tmpl | (uint64_t)((row + 2 * RA * 16) >> 4);
        if constexpr (F16) {
          wgmma<N, true>(acc[mt], a_hi, b_hi, first);
        } else {
          wgmma<N>(acc[mt], a_hi, b_hi, first);
          wgmma<N>(acc[mt], a_hi, b_lo, 1u);
          wgmma<N>(acc[mt], a_lo, b_hi, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();            // the previous group has retired: its stages may be refilled
      if (lane0) {
        if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
        if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
      }
      pend_w = (int)rw.s;
      pend_a = (A_FROM_RING && j == k - 1) ? (int)ra.s : -1;
      rw.next<NW>();
    }
    if constexpr (A_FROM_RING) ra.next<NA>();
  }
  wgmma_wait<0>();
  if (lane0) {
    if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
    if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
  }
}

// consumer warpgroup, row-block ring (SUB): acc (+)= sum over chunks c < nch and taps j < k of A(row wg * 64 + j * dil
// of the row step) . W(c, j) for the warpgroup's one 64-row block of a row step, whose chunks arrive SUB_CG per ring
// stage.  Per accumulator the (chunk, tap, plane product) sequence is the one consume() issues.
template <int N, int NW, int NAS, bool F16>
__device__ __forceinline__ void consume_rows(float (&acc)[N / 2], int wg, uint32_t a_st_u32, uint64_t* a_full, uint64_t* a_empty, Ring& ra,
                                             uint32_t w_st_u32, uint64_t* w_full, uint64_t* w_empty, Ring& rw, int nch, int k, int dil,
                                             int* err, long long& w_a, long long& w_w) {
  const uint64_t a_tmpl = make_desc(0, SUB_RS * 16, 128);
  const uint64_t b_tmpl = make_desc(0, (F16 ? 1 : 2) * N * 16, 128);
  const bool lane0 = (threadIdx.x & 31) == 0;
  int pend_w = -1, pend_a = -1;
  for (int c0 = 0; c0 < nch; c0 += SUB_CG) {
    mbar_wait_t(&a_full[ra.s], ra.p, err, 2, w_a);
    const uint32_t a_blk = a_st_u32 + ra.s * SUB_STAGE + wg * 64 * 16;
    for (int cl = 0; cl < SUB_CG; ++cl) {
      for (int j = 0; j < k; ++j) {
        mbar_wait_t(&w_full[rw.s], rw.p, err, 3, w_w);
        const uint32_t w_base = w_st_u32 + rw.s * (N * 64);
        const uint64_t b_hi = b_tmpl | (uint64_t)(w_base >> 4);
        const uint64_t b_lo = b_tmpl | (uint64_t)((w_base + N * 16) >> 4);
        const uint32_t first = ((c0 + cl) | j) != 0 ? 1u : 0u;
        const uint32_t row = a_blk + cl * SUB_CSB + j * dil * 16;
        const uint64_t a_hi = a_tmpl | (uint64_t)(row >> 4);
        const uint64_t a_lo = a_tmpl | (uint64_t)((row + 2 * SUB_RS * 16) >> 4);
        wgmma_fence();
        if constexpr (F16) {
          wgmma<N, true>(acc, a_hi, b_hi, first);
        } else {
          wgmma<N>(acc, a_hi, b_hi, first);
          wgmma<N>(acc, a_hi, b_lo, 1u);
          wgmma<N>(acc, a_lo, b_hi, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();          // the previous group has retired: its stages may be refilled
        if (lane0) {
          if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
          if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
        }
        pend_w = (int)rw.s;
        pend_a = (cl == SUB_CG - 1 && j == k - 1) ? (int)ra.s : -1;
        rw.next<NW>();
      }
    }
    ra.next<NAS>();
  }
  wgmma_wait<0>();
  if (lane0) {
    if (pend_w >= 0) mbar_arrive(&w_empty[pend_w]);
    if (pend_a >= 0) mbar_arrive(&a_empty[pend_a]);
  }
}

// 16-byte global -> shared copy that bypasses the registers (cp.async, L1 not allocated)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// barriers: a_full[NA] a_empty[NA] w_full[nw] w_empty[nw] q_full[NQ] q_empty[NQ], then the NQ tile ids
__device__ __forceinline__ void init_barriers(uint64_t* bars, int nw) {
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + NA;
  uint64_t* w_full = bars + 2 * NA;
  uint64_t* w_empty = bars + 2 * NA + nw;
  uint64_t* q_full = bars + 2 * NA + 2 * nw;
  uint64_t* q_empty = q_full + NQ;
  for (int i = 0; i < NA; ++i) { mbar_init(&a_full[i], NCONV); mbar_init(&a_empty[i], NCONS / 32); }
  for (int i = 0; i < nw; ++i) { mbar_init(&w_full[i], 1); mbar_init(&w_empty[i], NCONS / 32); }
  for (int i = 0; i < NQ; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], NREADERS); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ TileQueue tile_queue(uint64_t* bars, int nw) {
  uint64_t* q_full = bars + 2 * NA + 2 * nw;
  return TileQueue{reinterpret_cast<int*>(q_full + 2 * NQ), q_full, q_full + NQ, Ring{}};
}

// sub-row output (TcLaunch::out_sub): the element of the batch row's output that column col of tile row tau of problem
// P goes to
__device__ __forceinline__ int sub_elem(const TcLaunch& L, const TcProb& P, int tau, int col) {
  return (tau * P.out_stride + P.out_off) * L.out_ld + P.out_e0 + col;
}

// Tile loops of the roles.  The producer lane takes tickets one tile ahead of the tile it streams weights for, so the
// converters learn their next tile before they finish the current one.
#define PRODUCER_TILES                                                                     \
  TileQueue q = tile_queue(bars, NW);                                                      \
  long long w_q = 0;                                                                       \
  int t_next = blockIdx.x;                                                                 \
  q.put(t_next, L.err, w_q);                                                               \
  auto next_tile = [&]() {                                                                 \
    const int t = t_next;                                                                  \
    if (t >= 0) { t_next = take_ticket(L.sched, L.ntiles); q.put(t_next, L.err, w_q); }    \
    return t;                                                                              \
  };
#define READER_TILES                                                                       \
  TileQueue q = tile_queue(bars, NW);                                                      \
  long long w_q = 0;                                                                       \
  auto next_tile = [&]() { return q.get(L.err, w_q); };

// EPI = 0: bias (+ residual) only -- the HiFiGAN generator's hot path.  EPI = 1: bias, eval BatchNorm,
// tanh / relu, residual, partial N tile (acoustic model convs and GEMMs).  SUB: sub-row output (TcLaunch::out_sub, EPI 0
// only, the ConvTranspose); a template flag so that the ResBlock launches keep their epilogue as it is.
template <int N, int EPI, int MW, bool F16, bool SUB>
__global__ void __launch_bounds__(NTHREADS, 1) tc_conv_kernel(const __grid_constant__ TcLaunch L) {
  static_assert(!SUB || EPI == 0, "sub-row output uses the plain epilogue");
  using Cfg = TcCfg<N, MW, 0, EPI == 0, SUB>;
  constexpr int R = Cfg::R, RA = Cfg::RA, NW = Cfg::NW, NAS = Cfg::NAS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* a_st = smem;
  uint8_t* w_st = smem + Cfg::A_BYTES;
  // [NCWG][EPI_WG]; indexed from smem_raw so that its accesses compile to shared-memory instructions
  float* epi_st = reinterpret_cast<float*>(smem_raw + (w_st + NW * Cfg::W_STAGE - smem_raw));
  uint64_t* bars = reinterpret_cast<uint64_t*>(w_st + NW * Cfg::W_STAGE + Cfg::EPI_STAGE);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + NA;
  uint64_t* w_full = bars + 2 * NA;
  uint64_t* w_empty = bars + 2 * NA + NW;

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  if (tid == 0) init_barriers(bars, NW);
  __syncthreads();

  const int nch = L.Cin / 16;

  // every role walks the same tile sequence (next_tile); a tile is (problem, batch row, row tile).
  // Input rows outside [in_lo, valid) read as zero.  Output row tau is written while tau < valid, or, with per-row
  // bounds (TcProb::rb, plain epilogue only), while its output row tau * out_stride + out_off stays below out_hi.
  // SUB bounds each out_sub-float output row of a tile row instead: an element e of the batch row's output is written
  // iff 0 <= e < e_lim, e_lim = out_sub x (the first output row not written).
  constexpr bool ROW_BOUNDS = EPI == 0;
#define TILE_LOOP_BEGIN                                                           \
  for (int tile; (tile = next_tile()) >= 0;) {                                    \
    const Tile td = decode_tile(tile, L.nprob, L.tiles_per_row);                   \
    const int b = td.b;                                                            \
    const int tau0 = td.tt * R;                                                    \
    const TcProb& P = L.p[td.pi];                                                  \
    int valid = L.T_rows, in_lo = 0, out_hi = 0;                                  \
    if (ROW_BOUNDS && P.rb) {                                                     \
      in_lo = P.rb[3 * b]; valid = P.rb[3 * b + 1]; out_hi = P.rb[3 * b + 2];     \
      if (!SUB && tau0 * P.out_stride + P.out_off >= out_hi) continue;            \
    } else {                                                                      \
      if (L.len) {                                                                \
        const int v = L.len[b] * L.len_mul;                                       \
        valid = v < valid ? v : valid;                                            \
      }                                                                           \
      if (!SUB && tau0 >= valid) continue;                                        \
    }                                                                             \
    const int e_lim = SUB ? (P.rb ? out_hi * L.out_sub : valid * L.out_ld) : 0;   \
    if (SUB && sub_elem(L, P, tau0, 0) >= e_lim) continue;
#define TILE_LOOP_END }

  if (warp == PROD_WARP) {
    // ============================ weight producer ============================
    if ((tid & 31) == 0) {
      Ring rw;
      long long w_e = 0;
      PRODUCER_TILES
      TILE_LOOP_BEGIN
        (void)b; (void)tau0; (void)in_lo; (void)valid; (void)out_hi; (void)e_lim;
        // SUB: the consumers run the tile's MW row steps one after another, each over all (chunk, tap) blocks
        for (int mt = 0; mt < (SUB ? MW : 1); ++mt) produce_weights<N, NW, F16>(w_st, w_full, w_empty, rw, P.wpk, nch, P.k, L.err, w_e);
      TILE_LOOP_END
      if (L.dbg) L.dbg[(size_t)blockIdx.x * 16 + 4] = w_e;
    }
  } else if (warp > PROD_WARP) {
    // ============================ activation converters ============================
    const int ct = tid - NCONS - 32;
    Ring ra;
    long long w_ae = 0;
    READER_TILES
    TILE_LOOP_BEGIN
      const int k = P.k, dil = P.dil;
      const size_t in_base = (size_t)b * L.T_rows * L.in_ld;
      const float* x1 = L.pre_mode == 2 ? P.x1 + in_base : nullptr;
      const float* x2 = L.pre_mode == 2 ? P.x2 + in_base : nullptr;
      if constexpr (SUB) {
        // row step mt (NCWG x 64 rows + halo), SUB_CG chunks per stage
        for (int mt = 0; mt < MW; ++mt)
          for (int c0 = 0; c0 < nch; c0 += SUB_CG) {
            mbar_wait_t(&a_empty[ra.s], ra.p ^ 1, L.err, 5, w_ae);
            convert_rows<SUB_CG * 4, SUB_RS, SUB_CSB, F16, true>(a_st + ra.s * SUB_STAGE, ct, P.x0 + in_base, x1, x2, L.in_ld, c0 * 16,
                                                            tau0 + P.in_off + mt * NCWG * 64, NCWG * 64 + (k - 1) * dil, in_lo, valid,
                                                            L.pre_mode, L.pre_slope);
            fence_proxy_async();
            mbar_arrive(&a_full[ra.s]);
            ra.next<NAS>();
          }
      } else {
        for (int c = 0; c < nch; ++c) {
          mbar_wait_t(&a_empty[ra.s], ra.p ^ 1, L.err, 5, w_ae);
          convert_chunk<RA, F16>(a_st + ra.s * Cfg::A_STAGE, ct, P.x0 + in_base, x1, x2, L.in_ld, c, tau0 + P.in_off, R + (k - 1) * dil,
                            in_lo, valid, L.pre_mode, L.pre_slope);
          fence_proxy_async();
          mbar_arrive(&a_full[ra.s]);
          ra.next<NA>();
        }
      }
      (void)out_hi; (void)e_lim;
    TILE_LOOP_END
    if (L.dbg && ct == 0) L.dbg[(size_t)blockIdx.x * 16 + 5] = w_ae;
  } else {
    // ============================ consumers: wgmma + epilogue ============================
    const int wg = warp >> 2, lane = tid & 31;
    float acc[MW][N / 2];
    Ring ra, rw;
    long long w_a = 0, w_w = 0, t_epi = 0;
    const long long t_begin = clock64();
    const int n_valid = (EPI && L.n_valid > 0) ? L.n_valid : N;
    const int post_act = EPI ? L.post_act : 0;
    // plain epilogue (EPI = 0): this warpgroup's staging rows; the accumulator fragment's row and first column; a
    // thread's first staged row and float4 column when the warpgroup walks the rows (RPS rows per step, NQ4 steps)
    constexpr int EPI_NC = Cfg::EPI_NC, EPI_LD = Cfg::EPI_LD, RPS = 128 / (EPI_NC / 4), NQ4 = 64 / RPS;
    float* stg = epi_st + wg * Cfg::EPI_WG;
    float* stg_bias = stg + 64 * EPI_LD;
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);
    const int dr = (tid & 127) / (EPI_NC / 4), dq = (tid & 127) % (EPI_NC / 4);
    READER_TILES
    TILE_LOOP_BEGIN
      const size_t out_base = (size_t)b * L.rows_out * (SUB ? L.out_sub : L.out_ld);
      const int ostride = P.out_stride, ooff = P.out_off, oe0 = SUB ? P.out_e0 : 0;
      // output row tau is stored while it is valid; the condition is monotone in tau
      auto row_ok = [&](int tau) { return (ROW_BOUNDS && P.rb) ? tau * ostride + ooff < out_hi : tau < valid; };
      // ... and the float4 at element e (of tile row tau) of the batch row's output (plain epilogue); with sub-row output
      // it lies in one output row (out_sub % 4 == 0)
      auto elem_ok = [&](int tau, int e) { return SUB ? e >= 0 && e < e_lim : row_ok(tau); };
      // first row of the warpgroup's 64-row block mt: the warpgroup's MW blocks are adjacent, or (SUB) block mt of each
      // warpgroup lies in row step mt
      auto blk_row = [&](int mt) { return tau0 + (SUB ? mt * NCWG + wg : wg * MW + mt) * 64; };
      // cp.async the residual of pass (mt, nh) -- rows tau0 + (wg * MW + mt) * 64..., columns nh * EPI_NC... -- into
      // the staging rows; wait_pass makes every thread's copies visible to the warpgroup
      auto fetch_pass = [&](int mt, int nh) {
        if (P.resid) {
          const int blk = blk_row(mt);
#pragma unroll
          for (int i = 0; i < NQ4; ++i) {
            const int row = i * RPS + dr, tau = blk + row;
            const int e = (tau * ostride + ooff) * L.out_ld + oe0 + nh * EPI_NC + dq * 4;
            if (elem_ok(tau, e)) cp_async16(stg + row * EPI_LD + dq * 4, P.resid + out_base + e);
          }
        }
        cp_async_commit();
      };
      auto wait_pass = [&]() {
        cp_async_wait_all();
        named_bar(2 + wg, 128);
      };
      if constexpr (EPI == 0) {
        // the tile's bias (read by the fragments from shared memory, so the compiler keeps no copy of it in registers)
        // and the first pass's residual are requested before the wgmmas
        if ((tid & 127) < N / 4) cp_async16(stg_bias + (tid & 127) * 4, P.bias + (tid & 127) * 4);
        fetch_pass(0, 0);
      }
      if constexpr (SUB) {
#pragma unroll
        for (int mt = 0; mt < MW; ++mt)
          consume_rows<N, NW, NAS, F16>(acc[mt], wg, smem_u32(a_st), a_full, a_empty, ra, smem_u32(w_st), w_full, w_empty, rw, nch, P.k,
                                        P.dil, L.err, w_a, w_w);
      } else {
        consume<N, MW, RA, NW, true, false, F16>(acc, wg, smem_u32(a_st), a_full, a_empty, ra, smem_u32(w_st), w_full, w_empty, rw, nch,
                                                 P.k, P.dil, L.err, w_a, w_w);
      }
      const long long t_epi0 = clock64();
      if constexpr (EPI == 0) {
        // Staged through shared memory, one pass per 64-row block of the warpgroup and EPI_NC columns: the pass's
        // residual rows are copied into the staging rows with cp.async (pass 0's at tile start, so they arrive under
        // the wgmmas; a later pass's as soon as the previous one has left), the accumulator fragments add bias and the
        // staged residual in place, and the warpgroup stores the rows in float4 units.  The residual is the layer's
        // input, read from DRAM: this way a tile waits for it at most once per pass instead of once per fragment pair.
        wait_pass();
#pragma unroll
        for (int mt = 0; mt < MW; ++mt) {
          // uniform over the warpgroup: past the last output row, so no later row of it is stored
          const int blk = blk_row(mt);
          if (SUB ? sub_elem(L, P, blk, 0) >= e_lim : !row_ok(blk)) break;
#pragma unroll
          for (int nh = 0; nh < N / EPI_NC; ++nh) {
            if (mt + nh > 0 && P.resid) {
              fetch_pass(mt, nh);
              wait_pass();
            }
#pragma unroll
            for (int jn = 0; jn < EPI_NC / 8; ++jn) {
              const int col = jn * 8 + fc, e = (nh * (EPI_NC / 8) + jn) * 4;
              const float2 bi = *reinterpret_cast<const float2*>(stg_bias + nh * EPI_NC + col);
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float2* s = reinterpret_cast<float2*>(stg + (fr + 8 * h) * EPI_LD + col);
                float2 o = make_float2(acc[mt][e + 2 * h] + bi.x, acc[mt][e + 2 * h + 1] + bi.y);
                if (P.resid) {
                  const float2 r = *s;
                  o.x += r.x; o.y += r.y;
                }
                *s = o;
              }
            }
            named_bar(2 + wg, 128);
#pragma unroll
            for (int i = 0; i < NQ4; ++i) {
              const int row = i * RPS + dr, tau = blk + row;
              const int e = (tau * ostride + ooff) * L.out_ld + oe0 + nh * EPI_NC + dq * 4;
              if (elem_ok(tau, e))
                *reinterpret_cast<float4*>(P.out + out_base + e) = *reinterpret_cast<const float4*>(stg + row * EPI_LD + dq * 4);
            }
            named_bar(2 + wg, 128);   // stored before the next pass or tile rewrites the staging rows
          }
        }
      } else {
        const int row_w = tau0 + wg * MW * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int mt = 0; mt < MW; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int tau = row_w + mt * 64 + 8 * h;
            if (!row_ok(tau)) continue;
            const size_t orow = out_base + (size_t)(tau * ostride + ooff) * L.out_ld;
#pragma unroll
            for (int jn = 0; jn < N / 8; ++jn) {
              const int col = jn * 8 + 2 * (lane & 3);
              if (col >= n_valid) continue;
              float2 o = make_float2(acc[mt][jn * 4 + 2 * h], acc[mt][jn * 4 + 2 * h + 1]);
              const float2 bi = __ldg(reinterpret_cast<const float2*>(P.bias + col));
              o.x += bi.x; o.y += bi.y;
              if (P.bn_mean) {
                const float2 mu = __ldg(reinterpret_cast<const float2*>(P.bn_mean + col));
                const float2 iv = __ldg(reinterpret_cast<const float2*>(P.bn_inv + col));
                const float2 of = __ldg(reinterpret_cast<const float2*>(P.bn_off + col));
                o.x = (o.x - mu.x) * iv.x + of.x; o.y = (o.y - mu.y) * iv.y + of.y;
              }
              if (post_act == 1) { o.x = tanhf(o.x); o.y = tanhf(o.y); }
              else if (post_act == 2) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); }
              if (P.resid) {
                const float2 r = __ldg(reinterpret_cast<const float2*>(P.resid + orow + col));
                o.x += r.x; o.y += r.y;
              }
              *reinterpret_cast<float2*>(P.out + orow + col) = o;
            }
          }
      }
      t_epi += clock64() - t_epi0;
    TILE_LOOP_END
    if (L.dbg && tid == 0) {
      long long* d = L.dbg + (size_t)blockIdx.x * 16;
      d[0] = clock64() - t_begin; d[1] = t_epi; d[2] = w_a; d[3] = w_w;
    }
  }
#undef TILE_LOOP_BEGIN
#undef TILE_LOOP_END
}

// Fused ResBlock1 pair:  y = conv2(lrelu(conv1(lrelu(x)) + b1)) + b2 + x  for C = N in {32, 64}, both convs with zero
// padding at each row's true end (hifigan/model.py:44-51).  A tile stores R_OUT output rows [tau0, tau0 + R_OUT) and
// computes the intermediate on rows [tau0 - h2, tau0 - h2 + R) (h2 = (k - 1) / 2, conv2's padding) entirely on chip.
// A2_REGS: conv2 takes its A operand from registers (ldmatrix + register-A wgmma) instead of from shared memory.
// F16: both convs on fp16 operands; the intermediate is one saturated fp16 plane.
template <int N, int MW, bool A2_REGS, bool F16>
__global__ void __launch_bounds__(NTHREADS, 1) tc_pair_kernel(const __grid_constant__ TcPairLaunch L) {
  using Cfg = TcCfg<N, MW, 1>;
  constexpr int R = Cfg::R, R_OUT = Cfg::R_OUT, RA = Cfg::RA, NW = Cfg::NW, NCH = N / 16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* a_st = smem;
  uint8_t* w_st = smem + NA * Cfg::A_STAGE;
  uint8_t* mid = w_st + NW * Cfg::W_STAGE;                   // [chunk][plane][k-half][RA rows][16 B]: conv2's A operand
  uint64_t* bars = reinterpret_cast<uint64_t*>(mid + Cfg::NCH2 * Cfg::A_STAGE);
  uint64_t* a_full = bars;
  uint64_t* a_empty = bars + NA;
  uint64_t* w_full = bars + 2 * NA;
  uint64_t* w_empty = bars + 2 * NA + NW;

  const int tid = threadIdx.x;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  if (tid == 0) init_barriers(bars, NW);
  __syncthreads();

#define TILE_LOOP_BEGIN                                                   \
  for (int tile; (tile = next_tile()) >= 0;) {                            \
    const Tile td = decode_tile(tile, L.nprob, L.tiles_per_row);        \
    const int b = td.b;                                                    \
    const int tau0 = td.tt * R_OUT;                                        \
    int valid = L.T_rows;                                                 \
    if (L.len) {                                                          \
      const int v = L.len[b] * L.len_mul;                                 \
      valid = v < valid ? v : valid;                                      \
    }                                                                     \
    if (tau0 >= valid) continue;                                          \
    const TcPairProb& P = L.p[td.pi];                                      \
    const int k = P.k, dil = P.dil, h2 = (k - 1) / 2;
#define TILE_LOOP_END }

  if (warp == PROD_WARP) {
    if ((tid & 31) == 0) {
      Ring rw;
      long long w_e = 0;
      PRODUCER_TILES
      TILE_LOOP_BEGIN
        (void)b; (void)tau0; (void)dil; (void)h2;
        produce_weights<N, NW, F16>(w_st, w_full, w_empty, rw, P.w1pk, NCH, k, L.err, w_e);
        produce_weights<N, NW, F16>(w_st, w_full, w_empty, rw, P.w2pk, NCH, k, L.err, w_e);
      TILE_LOOP_END
    }
  } else if (warp > PROD_WARP) {
    const int ct = tid - NCONS - 32;
    Ring ra;
    long long w_ae = 0;
    READER_TILES
    TILE_LOOP_BEGIN
      const float* x = P.x + (size_t)b * L.T_rows * N;
      const int row_base = tau0 - h2 - (k - 1) * dil / 2;
      for (int c = 0; c < NCH; ++c) {
        mbar_wait_t(&a_empty[ra.s], ra.p ^ 1, L.err, 5, w_ae);
        convert_chunk<RA, F16>(a_st + ra.s * Cfg::A_STAGE, ct, x, nullptr, nullptr, N, c, row_base, R + (k - 1) * dil, 0, valid, 1, L.slope);
        fence_proxy_async();
        mbar_arrive(&a_full[ra.s]);
        ra.next<NA>();
      }
    TILE_LOOP_END
  } else {
    const int wg = warp >> 2, lane = tid & 31;
    float acc[MW][N / 2];
    Ring ra, rw;
    long long w_a = 0, w_w = 0;
    const long long t_begin = clock64();
    const float slope = L.slope;
    READER_TILES
    TILE_LOOP_BEGIN
      // ---- conv1 over the R intermediate rows ----
      consume<N, MW, RA, NW, true, false, F16>(acc, wg, smem_u32(a_st), a_full, a_empty, ra, smem_u32(w_st), w_full, w_empty, rw, NCH, k, dil,
                                               L.err, w_a, w_w);
      // ---- + b1, lrelu, zero outside the row, hi/lo split (or fp16) -> conv2's operand (rows of this warpgroup only) ----
      const int lr_w = wg * MW * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int mt = 0; mt < MW; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int lr = lr_w + mt * 64 + 8 * h;
          const int u = tau0 - h2 + lr;
          const bool inside = u >= 0 && u < valid;
#pragma unroll
          for (int jn = 0; jn < N / 8; ++jn) {
            const int col = jn * 8 + 2 * (lane & 3);
            const float2 bi = __ldg(reinterpret_cast<const float2*>(P.b1 + col));
            const float v0 = inside ? lrelu(acc[mt][jn * 4 + 2 * h] + bi.x, slope) : 0.f;
            const float v1 = inside ? lrelu(acc[mt][jn * 4 + 2 * h + 1] + bi.y, slope) : 0.f;
            uint8_t* dst = mid + (col >> 4) * Cfg::A_STAGE + (((col >> 3) & 1) * RA + lr) * 16 + (col & 7) * 2;
            if constexpr (F16) {
              *reinterpret_cast<uint32_t*>(dst) = f16x2_sat(v0, v1);
            } else {
              const __nv_bfloat162 hi = __floats2bfloat162_rn(v0, v1);
              const __nv_bfloat162 lo = __floats2bfloat162_rn(v0 - __low2float(hi), v1 - __high2float(hi));
              *reinterpret_cast<__nv_bfloat162*>(dst) = hi;
              *reinterpret_cast<__nv_bfloat162*>(dst + 2 * RA * 16) = lo;
            }
          }
        }
      fence_proxy_async();
      named_bar(1, NCONS);          // conv2 of a row reads intermediate rows of the other warpgroup
      // ---- conv2 (dilation 1) ----
      consume<N, MW, RA, NW, false, A2_REGS, F16>(acc, wg, smem_u32(mid), a_full, a_empty, ra, smem_u32(w_st), w_full, w_empty, rw, NCH, k, 1,
                                                  L.err, w_a, w_w);
      named_bar(1, NCONS);          // both warpgroups are done reading the intermediate before the next tile rewrites it
      // ---- + b2 + x ----
      const float* x = P.x + (size_t)b * L.T_rows * N;
      float* out = P.out + (size_t)b * L.T_rows * N;
#pragma unroll
      for (int mt = 0; mt < MW; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int lr = lr_w + mt * 64 + 8 * h;
          const int tau = tau0 + lr;
          if (lr >= R_OUT || tau >= valid) continue;
#pragma unroll
          for (int jn = 0; jn < N / 8; ++jn) {
            const int col = jn * 8 + 2 * (lane & 3);
            const float2 bi = __ldg(reinterpret_cast<const float2*>(P.b2 + col));
            const float2 r = __ldg(reinterpret_cast<const float2*>(x + (size_t)tau * N + col));
            float2 o;
            o.x = acc[mt][jn * 4 + 2 * h] + bi.x + r.x;
            o.y = acc[mt][jn * 4 + 2 * h + 1] + bi.y + r.y;
            *reinterpret_cast<float2*>(out + (size_t)tau * N + col) = o;
          }
        }
    TILE_LOOP_END
    if (L.dbg && tid == 0) {
      long long* d = L.dbg + (size_t)blockIdx.x * 16;
      d[0] = clock64() - t_begin; d[2] = w_a; d[3] = w_w;
    }
  }
#undef TILE_LOOP_BEGIN
#undef TILE_LOOP_END
}

// fp32 Haiku conv weight w[k][Cin][Cout_total] -> packed blocks for output columns [n0, n0+N):
//   bf16x3: [chunk c = Cin/16][tap j][k-half][plane hi|lo][n][8] bf16
//   fp16:   [chunk c = Cin/16][tap j][k-half][n][8] fp16, saturated to +-65504
template <bool F16>
__global__ void pack_w_kernel(const float* __restrict__ w, uint16_t* __restrict__ dst, int k, int Cin, int Cout_total, int n0, int N) {
  const size_t total = (size_t)k * Cin * N;
  for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int n = idx % N;
    const int i = (idx / N) % Cin;
    const int j = idx / ((size_t)N * Cin);
    const float v = (n0 + n) < Cout_total ? w[((size_t)j * Cin + i) * Cout_total + n0 + n] : 0.f;
    const int c = i / 16, kh = (i % 16) / 8, e = i % 8;
    if constexpr (F16) {
      const size_t blk = ((size_t)c * k + j) * (size_t)(2 * N * 8);
      dst[blk + ((size_t)kh * N + n) * 8 + e] = (uint16_t)(f16x2_sat(v, 0.f) & 0xffffu);
      continue;
    }
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    const size_t blk = ((size_t)c * k + j) * (size_t)(4 * N * 8);
    dst[blk + ((size_t)(kh * 2 + 0) * N + n) * 8 + e] = __bfloat16_as_ushort(hi);   // [k-half][plane hi|lo][n][8]: hi and lo rows of a
    dst[blk + ((size_t)(kh * 2 + 1) * N + n) * 8 + e] = __bfloat16_as_ushort(lo);   // k-half are adjacent, so [W_hi | W_lo] is also one 2N-row operand
  }
}

template <int N, int EPI, int MW, bool F16, bool SUB = false>
int launch_cfg(vtts_ctx* ctx, TcLaunch& L, cudaStream_t st) {
  using Cfg = TcCfg<N, MW, 0, EPI == 0, SUB>;
  static bool attr_done_dev[64] = {};   // function attributes are per device (a process may hold contexts on several GPUs)
  if (!attr_done_dev[ctx->device & 63]) {
    VTTS_CUDA(cudaFuncSetAttribute(tc_conv_kernel<N, EPI, MW, F16, SUB>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done_dev[ctx->device & 63] = true;
  }
  for (int i = 0; i < L.nprob; ++i)
    if ((L.p[i].k - 1) * L.p[i].dil > (SUB ? SUB_HALO : HALO)) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: halo too large");
  if (SUB && L.Cin % (SUB_CG * 16)) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: sub-row output needs Cin %% %d == 0, not %d", SUB_CG * 16, L.Cin);
  // the expensive problems (large k) first: within each row tile they are handed out before the cheap ones
  std::stable_sort(L.p, L.p + L.nprob, [](const TcProb& a, const TcProb& b) { return a.k > b.k; });
  L.tiles_per_row = ((L.tile_rows > 0 ? L.tile_rows : L.T_rows) + Cfg::R - 1) / Cfg::R;
  L.ntiles = L.nprob * L.tiles_per_row * L.B;
  const int grid = L.ntiles < ctx->sm_count ? L.ntiles : ctx->sm_count;
  tc_conv_kernel<N, EPI, MW, F16, SUB><<<grid, NTHREADS, Cfg::SMEM_BYTES, st>>>(L);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

// rows per warpgroup (MW x 64): as many as keep the accumulators at <= 128 registers per thread
template <int N>
int launch_n(vtts_ctx* ctx, TcLaunch& L, cudaStream_t st) {
  constexpr int MW = N >= 256 ? 1 : (N == 128 ? 2 : 4);
  bool generic = L.post_act != 0 || (L.n_valid > 0 && L.n_valid < N);
  bool rb = false;
  for (int i = 0; i < L.nprob; ++i) {
    generic |= L.p[i].bn_mean != nullptr;
    rb |= L.p[i].rb != nullptr;
  }
  if ((rb || L.out_sub) && generic) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: per-row bounds and sub-row output use the plain epilogue");
  // a float4 of the plain epilogue lies in one output row
  if (L.out_sub < 0 || (L.out_sub && (L.out_sub % 4 || L.out_ld % L.out_sub)))
    return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: output rows of %d floats in tile rows of %d", L.out_sub, L.out_ld);
  if (!generic) {
    // the plain epilogue copies the bias and the residual and stores the output in float4 row segments, at 32-bit
    // offsets within a batch row
    const int row_w = L.out_sub ? L.out_sub : L.out_ld;
    if ((int64_t)L.rows_out * row_w > INT32_MAX) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: %d output rows of %d", L.rows_out, row_w);
    bool aligned = L.out_ld % 4 == 0;
    for (int i = 0; i < L.nprob; ++i) aligned &= (((uintptr_t)L.p[i].out | (uintptr_t)L.p[i].resid | (uintptr_t)L.p[i].bias) & 15) == 0;
    if (!aligned) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: the plain epilogue needs 16-byte aligned out / resid rows and bias (out_ld %d)", L.out_ld);
  }
  // fp16 operands serve the generator, whose convs all use the plain epilogue
  if (L.f16 && generic) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: fp16 operands use the plain epilogue");
  if (L.f16) return L.out_sub ? launch_cfg<N, 0, MW, true, true>(ctx, L, st) : launch_cfg<N, 0, MW, true>(ctx, L, st);
  if (generic) return launch_cfg<N, 1, MW, false>(ctx, L, st);
  return L.out_sub ? launch_cfg<N, 0, MW, false, true>(ctx, L, st) : launch_cfg<N, 0, MW, false>(ctx, L, st);
}

template <int N, int MW, bool A2_REGS, bool F16 = false>
int launch_pair(vtts_ctx* ctx, TcPairLaunch& L, cudaStream_t st) {
  using Cfg = TcCfg<N, MW, 1>;
  static bool attr_done_dev[64] = {};
  if (!attr_done_dev[ctx->device & 63]) {
    VTTS_CUDA(cudaFuncSetAttribute(tc_pair_kernel<N, MW, A2_REGS, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_done_dev[ctx->device & 63] = true;
  }
  for (int i = 0; i < L.nprob; ++i)
    if (L.p[i].k - 1 > PAIR_OVERLAP || (L.p[i].k - 1) * L.p[i].dil > HALO) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_pair: halo too large");
  // expensive problems (large k) first: within each row tile they are handed out before the cheap ones
  std::stable_sort(L.p, L.p + L.nprob, [](const TcPairProb& a, const TcPairProb& b) { return a.k > b.k; });
  L.tiles_per_row = (L.T_rows + Cfg::R_OUT - 1) / Cfg::R_OUT;
  L.ntiles = L.nprob * L.tiles_per_row * L.B;
  const int grid = L.ntiles < ctx->sm_count ? L.ntiles : ctx->sm_count;
  tc_pair_kernel<N, MW, A2_REGS, F16><<<grid, NTHREADS, Cfg::SMEM_BYTES, st>>>(L);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

size_t vtts_tc_packed_elems(int k, int Cin, int N, bool f16) { return (size_t)k * Cin * N * (f16 ? 1 : 2); }

int vtts_tc_pack_weights(vtts_ctx* ctx, const float* w, void* dst, int k, int Cin, int Cout_total, int n0, int N, bool f16) {
  if (f16) pack_w_kernel<true><<<256, 256>>>(w, reinterpret_cast<uint16_t*>(dst), k, Cin, Cout_total, n0, N);
  else pack_w_kernel<false><<<256, 256>>>(w, reinterpret_cast<uint16_t*>(dst), k, Cin, Cout_total, n0, N);
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

int vtts_tc_tile_n(int Cout) { return Cout <= 32 ? 32 : (Cout <= 64 ? 64 : (Cout <= 128 ? 128 : 256)); }

size_t vtts_tc_conv_packed_bytes(int k, int Cin, int Cout, bool f16) {
  const int N = vtts_tc_tile_n(Cout), nt = (Cout + N - 1) / N;
  return ((vtts_tc_packed_elems(k, Cin, N, f16) * 2 + 255) & ~size_t(255)) * nt;
}

int vtts_tc_pack_conv(vtts_ctx* ctx, const float* w, int k, int Cin, int Cout, bool f16, char*& cursor, std::vector<void*>& out) {
  const int N = vtts_tc_tile_n(Cout), nt = (Cout + N - 1) / N;
  for (int t = 0; t < nt; ++t) {
    int rc = vtts_tc_pack_weights(ctx, w, cursor, k, Cin, Cout, t * N, N, f16);
    if (rc) return rc;
    out.push_back(cursor);
    cursor += (vtts_tc_packed_elems(k, Cin, N, f16) * 2 + 255) & ~size_t(255);
  }
  return VTTS_OK;
}

int vtts_conv_dispatch(vtts_ctx* ctx, const ConvLaunch& L, void* const* wpk, cudaStream_t st) {
  // the fp16 mode covers the generator only: here (acoustic and duration models) it runs bf16x3 like mode 1
  if (ctx->precision == VTTS_PRECISION_FP32 || wpk == nullptr) return vtts_launch_conv(ctx, L, st);
  const int N = vtts_tc_tile_n(L.Cout), nt = (L.Cout + N - 1) / N;
  TcLaunch TL;
  auto reset = [&]() {
    memset(&TL, 0, sizeof(TL));
    TL.Cin = L.Cin; TL.N = N; TL.in_ld = L.Cin; TL.out_ld = L.Cout; TL.B = L.B; TL.T_rows = L.T_rows; TL.rows_out = L.rows_out;
    TL.len = L.len; TL.len_mul = L.len_mul; TL.pre_mode = L.pre_mode; TL.pre_slope = L.pre_slope; TL.post_act = L.post_act;
    TL.n_valid = (L.Cout % N) ? (L.Cout % N) : N;   // only meaningful when nt == 1 or for the last tile (handled below)
  };
  reset();
  // tiles that are completely valid and a partial last tile need different n_valid -> separate launches
  for (int pass = 0; pass < 2; ++pass) {
    const bool partial = pass == 1;
    if (partial && (L.Cout % N) == 0) break;
    reset();
    TL.n_valid = partial ? (L.Cout % N) : N;
    for (int pi = 0; pi < L.nprob; ++pi) {
      const ConvProb& cp = L.p[pi];
      for (int t = 0; t < nt; ++t) {
        const bool is_partial = (t == nt - 1) && (L.Cout % N) != 0;
        if (is_partial != partial) continue;
        const int n0 = t * N;
        TcProb q;
        memset(&q, 0, sizeof(q));
        q.x0 = cp.x0; q.x1 = cp.x1; q.x2 = cp.x2;
        q.wpk = wpk[pi * nt + t];
        q.bias = cp.bias + n0;
        q.resid = cp.resid ? cp.resid + n0 : nullptr;
        if (cp.bn_mean) { q.bn_mean = cp.bn_mean + n0; q.bn_inv = cp.bn_inv + n0; q.bn_off = cp.bn_off + n0; }
        q.out = cp.out + n0;
        q.k = cp.k; q.dil = cp.dil; q.in_off = cp.in_off; q.out_stride = cp.out_stride; q.out_off = cp.out_off;
        TL.p[TL.nprob++] = q;
        if (TL.nprob == 8) {
          int rc = vtts_launch_tc_conv(ctx, TL, st);
          if (rc) return rc;
          TL.nprob = 0;
        }
      }
    }
    if (TL.nprob > 0) {
      int rc = vtts_launch_tc_conv(ctx, TL, st);
      if (rc) return rc;
    }
  }
  return VTTS_OK;
}

int vtts_launch_tc_conv(vtts_ctx* ctx, TcLaunch& L, cudaStream_t st) {
  if (L.nprob < 1 || L.nprob > 8) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: nprob %d", L.nprob);
  if (L.Cin % 16 != 0) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: Cin %d", L.Cin);
  for (int i = 0; i < L.nprob; ++i)
    if (L.p[i].k < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: k");
  L.sched = ctx->d_tc_sched;
  L.err = ctx->d_err;
  L.dbg = ctx->tc_dbg_on ? ctx->d_tc_dbg : nullptr;
  switch (L.N) {
    case 256: return launch_n<256>(ctx, L, st);
    case 128: return launch_n<128>(ctx, L, st);
    case 64: return launch_n<64>(ctx, L, st);
    case 32: return launch_n<32>(ctx, L, st);
    default: return ctx->fail(VTTS_ERR_BAD_ARG, "tc_conv: N %d unsupported", L.N);
  }
}

int vtts_launch_tc_pair(vtts_ctx* ctx, TcPairLaunch& L, cudaStream_t st) {
  if (L.nprob < 1 || L.nprob > 3) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_pair: nprob %d", L.nprob);
  for (int i = 0; i < L.nprob; ++i)
    if (L.p[i].k < 1 || L.p[i].x == L.p[i].out) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_pair: bad problem %d", i);
  L.sched = ctx->d_tc_sched;
  L.err = ctx->d_err;
  L.dbg = ctx->tc_dbg_on ? ctx->d_tc_dbg : nullptr;
  if (L.N != 32 && L.N != 64) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_pair: C %d unsupported (32 or 64)", L.N);
  // vtts_ctx::pair_ts: 2 = 256-row tiles (default), 1 = the same with conv2's A operand in registers, 0 = 128-row tiles
  if (L.f16) {
    if (ctx->pair_ts != 2) return ctx->fail(VTTS_ERR_BAD_ARG, "tc_pair: fp16 operands exist for the default pair form (256-row tiles) only, not form %d", ctx->pair_ts);
    return L.N == 64 ? launch_pair<64, 2, false, true>(ctx, L, st) : launch_pair<32, 2, false, true>(ctx, L, st);
  }
  if (ctx->pair_ts == 1) return L.N == 64 ? launch_pair<64, 2, true>(ctx, L, st) : launch_pair<32, 2, true>(ctx, L, st);
  if (ctx->pair_ts == 0) return L.N == 64 ? launch_pair<64, 1, false>(ctx, L, st) : launch_pair<32, 1, false>(ctx, L, st);
  return L.N == 64 ? launch_pair<64, 2, false>(ctx, L, st) : launch_pair<32, 2, false>(ctx, L, st);
}
