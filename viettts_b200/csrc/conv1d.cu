// Generic NWC float32 conv1d as an implicit GEMM on the FP32 pipe (strict-parity path).
//
// Restates hk.Conv1D as used at vietTTS/hifigan/model.py:21-41,83,107 and
// vietTTS/nat/model.py:16-18,91-92 (w[K,Cin,Cout], zero padding at the true sequence
// ends), with the surrounding element-wise work of the reference fused in:
//   * leaky_relu on the input            (hifigan/model.py:46,48,112)
//   * (r0+r1+r2)/3 of three resblocks     (hifigan/model.py:115-121) on the input
//   * bias, eval BatchNorm, tanh / relu   (nat/model.py:28-34,116-120)
//   * residual add                        (hifigan/model.py:50, nat/model.py:144)
// A launch carries up to 8 independent "problems" (blockIdx.z) that share shapes but not
// weights: the three resblocks of a stage, or the `stride` output phases of a
// ConvTranspose (hifigan/model.py:87-95), each phase being a 2-tap conv whose output
// rows are interleaved with stride `out_stride`.
//
// Tiling: CTA = TM output rows x TN output channels, 256 threads, 8x8 outputs per
// thread (rows strided by TM/8 so that shared-memory reads of the activation tile are
// warp broadcasts for any tap offset j*dilation).  K loop = (16-channel chunk) x (tap);
// the activation chunk [16][TM + (k-1)d] is staged once per chunk (transposed, with
// the input transform applied), the 16 x TN weight slice of every tap is double
// buffered with cp.async.
#include "vtts_internal.cuh"

namespace {

constexpr int KC = 16;
constexpr int HALO_MAX = 50;  // (k-1)*d max = 10*5

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool pred) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = pred ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}

template <int TM, int TN>
struct ConvCfg {
  static constexpr int NTN = TN / 8;
  static constexpr int NTM = TM / 8;
  static_assert(NTN * NTM == 256, "256 threads");
  static constexpr int XS_ROWS = TM + HALO_MAX;
  static constexpr int XS_STRIDE = ((XS_ROWS + 7) / 8) * 8 + 2;  // == 2 mod 8: conflict-free transposed stores
  static constexpr int SMEM_BYTES = (KC * XS_STRIDE + 2 * KC * TN) * 4;
};

__device__ __forceinline__ float lrelu(float v, float s) { return v >= 0.f ? v : s * v; }

template <int TM, int TN>
__global__ void __launch_bounds__(256, 2) conv1d_nwc_kernel(const __grid_constant__ ConvLaunch L) {
  using Cfg = ConvCfg<TM, TN>;
  constexpr int NTM = Cfg::NTM, NTN = Cfg::NTN, XS = Cfg::XS_STRIDE;
  extern __shared__ __align__(16) float smem[];
  float* xs = smem;
  float* ws = smem + KC * XS;

  const int nprob = L.nprob;
  const int pi = blockIdx.z % nprob;
  const int n0 = (blockIdx.z / nprob) * TN;
  const ConvProb& P = L.p[pi];
  const int b = blockIdx.y;
  const int tau0 = blockIdx.x * TM;
  int valid = L.T_rows;
  if (L.len) {
    int v = L.len[b] * L.len_mul;
    valid = v < valid ? v : valid;
  }
  if (tau0 >= valid) return;

  const int Cin = L.Cin, Cout = L.Cout;
  const int k = P.k, dil = P.dil;
  const int rows = TM + (k - 1) * dil;
  const int tid = threadIdx.x;
  const int tn = tid % NTN, tm = tid / NTN;
  const int pre_mode = L.pre_mode;
  const float slope = L.pre_slope;

  const size_t in_base = (size_t)b * L.T_rows * Cin;
  const float* __restrict__ x0 = P.x0 + in_base;
  const float* __restrict__ x1 = pre_mode == 2 ? P.x1 + in_base : nullptr;
  const float* __restrict__ x2 = pre_mode == 2 ? P.x2 + in_base : nullptr;
  const float* __restrict__ wg = P.w;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int n = 0; n < 8; ++n) acc[i][n] = 0.f;

  const int nsteps = (Cin / KC) * k;

  auto issue_ws = [&](int c, int j, int buf) {
    const float* wsrc = wg + ((size_t)j * Cin + (size_t)c * KC) * Cout + n0;
    float* wdst = ws + buf * KC * TN;
    for (int e = tid; e < KC * TN / 4; e += 256) {
      int kc = e / (TN / 4), n4 = (e % (TN / 4)) * 4;
      bool ok = (n0 + n4) < Cout;
      cp_async16(wdst + kc * TN + n4, ok ? (const void*)(wsrc + (size_t)kc * Cout + n4) : (const void*)wg, ok);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };

  auto load_xs = [&](int c) {
    const int c0 = c * KC;
    const int row_base = tau0 + P.in_off;
    for (int e = tid; e < rows * 4; e += 256) {
      int rr = e >> 2, q = e & 3;
      int r = row_base + rr;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r >= 0 && r < valid) {
        size_t off = (size_t)r * Cin + c0 + q * 4;
        v = __ldg(reinterpret_cast<const float4*>(x0 + off));
        if (pre_mode == 2) {
          float4 a = __ldg(reinterpret_cast<const float4*>(x1 + off));
          float4 bb = __ldg(reinterpret_cast<const float4*>(x2 + off));
          v.x = ((v.x + a.x) + bb.x) / 3.0f;
          v.y = ((v.y + a.y) + bb.y) / 3.0f;
          v.z = ((v.z + a.z) + bb.z) / 3.0f;
          v.w = ((v.w + a.w) + bb.w) / 3.0f;
        }
        if (pre_mode >= 1) {
          v.x = lrelu(v.x, slope);
          v.y = lrelu(v.y, slope);
          v.z = lrelu(v.z, slope);
          v.w = lrelu(v.w, slope);
        }
      }
      float* d = xs + (q * 4) * XS + rr;
      d[0] = v.x;
      d[XS] = v.y;
      d[2 * XS] = v.z;
      d[3 * XS] = v.w;
    }
  };

  issue_ws(0, 0, 0);
  int buf = 0, c = 0, j = 0;
  for (int step = 0; step < nsteps; ++step) {
    if (j == 0) {
      if (step > 0) __syncthreads();  // all warps finished reading the previous activation chunk
      load_xs(c);
    }
    asm volatile("cp.async.wait_group 0;\n" ::);
    __syncthreads();
    int jn = j + 1, cn = c;
    if (jn == k) {
      jn = 0;
      cn = c + 1;
    }
    if (step + 1 < nsteps) issue_ws(cn, jn, buf ^ 1);

    const float* wb = ws + buf * KC * TN + tn * 8;
    const float* xb = xs + tm + j * dil;
#pragma unroll
    for (int kc = 0; kc < KC; ++kc) {
      float a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = xb[kc * XS + i * NTM];
      const float4 b0 = *reinterpret_cast<const float4*>(wb + kc * TN);
      const float4 b1 = *reinterpret_cast<const float4*>(wb + kc * TN + 4);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i][0] = fmaf(a[i], b0.x, acc[i][0]);
        acc[i][1] = fmaf(a[i], b0.y, acc[i][1]);
        acc[i][2] = fmaf(a[i], b0.z, acc[i][2]);
        acc[i][3] = fmaf(a[i], b0.w, acc[i][3]);
        acc[i][4] = fmaf(a[i], b1.x, acc[i][4]);
        acc[i][5] = fmaf(a[i], b1.y, acc[i][5]);
        acc[i][6] = fmaf(a[i], b1.z, acc[i][6]);
        acc[i][7] = fmaf(a[i], b1.w, acc[i][7]);
      }
    }
    buf ^= 1;
    j = jn;
    c = cn;
  }

  // ---- epilogue: bias, BatchNorm(eval), activation, residual ----
  const size_t out_base = (size_t)b * L.rows_out * Cout;
  const bool has_bn = P.bn_mean != nullptr;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int n = n0 + tn * 8 + h * 4;
    if (n >= Cout) continue;
    const float4 bi = __ldg(reinterpret_cast<const float4*>(P.bias + n));
    float4 mu = make_float4(0, 0, 0, 0), iv = make_float4(1, 1, 1, 1), of = make_float4(0, 0, 0, 0);
    if (has_bn) {
      mu = __ldg(reinterpret_cast<const float4*>(P.bn_mean + n));
      iv = __ldg(reinterpret_cast<const float4*>(P.bn_inv + n));
      of = __ldg(reinterpret_cast<const float4*>(P.bn_off + n));
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int tau = tau0 + tm + i * NTM;
      if (tau >= valid) continue;
      const size_t o = out_base + (size_t)(tau * P.out_stride + P.out_off) * Cout + n;
      float4 v;
      v.x = acc[i][h * 4 + 0] + bi.x;
      v.y = acc[i][h * 4 + 1] + bi.y;
      v.z = acc[i][h * 4 + 2] + bi.z;
      v.w = acc[i][h * 4 + 3] + bi.w;
      if (has_bn) {
        v.x = (v.x - mu.x) * iv.x + of.x;
        v.y = (v.y - mu.y) * iv.y + of.y;
        v.z = (v.z - mu.z) * iv.z + of.z;
        v.w = (v.w - mu.w) * iv.w + of.w;
      }
      if (L.post_act == 1) {
        v.x = tanhf(v.x); v.y = tanhf(v.y); v.z = tanhf(v.z); v.w = tanhf(v.w);
      } else if (L.post_act == 2) {
        v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
      }
      if (P.resid) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(P.resid + o));
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      *reinterpret_cast<float4*>(P.out + o) = v;
    }
  }
}

template <int TM, int TN>
int launch_cfg(vtts_ctx* ctx, const ConvLaunch& L, cudaStream_t st) {
  using Cfg = ConvCfg<TM, TN>;
  dim3 grid((L.T_rows + TM - 1) / TM, L.B, L.nprob * ((L.Cout + TN - 1) / TN));
  conv1d_nwc_kernel<TM, TN><<<grid, 256, Cfg::SMEM_BYTES, st>>>(L);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  return VTTS_OK;
}

}  // namespace

int vtts_launch_conv(vtts_ctx* ctx, const ConvLaunch& L, cudaStream_t st) {
  if (L.nprob < 1 || L.nprob > 8) return ctx->fail(VTTS_ERR_BAD_ARG, "conv: nprob %d", L.nprob);
  if (L.Cin % KC != 0 || L.Cout % 4 != 0) return ctx->fail(VTTS_ERR_BAD_ARG, "conv: Cin %d / Cout %d unsupported", L.Cin, L.Cout);
  if (L.B < 1 || L.B > 65535 || L.T_rows < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "conv: B %d T %d", L.B, L.T_rows);
  for (int i = 0; i < L.nprob; ++i)
    if ((L.p[i].k - 1) * L.p[i].dil > HALO_MAX || L.p[i].k < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "conv: halo too large");
  if (L.Cout <= 32) return launch_cfg<512, 32>(ctx, L, st);
  if (L.Cout <= 64) return launch_cfg<256, 64>(ctx, L, st);
  return launch_cfg<128, 128>(ctx, L, st);
}

namespace {
__global__ void bn_inv_kernel(const float* __restrict__ scale, const float* __restrict__ var, float* __restrict__ inv, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) inv[i] = scale[i] * rsqrtf(var[i] + 1e-5f);
}
}  // namespace

void vtts_bn_inv(const float* scale, const float* var, float* inv, int n) {
  bn_inv_kernel<<<(n + 255) / 256, 256>>>(scale, var, inv, n);
}
