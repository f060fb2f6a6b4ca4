// C ABI of libviettts_b200.so (see include/viettts_b200.h for the contract and the reference
// interfaces each entry point replaces).
#include <stdarg.h>

#include <algorithm>

#include <dlfcn.h>

#include "stream_common.cuh"

std::string g_vtts_create_error;

int vtts_ctx::fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  err = buf;
  return code;
}

int vtts_ctx::ensure_ws(size_t bytes) {
  vtts_ctx* ctx = this;
  if (bytes <= ws_bytes) return VTTS_OK;
  clear_taps();   // they point into the workspace freed here
  if (ws) {
    VTTS_CUDA(cudaDeviceSynchronize());
    cudaFree(ws);
    ws = nullptr;
    ws_bytes = 0;
  }
  size_t want = bytes + bytes / 8;
  cudaError_t e = cudaMalloc(&ws, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    want = bytes;
    e = cudaMalloc(&ws, want);
  }
  if (e != cudaSuccess) {
    cudaGetLastError();
    ws = nullptr;
    return fail(VTTS_ERR_OOM, "workspace of %zu bytes: %s", bytes, cudaGetErrorString(e));
  }
  ws_bytes = want;
  return VTTS_OK;
}

int vtts_ctx::ensure_staging(size_t host_bytes, size_t dev_bytes) {
  vtts_ctx* ctx = this;
  if (host_bytes > hpin_bytes) {
    if (hpin) cudaFreeHost(hpin);
    hpin = nullptr;
    hpin_bytes = 0;
    VTTS_CUDA(cudaMallocHost(&hpin, host_bytes));
    hpin_bytes = host_bytes;
  }
  if (dev_bytes > dstage_bytes) {
    if (dstage) {
      VTTS_CUDA(cudaDeviceSynchronize());
      cudaFree(dstage);
    }
    dstage = nullptr;
    dstage_bytes = 0;
    cudaError_t e = cudaMalloc(&dstage, dev_bytes);
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(VTTS_ERR_OOM, "device staging of %zu bytes: %s", dev_bytes, cudaGetErrorString(e));
    }
    dstage_bytes = dev_bytes;
  }
  return VTTS_OK;
}

// ---- canonical blob layouts ------------------------------------------------------------------------
const std::vector<TensorSpec>& vtts_hifigan_specs() {
  static std::vector<TensorSpec> s;
  if (!s.empty()) return s;
  s.push_back({"conv_pre.w[7,80,512]", 7 * 80 * 512});
  s.push_back({"conv_pre.b", 512});
  int C = 512;
  for (int i = 0; i < 4; ++i) {
    s.push_back({"ups.w[K,C/2,C]", (int64_t)vc::hg_upk(i) * (C / 2) * C});
    s.push_back({"ups.b", C / 2});
    C /= 2;
  }
  C = 256;
  for (int n = 0; n < 12; ++n) {
    const int k = vc::hg_rbk(n % 3);
    const int ch = 256 >> (n / 3);
    for (int which = 0; which < 2; ++which)
      for (int m = 0; m < 3; ++m) {
        s.push_back({"resblock.conv.w[k,C,C]", (int64_t)k * ch * ch});
        s.push_back({"resblock.conv.b", ch});
      }
  }
  s.push_back({"conv_post.w[7,32,1]", 7 * 32});
  s.push_back({"conv_post.b", 1});
  return s;
}

const std::vector<TensorSpec>& vtts_acoustic_specs() {
  static std::vector<TensorSpec> s;
  if (!s.empty()) return s;
  s.push_back({"embed[256,256]", 256 * 256});
  for (int i = 0; i < 3; ++i) {
    s.push_back({"enc.conv.w[3,256,256]", 3 * 256 * 256});
    s.push_back({"enc.conv.b", 256});
    s.push_back({"enc.bn.scale", 256});
    s.push_back({"enc.bn.offset", 256});
    s.push_back({"enc.bn.mean", 256});
    s.push_back({"enc.bn.var", 256});
  }
  for (int d = 0; d < 2; ++d) {
    s.push_back({"enc.lstm.w[512,1024]", 512 * 1024});
    s.push_back({"enc.lstm.b", 1024});
  }
  s.push_back({"dec.lstm0.w[1280,2048]", 1280 * 2048});
  s.push_back({"dec.lstm0.b", 2048});
  s.push_back({"dec.lstm1.w[1792,2048]", 1792 * 2048});
  s.push_back({"dec.lstm1.b", 2048});
  s.push_back({"proj.w[1024,80]", 1024 * 80});
  s.push_back({"proj.b", 80});
  s.push_back({"prenet.fc1.w[80,256]", 80 * 256});
  s.push_back({"prenet.fc2.w[256,256]", 256 * 256});
  const int dims[6] = {80, 512, 512, 512, 512, 80};
  for (int i = 0; i < 5; ++i) {
    s.push_back({"postnet.conv.w[5,cin,cout]", (int64_t)5 * dims[i] * dims[i + 1]});
    s.push_back({"postnet.conv.b", dims[i + 1]});
    if (i < 4) {
      s.push_back({"postnet.bn.scale", 512});
      s.push_back({"postnet.bn.offset", 512});
      s.push_back({"postnet.bn.mean", 512});
      s.push_back({"postnet.bn.var", 512});
    }
  }
  return s;
}

// duration checkpoint: the TokenEncoder tensors in the acoustic blob's order, then the projection head
const std::vector<TensorSpec>& vtts_duration_specs() {
  static std::vector<TensorSpec> s;
  if (!s.empty()) return s;
  const std::vector<TensorSpec>& a = vtts_acoustic_specs();
  for (int i = 0; i <= aci::ENC_LSTM_B_B; ++i) s.push_back(a[i]);
  s.push_back({"proj.fc1.w[512,256]", 512 * 256});
  s.push_back({"proj.fc1.b", 256});
  s.push_back({"proj.fc2.w[256,1]", 256});
  s.push_back({"proj.fc2.b", 1});
  return s;
}

static int64_t total_floats(const std::vector<TensorSpec>& s) {
  int64_t t = 0;
  for (auto& e : s) t += e.n;
  return t;
}

static std::vector<size_t> spec_floats(const std::vector<TensorSpec>& specs) {
  std::vector<size_t> n;
  for (auto& e : specs) n.push_back((size_t)e.n);
  return n;
}
// floats of one arena of vtts_alloc_tensors
static size_t arena_floats(const std::vector<size_t>& n) {
  size_t total = 0;
  for (size_t x : n) total += (x + 63) & ~size_t(63);
  return total;
}

int vtts_alloc_tensors(vtts_ctx* ctx, const std::vector<size_t>& n, float** store, std::vector<float*>& ptrs) {
  const size_t total = arena_floats(n);
  if (*store) {
    VTTS_CUDA(cudaDeviceSynchronize());
    cudaFree(*store);
    *store = nullptr;
  }
  VTTS_CUDA(cudaMalloc(store, total * sizeof(float)));
  VTTS_CUDA(cudaMemset(*store, 0, total * sizeof(float)));
  ptrs.resize(n.size());
  size_t off = 0;
  for (size_t i = 0; i < n.size(); ++i) {
    ptrs[i] = *store + off;
    off += (n[i] + 63) & ~size_t(63);
  }
  return VTTS_OK;
}

int vtts_pack_convs(vtts_ctx* ctx, ModelWeights& m, const std::vector<PackSpec>& convs) {
  size_t bytes = 0;
  for (auto& c : convs) {
    if (!c.w) return ctx->fail(VTTS_ERR_BAD_ARG, "packing table entry without a weight");
    bytes += vtts_tc_conv_packed_bytes(c.k, c.Cin, c.Cout, c.f16);
  }
  if (m.wpk) cudaFree(m.wpk);
  m.wpk = nullptr;
  VTTS_CUDA(cudaMalloc(&m.wpk, bytes));
  char* cur = (char*)m.wpk;
  m.wpk_t.clear();
  m.tile0.clear();
  for (auto& c : convs) {
    m.tile0.push_back((int)m.wpk_t.size());
    int rc = vtts_tc_pack_conv(ctx, c.w, c.k, c.Cin, c.Cout, c.f16, cur, m.wpk_t);
    if (rc) return rc;
  }
  return VTTS_OK;
}

void vtts_free_weights(ModelWeights& m) {
  cudaFree(m.blob);
  cudaFree(m.derived);
  cudaFree(m.wpk);
  m = ModelWeights();
}

namespace {
// the models of a context, in the bit order of vtts_broadcast_weights
struct ModelSlot {
  ModelWeights vtts_ctx::*w;
  const std::vector<TensorSpec>& (*specs)();
  int (*prepare)(vtts_ctx*);
};
const ModelSlot kModels[3] = {{&vtts_ctx::hg, vtts_hifigan_specs, vtts_hifigan_prepare},
                              {&vtts_ctx::ac, vtts_acoustic_specs, vtts_acoustic_prepare},
                              {&vtts_ctx::du, vtts_duration_specs, vtts_duration_prepare}};

// copies a contiguous blob (host or device) into the slot's tensors, then derives and packs
int load_model(vtts_ctx* ctx, const ModelSlot& ms, const float* blob, int64_t n_floats) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  ModelWeights& m = ctx->*ms.w;
  const std::vector<TensorSpec>& specs = ms.specs();
  m.loaded = false;
  if (!blob) return ctx->fail(VTTS_ERR_BAD_ARG, "load: null blob");
  if (n_floats != total_floats(specs))
    return ctx->fail(VTTS_ERR_BAD_ARG, "load: blob has %lld floats, expected %lld", (long long)n_floats, (long long)total_floats(specs));
  int rc = vtts_alloc_tensors(ctx, spec_floats(specs), &m.blob, m.t);
  if (rc) return rc;
  int64_t src = 0;
  for (size_t i = 0; i < specs.size(); ++i) {
    VTTS_CUDA(cudaMemcpy(m.t[i], blob + src, (size_t)specs[i].n * sizeof(float), cudaMemcpyDefault));
    src += specs[i].n;
  }
  rc = ms.prepare(ctx);
  if (rc) return rc;
  m.loaded = true;
  return VTTS_OK;
}
}  // namespace

// ---- NCCL, bound at run time (the library has no link-time dependency on it: single-GPU users never load it) ----
namespace {
struct NcclApi {
  void* h = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
NcclApi g_nccl;
const char* nccl_bind() {
  if (g_nccl.Broadcast) return nullptr;
  const char* env = getenv("VTTS_NCCL_LIB");
  void* h = nullptr;
  if (env) h = dlopen(env, RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);        // the copy the host process (e.g. torch) already loaded
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) return "libnccl.so.2 not found (set VTTS_NCCL_LIB to its path)";
  g_nccl.h = h;
  g_nccl.Broadcast = (decltype(g_nccl.Broadcast))dlsym(h, "ncclBroadcast");
  g_nccl.GroupStart = (decltype(g_nccl.GroupStart))dlsym(h, "ncclGroupStart");
  g_nccl.GroupEnd = (decltype(g_nccl.GroupEnd))dlsym(h, "ncclGroupEnd");
  g_nccl.GetErrorString = (decltype(g_nccl.GetErrorString))dlsym(h, "ncclGetErrorString");
  if (!g_nccl.Broadcast || !g_nccl.GroupStart || !g_nccl.GroupEnd) {
    g_nccl.Broadcast = nullptr;
    return "libnccl.so.2 lacks ncclBroadcast / ncclGroupStart / ncclGroupEnd";
  }
  return nullptr;
}
}  // namespace

extern "C" {

int vtts_version(void) { return 1; }

int vtts_create(int device, vtts_ctx** out) {
  if (!out) {
    g_vtts_create_error = "vtts_create: out is NULL";
    return VTTS_ERR_BAD_ARG;
  }
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    g_vtts_create_error = std::string("vtts_create: no CUDA device (") + cudaGetErrorString(e) + "); there is no CPU fallback";
    cudaGetLastError();
    return VTTS_ERR_NO_DEVICE;
  }
  if (device < 0 || device >= n) {
    g_vtts_create_error = "vtts_create: device index out of range";
    return VTTS_ERR_BAD_ARG;
  }
  cudaDeviceProp prop;
  if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) {
    g_vtts_create_error = std::string("vtts_create: ") + cudaGetErrorString(e);
    return VTTS_ERR_CUDA;
  }
  if (prop.major != 9 || prop.minor != 0) {
    char buf[256];
    snprintf(buf, sizeof(buf), "vtts_create: device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
    g_vtts_create_error = buf;
    return VTTS_ERR_NO_DEVICE;
  }
  vtts_ctx* ctx = new vtts_ctx();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->cc_major = prop.major;
  ctx->cc_minor = prop.minor;
  ctx->hbm_bytes = prop.totalGlobalMem;
  if ((e = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking)) != cudaSuccess) {
    g_vtts_create_error = std::string("vtts_create: ") + cudaGetErrorString(e);
    delete ctx;
    return VTTS_ERR_CUDA;
  }
  for (int i = 0; i < vtts_ctx::NSTAGE; ++i) {
    cudaEventCreate(&ctx->ev0[i]);
    cudaEventCreate(&ctx->ev1[i]);
  }
  if ((e = cudaEventCreateWithFlags(&ctx->tail, cudaEventDisableTiming)) != cudaSuccess) {
    g_vtts_create_error = std::string("vtts_create: ") + cudaGetErrorString(e);
    delete ctx;
    return VTTS_ERR_CUDA;
  }
  if (cudaMalloc(&ctx->d_err, sizeof(int)) != cudaSuccess || cudaMemset(ctx->d_err, 0, sizeof(int)) != cudaSuccess) {
    g_vtts_create_error = "vtts_create: cannot allocate the error flag";
    delete ctx;
    return VTTS_ERR_CUDA;
  }
  if (cudaMalloc(&ctx->d_tc_sched, 2 * sizeof(int)) != cudaSuccess || cudaMemset(ctx->d_tc_sched, 0, 2 * sizeof(int)) != cudaSuccess) {
    g_vtts_create_error = "vtts_create: cannot allocate the tile scheduler counters";
    delete ctx;
    return VTTS_ERR_CUDA;
  }
  if (cudaMalloc(&ctx->d_tc_dbg, 256 * 16 * sizeof(long long)) != cudaSuccess) {
    g_vtts_create_error = "vtts_create: cannot allocate the profiling counters";
    delete ctx;
    return VTTS_ERR_CUDA;
  }
  cudaMemset(ctx->d_tc_dbg, 0, 256 * 16 * sizeof(long long));
  *out = ctx;
  return VTTS_OK;
}

int vtts_destroy(vtts_ctx* ctx) {
  if (!ctx) return VTTS_OK;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& m : kModels) vtts_free_weights(ctx->*m.w);
  vtts_resample_free(ctx);
  cudaFree(ctx->mel_fb); cudaFree(ctx->mel_lo); cudaFree(ctx->mel_hi); cudaFree(ctx->fft_tw); cudaFree(ctx->hann);
  cudaFree(ctx->ws); cudaFree(ctx->dstage); cudaFree(ctx->d_err); cudaFree(ctx->d_tc_sched); cudaFree(ctx->d_tc_dbg);
  if (ctx->hpin) cudaFreeHost(ctx->hpin);
  for (int i = 0; i < vtts_ctx::NSTAGE; ++i) {
    cudaEventDestroy(ctx->ev0[i]);
    cudaEventDestroy(ctx->ev1[i]);
  }
  if (ctx->tail) cudaEventDestroy(ctx->tail);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  delete ctx;
  return VTTS_OK;
}

const char* vtts_last_error(vtts_ctx* ctx) { return ctx ? ctx->err.c_str() : g_vtts_create_error.c_str(); }

int vtts_device_info(vtts_ctx* ctx, int* sm_count, int* cc_major, int* cc_minor, int64_t* hbm_bytes) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (sm_count) *sm_count = ctx->sm_count;
  if (cc_major) *cc_major = ctx->cc_major;
  if (cc_minor) *cc_minor = ctx->cc_minor;
  if (hbm_bytes) *hbm_bytes = (int64_t)ctx->hbm_bytes;
  return VTTS_OK;
}

int vtts_set_precision(vtts_ctx* ctx, int mode) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (mode != VTTS_PRECISION_FP32 && mode != VTTS_PRECISION_BF16X3 && mode != VTTS_PRECISION_FP16)
    return ctx->fail(VTTS_ERR_BAD_ARG, "set_precision: mode %d", mode);
  ctx->precision = mode;
  return VTTS_OK;
}

int vtts_get_precision(vtts_ctx* ctx) { return ctx ? ctx->precision : VTTS_ERR_BAD_ARG; }

int vtts_debug_substages(vtts_ctx* ctx, int enable, float* ms_out24) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  VTTS_CUDA(cudaDeviceSynchronize());
  if (ms_out24) {
    for (int i = 0; i < vtts_ctx::NSUB; ++i) {
      ms_out24[i] = 0.f;
      if ((i % 8) == 0 || !ctx->sub_set[i] || !ctx->sub_set[i - 1]) continue;
      float ms = 0.f;
      if (cudaEventElapsedTime(&ms, ctx->sub_ev[i - 1], ctx->sub_ev[i]) == cudaSuccess) ms_out24[i] = ms;
    }
  }
  for (int i = 0; i < vtts_ctx::NSUB; ++i) ctx->sub_set[i] = false;
  ctx->sub_on = enable != 0;
  return VTTS_OK;
}

int vtts_debug_tc_stats(vtts_ctx* ctx, int enable, int64_t* host_out_256x16) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());
  if (host_out_256x16) VTTS_CUDA(cudaMemcpy(host_out_256x16, ctx->d_tc_dbg, 256 * 16 * sizeof(long long), cudaMemcpyDeviceToHost));
  VTTS_CUDA(cudaMemset(ctx->d_tc_dbg, 0, 256 * 16 * sizeof(long long)));
  ctx->tc_dbg_on = (enable & 1) != 0;
  if (enable & 0x200) ctx->fuse_pairs = (enable >> 10) & 1;        // bit 9 set: bit 10 selects fused ResBlock pairs (tuning aid)
  if (enable & 0x800) ctx->pair_ts = (enable >> 12) & 3;           // bit 11 set: bits 12..13 select the pair kernel form (vtts_ctx::pair_ts)
  return VTTS_OK;
}

int vtts_debug_conv1d(vtts_ctx* ctx, int precision, const float* x_dev, const float* w_dev, const float* bias_dev,
                      const float* resid_dev, const int32_t* len_dev, int B, int T, int Cin, int Cout, int k, int dil,
                      float pre_slope, float* out_dev) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, nullptr);
  if (precision == VTTS_PRECISION_FP32) {
    ConvLaunch L;
    memset(&L, 0, sizeof(L));
    L.nprob = 1; L.Cin = Cin; L.Cout = Cout; L.B = B; L.T_rows = T; L.rows_out = T; L.len = len_dev; L.len_mul = 1;
    L.pre_mode = pre_slope == 1.0f ? 0 : 1; L.pre_slope = pre_slope; L.post_act = 0;
    L.p[0] = ConvProb{x_dev, nullptr, nullptr, w_dev, bias_dev, resid_dev, nullptr, nullptr, nullptr, out_dev, k, dil, -((k - 1) * dil) / 2, 1, 0};
    int rc = vtts_launch_conv(ctx, L, nullptr);
    if (rc) return rc;
  } else {
    const bool f16 = precision == VTTS_PRECISION_FP16;
    void* wpk = nullptr;
    VTTS_CUDA(cudaMalloc(&wpk, vtts_tc_packed_elems(k, Cin, Cout, f16) * 2));
    int rc = vtts_tc_pack_weights(ctx, w_dev, wpk, k, Cin, Cout, 0, Cout, f16);
    if (rc) { cudaFree(wpk); return rc; }
    TcLaunch TL;
    memset(&TL, 0, sizeof(TL));
    TL.nprob = 1; TL.Cin = Cin; TL.N = Cout; TL.in_ld = Cin; TL.out_ld = Cout; TL.B = B; TL.T_rows = T; TL.rows_out = T;
    TL.len = len_dev; TL.len_mul = 1; TL.pre_mode = pre_slope == 1.0f ? 0 : 1; TL.pre_slope = pre_slope; TL.f16 = f16;
    TL.p[0] = TcProb{x_dev, nullptr, nullptr, wpk, bias_dev, resid_dev, nullptr, nullptr, nullptr, out_dev, k, dil, -((k - 1) * dil) / 2, 1, 0};
    rc = vtts_launch_tc_conv(ctx, TL, nullptr);
    cudaError_t e = cudaDeviceSynchronize();
    cudaFree(wpk);
    if (rc) return rc;
    if (e != cudaSuccess) {
      return ctx->fail(VTTS_ERR_CUDA, "debug_conv1d (tensor path): %s", cudaGetErrorString(e));
    }
  }
  VTTS_CUDA(cudaDeviceSynchronize());
  return VTTS_OK;
}

namespace {
// vtts_debug_conv_dispatch on the temporary buffer `tmp`: BatchNorm inverses of every problem (nprob x Cout floats, the
// first inv_bytes), then the packed tiles of every problem, as the model's load and run code prepare them
int conv_dispatch_on(vtts_ctx* ctx, char* tmp, size_t inv_bytes, int nprob, const float* const* x, const float* const* w,
                     const float* const* bias, const float* const* bn, const float* const* resid, float* const* out,
                     const int32_t* len, int B, int T, int Cin, int Cout, int k, int dil, int post_act) {
  float* inv = reinterpret_cast<float*>(tmp);
  char* cursor = tmp + inv_bytes;
  std::vector<void*> wpk;
  ConvLaunch L;
  memset(&L, 0, sizeof(L));
  for (int p = 0; p < nprob; ++p) {
    int rc = vtts_tc_pack_conv(ctx, w[p], k, Cin, Cout, false, cursor, wpk);
    if (rc) return rc;
    ConvProb& q = L.p[p];
    q.x0 = x[p]; q.w = w[p]; q.bias = bias[p]; q.out = out[p]; q.resid = resid ? resid[p] : nullptr;
    q.k = k; q.dil = dil; q.in_off = -((k - 1) * dil) / 2; q.out_stride = 1;
    if (bn && bn[p]) {
      vtts_bn_inv(bn[p], bn[p] + 3 * Cout, inv + (size_t)p * Cout, Cout);
      q.bn_mean = bn[p] + 2 * Cout; q.bn_inv = inv + (size_t)p * Cout; q.bn_off = bn[p] + Cout;
    }
  }
  VTTS_CUDA(cudaGetLastError());
  L.nprob = nprob; L.Cin = Cin; L.Cout = Cout; L.B = B; L.T_rows = T; L.rows_out = T;
  L.len = len; L.len_mul = 1; L.pre_mode = 0; L.pre_slope = 1.f; L.post_act = post_act;
  return vtts_conv_dispatch(ctx, L, wpk.data(), nullptr);
}
}  // namespace

int vtts_debug_conv_dispatch(vtts_ctx* ctx, int precision, int nprob, const float* const* x, const float* const* w,
                             const float* const* bias, const float* const* bn, const float* const* resid, float* const* out,
                             const int32_t* len, int B, int T, int Cin, int Cout, int k, int dil, int post_act) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (precision < VTTS_PRECISION_FP32 || precision > VTTS_PRECISION_FP16)
    return ctx->fail(VTTS_ERR_BAD_ARG, "debug_conv_dispatch: precision %d", precision);
  if (nprob < 1 || nprob > 8 || !x || !w || !bias || !out)
    return ctx->fail(VTTS_ERR_BAD_ARG, "debug_conv_dispatch: nprob %d (1..8) and the x, w, bias and out arrays are required", nprob);
  for (int p = 0; p < nprob; ++p)
    if (!x[p] || !w[p] || !bias[p] || !out[p]) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_conv_dispatch: null buffer in problem %d", p);
  if (B < 1 || T < 1 || Cin < 16 || Cin % 16 != 0 || Cout < 4 || Cout % 4 != 0 || k < 1 || dil < 1 || post_act < 0 || post_act > 2)
    return ctx->fail(VTTS_ERR_BAD_ARG, "debug_conv_dispatch: B=%d T=%d Cin=%d Cout=%d k=%d dil=%d post_act=%d", B, T, Cin, Cout, k, dil,
                     post_act);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, nullptr);
  const size_t inv_bytes = ((size_t)nprob * Cout * sizeof(float) + 255) & ~size_t(255);
  char* tmp = nullptr;
  VTTS_CUDA(cudaMalloc(&tmp, inv_bytes + nprob * vtts_tc_conv_packed_bytes(k, Cin, Cout, false)));
  const int saved = ctx->precision;
  ctx->precision = precision;
  int rc = conv_dispatch_on(ctx, tmp, inv_bytes, nprob, x, w, bias, bn, resid, out, len, B, T, Cin, Cout, k, dil, post_act);
  ctx->precision = saved;
  const cudaError_t e = cudaDeviceSynchronize();
  cudaFree(tmp);
  if (rc) return rc;
  if (e != cudaSuccess) return ctx->fail(VTTS_ERR_CUDA, "debug_conv_dispatch: %s", cudaGetErrorString(e));
  return VTTS_OK;
}

int vtts_debug_pair(vtts_ctx* ctx, const float* x_dev, const float* w1_dev, const float* b1_dev, const float* w2_dev,
                    const float* b2_dev, const int32_t* len_dev, int B, int T, int C, int k, int dil, float slope, float* out_dev) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, nullptr);
  const bool f16 = ctx->precision == VTTS_PRECISION_FP16;   // the generator's operand format of the context's mode
  void* wpk = nullptr;
  const size_t bytes = vtts_tc_packed_elems(k, C, C, f16) * 2;
  VTTS_CUDA(cudaMalloc(&wpk, 2 * bytes));
  int rc = vtts_tc_pack_weights(ctx, w1_dev, wpk, k, C, C, 0, C, f16);
  if (!rc) rc = vtts_tc_pack_weights(ctx, w2_dev, (char*)wpk + bytes, k, C, C, 0, C, f16);
  if (rc) { cudaFree(wpk); return rc; }
  TcPairLaunch PL;
  memset(&PL, 0, sizeof(PL));
  PL.nprob = 1; PL.N = C; PL.B = B; PL.T_rows = T; PL.len = len_dev; PL.len_mul = 1; PL.slope = slope; PL.f16 = f16;
  PL.p[0] = TcPairProb{x_dev, wpk, (char*)wpk + bytes, b1_dev, b2_dev, out_dev, k, dil};
  rc = vtts_launch_tc_pair(ctx, PL, nullptr);
  cudaError_t e = cudaDeviceSynchronize();
  cudaFree(wpk);
  if (rc) return rc;
  if (e != cudaSuccess) return ctx->fail(VTTS_ERR_CUDA, "debug_pair: %s", cudaGetErrorString(e));
  return VTTS_OK;
}

int64_t vtts_hifigan_blob_floats(void) { return total_floats(vtts_hifigan_specs()); }
int64_t vtts_acoustic_blob_floats(void) { return total_floats(vtts_acoustic_specs()); }
int64_t vtts_duration_blob_floats(void) { return total_floats(vtts_duration_specs()); }

int vtts_load_hifigan(vtts_ctx* ctx, const float* blob, int64_t n_floats) { return load_model(ctx, kModels[0], blob, n_floats); }
int vtts_load_acoustic(vtts_ctx* ctx, const float* blob, int64_t n_floats) { return load_model(ctx, kModels[1], blob, n_floats); }
int vtts_load_duration(vtts_ctx* ctx, const float* blob, int64_t n_floats) { return load_model(ctx, kModels[2], blob, n_floats); }

// One start-up broadcast of the packed weights from `root` (SURVEY.md 8e: the only collective of the path).
int vtts_broadcast_weights(vtts_ctx* ctx, void* nccl_comm, int root, int is_root, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!nccl_comm) return ctx->fail(VTTS_ERR_BAD_ARG, "broadcast_weights: null communicator");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  if (const char* e = nccl_bind()) return ctx->fail(VTTS_ERR_NCCL, "broadcast_weights: %s", e);
  cudaStream_t st = (cudaStream_t)stream;
  auto nccl_ck = [&](int r, const char* what) -> int {
    if (r == 0) return VTTS_OK;
    return ctx->fail(VTTS_ERR_NCCL, "broadcast_weights: %s -> %s", what, g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "nccl error");
  };
  // which models travel: bit 0 hifigan, 1 acoustic, 2 duration (decided by the root's loaded state)
  int32_t* d_flags = nullptr;
  VTTS_CUDA(cudaMalloc(&d_flags, sizeof(int32_t)));
  int32_t flags = 0;
  for (int i = 0; i < 3 && is_root; ++i) flags |= (ctx->*kModels[i].w).loaded ? 1 << i : 0;
  VTTS_CUDA(cudaMemcpyAsync(d_flags, &flags, sizeof(flags), cudaMemcpyHostToDevice, st));
  int rc = nccl_ck(g_nccl.Broadcast(d_flags, d_flags, 1, /*ncclInt32*/ 2, root, nccl_comm, st), "ncclBroadcast(flags)");
  if (rc) { cudaFree(d_flags); return rc; }
  VTTS_CUDA(cudaMemcpyAsync(&flags, d_flags, sizeof(flags), cudaMemcpyDeviceToHost, st));
  VTTS_CUDA(cudaStreamSynchronize(st));
  cudaFree(d_flags);
  if (is_root && flags == 0) return ctx->fail(VTTS_ERR_NOT_LOADED, "broadcast_weights: the root context has no weights loaded");
  if (!is_root)
    for (int i = 0; i < 3; ++i)
      if (flags & (1 << i)) {
        ModelWeights& m = ctx->*kModels[i].w;
        m.loaded = false;
        rc = vtts_alloc_tensors(ctx, spec_floats(kModels[i].specs()), &m.blob, m.t);
        if (rc) return rc;
      }
  // the arenas have the same layout on every rank (it only depends on the tensor specs): ONE grouped broadcast
  rc = nccl_ck(g_nccl.GroupStart(), "ncclGroupStart");
  if (rc) return rc;
  for (int i = 0; i < 3; ++i)
    if (flags & (1 << i)) {
      float* blob = (ctx->*kModels[i].w).blob;
      rc = nccl_ck(g_nccl.Broadcast(blob, blob, arena_floats(spec_floats(kModels[i].specs())), /*ncclFloat32*/ 7, root, nccl_comm, st),
                   "ncclBroadcast(weights)");
      if (rc) { g_nccl.GroupEnd(); return rc; }
    }
  rc = nccl_ck(g_nccl.GroupEnd(), "ncclGroupEnd");
  if (rc) return rc;
  VTTS_CUDA(cudaStreamSynchronize(st));
  if (!is_root)
    for (int i = 0; i < 3; ++i)
      if (flags & (1 << i)) {
        rc = kModels[i].prepare(ctx);
        if (rc) return rc;
        (ctx->*kModels[i].w).loaded = true;
      }
  return VTTS_OK;
}

int vtts_load_mel_filterbank(vtts_ctx* ctx, const float* fb, int n_mels, int n_bins) {
  if (!ctx || !fb) return VTTS_ERR_BAD_ARG;
  if (n_mels != vc::MEL || n_bins != vc::NBINS) return ctx->fail(VTTS_ERR_BAD_ARG, "mel filterbank must be [80][513], got [%d][%d]", n_mels, n_bins);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  ctx->mel_loaded = false;
  if (!ctx->mel_fb) VTTS_CUDA(cudaMalloc(&ctx->mel_fb, (size_t)vc::MEL * vc::NBINS * sizeof(float)));
  VTTS_CUDA(cudaMemcpy(ctx->mel_fb, fb, (size_t)vc::MEL * vc::NBINS * sizeof(float), cudaMemcpyDefault));
  int rc = vtts_melspec_prepare(ctx);
  if (rc) return rc;
  ctx->mel_loaded = true;
  return VTTS_OK;
}

static void stage_begin(vtts_ctx* ctx, int stage, cudaStream_t st) {
  cudaEventRecord(ctx->ev0[stage], st);
  ctx->ev_stream[stage] = st;
}
static void stage_end(vtts_ctx* ctx, int stage, cudaStream_t st) {
  cudaEventRecord(ctx->ev1[stage], st);
  ctx->ev_valid[stage] = true;
}

int vtts_hifigan_forward(vtts_ctx* ctx, const float* mel_dev, const int32_t* n_frames_dev, int B, int T, float* wav_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!mel_dev || !wav_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "hifigan_forward: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  stage_begin(ctx, 0, st);
  int rc = vtts_hifigan_run(ctx, mel_dev, n_frames_dev, B, T, wav_dev, st);
  stage_end(ctx, 0, st);
  return rc;
}

int vtts_acoustic_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev, const float* dur_frames_dev,
                          const int32_t* n_frames_dev, const uint8_t* keep_mask_dev, int dropout_mode, uint64_t seed, int B, int L,
                          int N, float* mel_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens_dev || !dur_frames_dev || !mel_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_forward: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  // the acoustic workspace lives after the hifigan one is released: both share ctx->ws, so a
  // synthesize call sizes it for the larger of the two (see vtts_synthesize_host)
  int rc = ctx->ensure_ws(vtts_acoustic_ws_bytes(B, L, N));
  if (rc) return rc;
  stage_begin(ctx, 1, st);
  rc = vtts_acoustic_run(ctx, tokens_dev, lengths_dev, dur_frames_dev, n_frames_dev, keep_mask_dev, dropout_mode, seed, B, L, N,
                         mel_dev, st);
  stage_end(ctx, 1, st);
  return rc;
}

int vtts_acoustic_teacher_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev, const float* dur_frames_dev,
                                  const int32_t* n_frames_dev, const float* mels_in_dev, const uint8_t* keep_mask_dev,
                                  const uint8_t* zone_mask_dev, int dropout_mode, uint64_t seed, int B, int L, int N,
                                  float* mel1_dev_or_null, float* mel2_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens_dev || !dur_frames_dev || !mels_in_dev || !mel2_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "acoustic_teacher_forward: null pointer");
  int rc = vtts_teacher_mode_check(ctx, dropout_mode, B, N);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  rc = ctx->ensure_ws(vtts_acoustic_teacher_ws_bytes(B, L, N));
  if (rc) return rc;
  stage_begin(ctx, 1, st);
  rc = vtts_acoustic_teacher_run(ctx, tokens_dev, lengths_dev, dur_frames_dev, n_frames_dev, mels_in_dev, keep_mask_dev, zone_mask_dev,
                                 dropout_mode, seed, B, L, N, mel1_dev_or_null, mel2_dev, st);
  stage_end(ctx, 1, st);
  return rc;
}

int vtts_duration_forward(vtts_ctx* ctx, const int32_t* tokens_dev, const int32_t* lengths_dev, int B, int L, float* dur_sec_dev,
                          void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens_dev || !dur_sec_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "duration_forward: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ctx->ensure_ws(vtts_duration_ws_bytes(B, L));
  if (rc) return rc;
  stage_begin(ctx, 3, st);
  rc = vtts_duration_run(ctx, tokens_dev, lengths_dev, B, L, dur_sec_dev, st);
  stage_end(ctx, 3, st);
  return rc;
}

int vtts_melspec(vtts_ctx* ctx, const float* wav_dev, int B, int S, float* mel_dev, void* stream) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav_dev || !mel_dev) return ctx->fail(VTTS_ERR_BAD_ARG, "melspec: null pointer");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const CallOrder order(ctx, stream);
  cudaStream_t st = (cudaStream_t)stream;
  stage_begin(ctx, 2, st);
  int rc = vtts_melspec_run(ctx, wav_dev, B, S, mel_dev, st);
  stage_end(ctx, 2, st);
  return rc;
}

int vtts_debug_read(vtts_ctx* ctx, const char* name, float* host_out, int64_t n_floats) {
  if (!ctx || !name || !host_out) return VTTS_ERR_BAD_ARG;
  const float* src = nullptr;
  int64_t n = 0;
  if (!strcmp(name, "enc")) { src = ctx->tap_enc; n = ctx->tap_enc_n; }
  else if (!strcmp(name, "cond")) { src = ctx->tap_cond; n = ctx->tap_cond_n; }
  else if (!strcmp(name, "mel_pre")) { src = ctx->tap_melpre; n = ctx->tap_melpre_n; }
  else if (!strcmp(name, "dec_in")) { src = ctx->tap_decin; n = ctx->tap_decin_n; }
  else if (!strcmp(name, "dec_out")) { src = ctx->tap_decout; n = ctx->tap_decout_n; }
  else if (!strcmp(name, "dur_hidden")) { src = ctx->tap_durhid; n = ctx->tap_durhid_n; }
  else return ctx->fail(VTTS_ERR_BAD_ARG, "debug_read: unknown tap %s", name);
  if (!src)
    return ctx->fail(VTTS_ERR_BAD_ARG, "debug_read: tap %s is not set (the last call did not produce it, or the workspace it pointed into "
                     "was freed)", name);
  if (n_floats != n) return ctx->fail(VTTS_ERR_BAD_ARG, "debug_read: tap %s has %lld floats, asked %lld", name, (long long)n, (long long)n_floats);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());
  VTTS_CUDA(cudaMemcpy(host_out, src, (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  return VTTS_OK;
}

// ---- host-buffer entry points (staged through HostStage) ------------------------------------------
namespace {
// true if `p` is page-locked host memory known to CUDA (cudaHostAlloc / cudaHostRegister / torch pin_memory):
// results can then be copied D2H straight into the caller's buffer instead of through the context's staging area
bool is_pinned_host(const void* p) {
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeHost;
}
}  // namespace

int vtts_mel2wave_host(vtts_ctx* ctx, const float* mel, const int32_t* n_frames, int B, int T, float* wav) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!mel || !wav || B < 1 || T < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "mel2wave_host: bad argument");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t wav_b = (size_t)B * T * vc::HOP * 4;
  HostStage hs(ctx);
  const size_t o_mel = hs.in(mel, (size_t)B * T * vc::MEL * 4), o_nf = hs.in(n_frames, (size_t)B * 4), o_wav = hs.out(wav_b);
  int rc = hs.upload();
  if (!rc)
    rc = vtts_hifigan_forward(ctx, hs.dev<const float>(o_mel), n_frames ? hs.dev<const int32_t>(o_nf) : nullptr, B, T, hs.dev<float>(o_wav),
                              hs.st);
  if (!rc) rc = hs.fetch(o_wav, wav, wav_b, is_pinned_host(wav));
  return rc ? rc : hs.finish();
}

static int synth_common(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur, const int32_t* n_frames,
                        const uint8_t* keep, int mode, uint64_t seed, int B, int L, int N, float* mel_out, float* wav_out,
                        const int32_t* n_frames_voc = nullptr) {
  // n_frames_voc: optional per-row frame counts for the generator only (text2mel trims the trailing silence from the
  // mel AFTER the postnet, text2mel.py:99-102); default = n_frames
  if (!tokens || !dur || B < 1 || L < 1 || N < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "predict_mel/synthesize_host: bad argument");
  if (mode == VTTS_DROPOUT_MASK && !keep) return ctx->fail(VTTS_ERR_BAD_ARG, "dropout_mode MASK needs keep_mask");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t nf_b = (size_t)B * 4;
  const size_t keep_b = mode == VTTS_DROPOUT_MASK ? (size_t)B * N * 2 * vc::PRENET : 0;
  const size_t mel_b = (size_t)B * N * vc::MEL * 4, wav_b = wav_out ? (size_t)B * N * vc::HOP * 4 : 0;
  HostStage hs(ctx);
  const size_t o_tok = hs.in(tokens, (size_t)B * L * 4), o_len = hs.in(lengths, nf_b), o_dur = hs.in(dur, (size_t)B * L * 4);
  const size_t o_nf = hs.in(n_frames, nf_b), o_keep = hs.in(keep_b ? keep : nullptr, keep_b), o_nfv = hs.in(n_frames_voc, n_frames_voc ? nf_b : 0);
  const size_t o_mel = hs.out(mel_b), o_wav = hs.out(wav_b);
  int rc = hs.upload();
  if (rc) return rc;
  const int32_t* d_nf = n_frames ? hs.dev<const int32_t>(o_nf) : nullptr;
  rc = vtts_acoustic_forward(ctx, hs.dev<const int32_t>(o_tok), lengths ? hs.dev<const int32_t>(o_len) : nullptr, hs.dev<const float>(o_dur),
                             d_nf, keep_b ? hs.dev<const uint8_t>(o_keep) : nullptr, mode, seed, B, L, N, hs.dev<float>(o_mel), hs.st);
  if (!rc && mel_out) rc = hs.fetch(o_mel, mel_out, mel_b, is_pinned_host(mel_out));
  if (rc) return rc;
  if (wav_out) {
    // the hifigan workspace replaces the acoustic one: its kernels are stream-ordered after the acoustic ones,
    // but growing the workspace frees memory -> make sure `mel` (in dstage) is complete first
    size_t need = vtts_hifigan_ws_bytes(B, N);
    if (need > ctx->ws_bytes) VTTS_CUDA(cudaStreamSynchronize(hs.st));
    rc = vtts_hifigan_forward(ctx, hs.dev<const float>(o_mel), n_frames_voc ? hs.dev<const int32_t>(o_nfv) : d_nf, B, N, hs.dev<float>(o_wav),
                              hs.st);
    if (!rc) rc = hs.fetch(o_wav, wav_out, wav_b, is_pinned_host(wav_out));
    if (rc) return rc;
  }
  return hs.finish();
}

int vtts_predict_mel_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur_frames,
                          const int32_t* n_frames, const uint8_t* keep_mask, int dropout_mode, uint64_t seed, int B, int L, int N,
                          float* mel) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!mel) return ctx->fail(VTTS_ERR_BAD_ARG, "predict_mel_host: null output");
  return synth_common(ctx, tokens, lengths, dur_frames, n_frames, keep_mask, dropout_mode, seed, B, L, N, mel, nullptr);
}

int vtts_synthesize_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, const float* dur_frames,
                         const int32_t* n_frames, const uint8_t* keep_mask, int dropout_mode, uint64_t seed, int B, int L, int N,
                         float* mel_out_or_null, float* wav) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav) return ctx->fail(VTTS_ERR_BAD_ARG, "synthesize_host: null output");
  return synth_common(ctx, tokens, lengths, dur_frames, n_frames, keep_mask, dropout_mode, seed, B, L, N, mel_out_or_null, wav);
}

int vtts_predict_duration_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float* dur_sec) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens || !dur_sec || B < 1 || L < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "predict_duration_host: bad argument");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t dur_b = (size_t)B * L * 4;
  HostStage hs(ctx);
  const size_t o_tok = hs.in(tokens, (size_t)B * L * 4), o_len = hs.in(lengths, (size_t)B * 4), o_dur = hs.out(dur_b);
  int rc = hs.upload();
  // launches of at most 128 rows (a row's durations do not depend on the rows launched with it), one round trip
  for (size_t b0 = 0; b0 < (size_t)B && !rc; b0 += vc::LAUNCH_ROWS)
    rc = vtts_duration_forward(ctx, hs.dev<const int32_t>(o_tok) + b0 * L, lengths ? hs.dev<const int32_t>(o_len) + b0 : nullptr,
                               std::min(B - (int)b0, vc::LAUNCH_ROWS), L, hs.dev<float>(o_dur) + b0 * L, hs.st);
  if (!rc) rc = hs.fetch(o_dur, dur_sec, dur_b);
  return rc ? rc : hs.finish();
}

namespace {
__global__ void pcm16_to_float_kernel(const int16_t* __restrict__ in, float* __restrict__ out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = (float)in[i] * (1.0f / 32768.0f);                      // gta.py:32  wavs.astype(float32) / 2**15
}
}  // namespace

// forward_fn_ of vietTTS/nat/gta.py:28-41: int16 waveform -> MelFilter -> ground-truth mel shifted by one frame ->
// AcousticModel.__call__ (teacher forced, zoneout) -> mel2_hat.
int vtts_gta_host(vtts_ctx* ctx, const int16_t* wav_i16, const int32_t* wav_lengths, const int32_t* tokens, const int32_t* lengths,
                  const float* dur_sec, const uint8_t* keep_mask, const uint8_t* zone_mask, int dropout_mode, uint64_t seed, int B,
                  int L, int S, float* mel_gt_out_or_null, float* mel2_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav_i16 || !tokens || !dur_sec || !mel2_out || B < 1 || L < 1 || S < 512 || S % vc::HOP)
    return ctx->fail(VTTS_ERR_BAD_ARG, "gta_host: bad argument (S must be a multiple of %d, >= 512)", vc::HOP);
  if (dropout_mode == VTTS_DROPOUT_MASK && (!keep_mask || !zone_mask)) return ctx->fail(VTTS_ERR_BAD_ARG, "gta_host: MASK mode needs both masks");
  if (!ctx->mel_loaded) return ctx->fail(VTTS_ERR_NOT_LOADED, "gta_host: mel filterbank not loaded");
  const int N = S / vc::HOP;
  int rc = vtts_teacher_mode_check(ctx, dropout_mode, B, N);
  if (rc) return rc;
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::vector<float> dur((size_t)B * L);                              // gta.py:37  durations * sample_rate / (n_fft // 4), float32
  for (size_t i = 0; i < dur.size(); ++i) dur[i] = (dur_sec[i] * 16000.0f) / 256.0f;
  std::vector<int32_t> nf(B);                                         // gta.py:74  l = wav_length // hop
  for (int b = 0; b < B; ++b) {
    int n = wav_lengths ? wav_lengths[b] / vc::HOP : N;
    nf[b] = n < 1 ? 1 : (n > N ? N : n);
  }
  const size_t keep_b = dropout_mode == VTTS_DROPOUT_MASK ? (size_t)B * N * 2 * vc::PRENET : 0;
  const size_t zone_b = dropout_mode == VTTS_DROPOUT_MASK ? (size_t)B * N * 4 * vc::DEC_H : 0;
  const size_t mel_b = (size_t)B * N * vc::MEL * 4;
  HostStage hs(ctx);
  const size_t o_wav = hs.in(wav_i16, (size_t)B * S * 2), o_tok = hs.in(tokens, (size_t)B * L * 4), o_len = hs.in(lengths, (size_t)B * 4);
  const size_t o_dur = hs.in(dur.data(), dur.size() * 4), o_nf = hs.in(nf.data(), (size_t)B * 4);
  const size_t o_keep = hs.in(keep_b ? keep_mask : nullptr, keep_b), o_zone = hs.in(zone_b ? zone_mask : nullptr, zone_b);
  const size_t o_gt = hs.out(mel_b), o_out = hs.out(mel_b);
  const size_t o_wavf = hs.scratch((size_t)B * S * 4), o_in = hs.scratch(mel_b);
  rc = hs.upload();
  if (rc) return rc;
  cudaStream_t st = hs.st;
  pcm16_to_float_kernel<<<ctx->sm_count * 4, 256, 0, st>>>(hs.dev<const int16_t>(o_wav), hs.dev<float>(o_wavf), (size_t)B * S);
  ctx->launches++;
  VTTS_CUDA(cudaGetLastError());
  rc = vtts_melspec(ctx, hs.dev<const float>(o_wavf), B, S, hs.dev<float>(o_gt), st);
  if (rc) return rc;
  // inp_mels = concat(zeros[B,1,D], mels[:, :-1]) (gta.py:34-36)
  char* d_in = hs.dev<char>(o_in);
  VTTS_CUDA(cudaMemsetAsync(d_in, 0, mel_b, st));
  if (N > 1)
    VTTS_CUDA(cudaMemcpy2DAsync(d_in + vc::MEL * 4, (size_t)N * vc::MEL * 4, hs.dev<char>(o_gt), (size_t)N * vc::MEL * 4,
                                (size_t)(N - 1) * vc::MEL * 4, B, cudaMemcpyDeviceToDevice, st));
  rc = vtts_acoustic_teacher_forward(ctx, hs.dev<const int32_t>(o_tok), lengths ? hs.dev<const int32_t>(o_len) : nullptr,
                                     hs.dev<const float>(o_dur), hs.dev<const int32_t>(o_nf), hs.dev<const float>(o_in),
                                     keep_b ? hs.dev<const uint8_t>(o_keep) : nullptr, zone_b ? hs.dev<const uint8_t>(o_zone) : nullptr,
                                     dropout_mode, seed, B, L, N, nullptr, hs.dev<float>(o_out), st);
  if (!rc && mel_gt_out_or_null) rc = hs.fetch(o_gt, mel_gt_out_or_null, mel_b);
  if (!rc) rc = hs.fetch(o_out, mel2_out, mel_b);
  return rc ? rc : hs.finish();
}

// text2mel (vietTTS/nat/text2mel.py:85-103) + mel2wave for a batch of token rows, in one call:
//   predict_duration -> [host: silence clip, word-end zeroing, seconds -> frames, n_frames, trailing-silence trim]
//   -> AcousticModel.inference -> Generator.  The one unavoidable host round trip is the [B,L] duration matrix:
//   the frame count N (every later grid size) depends on it.
int vtts_tts_plan(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float silence_duration, float* dur_sec_out,
                  float* dur_frames_out, int32_t* n_frames_out, int32_t* n_emit_out) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens || !dur_frames_out || !n_frames_out || !n_emit_out || B < 1 || L < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "tts_plan: bad argument");
  for (int b = 0; b < B; ++b) {
    const int len = lengths ? lengths[b] : L;
    if (len < 1 || len > L) return ctx->fail(VTTS_ERR_BAD_ARG, "tts_plan: lengths[%d]=%d outside [1,%d]", b, len, L);
  }
  VTTS_CUDA(cudaSetDevice(ctx->device));
  std::vector<float> sec((size_t)B * L);
  int rc = vtts_predict_duration_host(ctx, tokens, lengths, B, L, sec.data());
  if (rc) return rc;
  float* frames = dur_frames_out;
  for (int b = 0; b < B; ++b) {
    const int len = lengths ? lengths[b] : L;
    double total = 0.0;
    for (int l = 0; l < L; ++l) {
      float d = l < len ? sec[(size_t)b * L + l] : 0.f;
      const int tok = tokens[(size_t)b * L + l];
      if (l < len && tok == vc::SIL_INDEX && d < silence_duration) d = silence_duration;   // text2mel.py:88-94
      if (tok == vc::WORD_END_INDEX) d = 0.f;                                              // text2mel.py:95-97
      sec[(size_t)b * L + l] = d;
      const float f = (d * 16000.0f) / 256.0f;                                             // text2mel.py:78 (float32)
      frames[(size_t)b * L + l] = f;
      total += f;
    }
    const int n = (int)(float)total;                                                       // text2mel.py:79
    int trim = 0;
    if (tokens[(size_t)b * L + len - 1] == vc::SIL_INDEX)                                  // text2mel.py:99-102
      trim = (int)((double)sec[(size_t)b * L + len - 1] * 16000.0 / 256.0);
    n_frames_out[b] = n;
    n_emit_out[b] = n - trim > 0 ? n - trim : 0;
  }
  if (dur_sec_out) memcpy(dur_sec_out, sec.data(), sec.size() * sizeof(float));
  return VTTS_OK;
}

int vtts_tts_host(vtts_ctx* ctx, const int32_t* tokens, const int32_t* lengths, int B, int L, float silence_duration,
                  int dropout_mode, uint64_t seed, int max_frames, float* dur_sec_out, int32_t* n_frames_out,
                  int32_t* n_max_out, float* wav) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!tokens || !n_frames_out || !n_max_out || !wav || B < 1 || L < 1 || max_frames < 1)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_host: bad argument");
  if (dropout_mode != VTTS_DROPOUT_OFF && dropout_mode != VTTS_DROPOUT_SEED && dropout_mode != VTTS_DROPOUT_REFERENCE)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_host: dropout_mode must be OFF, SEED or REFERENCE (the frame count is not known to the caller)");
  std::vector<float> frames((size_t)B * L);
  std::vector<int32_t> nf_ac(B), nf_voc(B);
  int rc = vtts_tts_plan(ctx, tokens, lengths, B, L, silence_duration, dur_sec_out, frames.data(), nf_ac.data(), nf_voc.data());
  if (rc) return rc;
  int n_max = 0;
  for (int b = 0; b < B; ++b) n_max = std::max(n_max, nf_ac[b]);
  memcpy(n_frames_out, nf_voc.data(), (size_t)B * sizeof(int32_t));
  *n_max_out = n_max;
  if (n_max < 1) return ctx->fail(VTTS_ERR_BAD_ARG, "tts_host: predicted durations sum to less than one frame");
  if (n_max > max_frames)
    return ctx->fail(VTTS_ERR_BAD_ARG, "tts_host: needs %d frames, caller buffer holds %d (n_max_out is set: retry with that size)", n_max, max_frames);
  return synth_common(ctx, tokens, lengths, frames.data(), nf_ac.data(), nullptr, dropout_mode, seed, B, L, n_max, nullptr, wav,
                      nf_voc.data());
}

int vtts_melspec_host(vtts_ctx* ctx, const float* wav, int B, int S, float* mel) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!wav || !mel || B < 1 || S < 512 || S % vc::HOP) return ctx->fail(VTTS_ERR_BAD_ARG, "melspec_host: bad argument");
  VTTS_CUDA(cudaSetDevice(ctx->device));
  const size_t mel_b = (size_t)B * (S / vc::HOP) * vc::MEL * 4;
  HostStage hs(ctx);
  const size_t o_wav = hs.in(wav, (size_t)B * S * 4), o_mel = hs.out(mel_b);
  int rc = hs.upload();
  if (!rc) rc = vtts_melspec(ctx, hs.dev<const float>(o_wav), B, S, hs.dev<float>(o_mel), hs.st);
  if (!rc) rc = hs.fetch(o_mel, mel, mel_b);
  return rc ? rc : hs.finish();
}

int64_t vtts_launch_count(vtts_ctx* ctx) { return ctx ? ctx->launches : 0; }

int vtts_last_stage_ms(vtts_ctx* ctx, int stage, float* ms) {
  if (!ctx || !ms || stage < 0 || stage >= vtts_ctx::NSTAGE) return VTTS_ERR_BAD_ARG;
  if (!ctx->ev_valid[stage]) return ctx->fail(VTTS_ERR_BAD_ARG, "last_stage_ms: stage %d has not run", stage);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaEventSynchronize(ctx->ev1[stage]));
  VTTS_CUDA(cudaEventElapsedTime(ms, ctx->ev0[stage], ctx->ev1[stage]));
  return VTTS_OK;
}

}  // extern "C"
