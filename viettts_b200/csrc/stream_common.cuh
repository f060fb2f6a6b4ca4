// Host-side pieces shared by the per-slot streams (resample, denoise, pitch, loudness, vocoder) and the *_host entry
// points: the slot protocol of a push, the device memory of a stream, and the staging of host buffers.
#pragma once
#include <memory>

#include "vtts_internal.cuh"

// ---- slot protocol -----------------------------------------------------------------------------------------------
// A push carries per slot n_new[s] in [0, F] new inputs and flags[s] (bit0 BEGIN, bit1 END).  A slot with neither is
// idle; any other push to a slot needs BEGIN unless the slot is open (BEGIN seen, END not yet).
struct SlotState {
  // per slot: inputs received since BEGIN, outputs emitted, open, inputs of the last push whose window tail has not
  // moved to the front yet
  std::vector<long long> P, E;
  std::vector<int> open, pending;

  explicit SlotState(int S) : P(S, 0), E(S, 0), open(S, 0), pending(S, 0) {}

  static bool active(const int32_t* n_new, const uint8_t* flags, int s) { return n_new[s] > 0 || flags[s] != 0; }

  // the shared checks of entry point `who`, slot by slot; extra(s) runs the stream's own checks of each non-idle slot
  // after them and returns non-zero to reject the push
  template <class Extra>
  int check(vtts_ctx* ctx, const char* who, int F, const int32_t* n_new, const uint8_t* flags, Extra&& extra) const {
    for (int s = 0; s < (int)open.size(); ++s) {
      if (n_new[s] < 0 || n_new[s] > F) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: n_new[%d]=%d outside [0, %d]", who, s, n_new[s], F);
      if (flags[s] & ~3u) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: flags[%d]=%u (bit0 BEGIN, bit1 END)", who, s, flags[s]);
      if (!active(n_new, flags, s)) continue;
      if (!(flags[s] & 1) && !open[s])
        return ctx->fail(VTTS_ERR_BAD_ARG, "%s: slot %d is not open (push BEGIN first, also after END)", who, s);
      const int rc = extra(s);
      if (rc) return rc;
    }
    return VTTS_OK;
  }
  int check(vtts_ctx* ctx, const char* who, int F, const int32_t* n_new, const uint8_t* flags) const {
    return check(ctx, who, F, n_new, flags, [](int) { return VTTS_OK; });
  }

  // the window step table of vtts_stream_window_prep: {inputs of the previous push, new inputs} per slot
  void prep(const int32_t* n_new, const uint8_t* flags, int* tbl) const {
    for (int s = 0; s < (int)open.size(); ++s) {
      const bool act = active(n_new, flags, s);
      tbl[2 * s] = act && !(flags[s] & 1) ? pending[s] : 0;
      tbl[2 * s + 1] = act ? n_new[s] : 0;
    }
  }

  // after the launches: the slots this push touched take their new input count and E1[s] outputs
  void commit(const int32_t* n_new, const uint8_t* flags, const long long* E1) {
    for (int s = 0; s < (int)open.size(); ++s) {
      if (!active(n_new, flags, s)) continue;
      const bool begin = flags[s] & 1, end = flags[s] & 2;
      P[s] = (begin ? 0 : P[s]) + n_new[s];
      E[s] = E1[s];
      open[s] = !end;
      pending[s] = end ? 0 : n_new[s];
    }
  }
};

// ---- stream memory -----------------------------------------------------------------------------------------------
// What every stream handle holds: its context, one device allocation (freed with the handle) and the slot state.
struct StreamBase {
  vtts_ctx* ctx;
  int S, F;                     // slots, largest chunk
  void* mem = nullptr;
  SlotState slots;
  StreamBase(vtts_ctx* c, int s, int f) : ctx(c), S(s), F(f), slots(s) {}
  ~StreamBase() { cudaFree(mem); }
};

// `carve(Arena&)` hands out the stream's buffers; it runs once to measure and once more on the zero-filled allocation
template <class Carve>
int stream_alloc(vtts_ctx* ctx, const char* who, StreamBase& sb, Carve&& carve) {
  Arena m(nullptr, 0, true);
  carve(m);
  cudaError_t e = cudaMalloc(&sb.mem, m.off);
  if (e == cudaSuccess) e = cudaMemset(sb.mem, 0, m.off);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return ctx->fail(e == cudaErrorMemoryAllocation ? VTTS_ERR_OOM : VTTS_ERR_CUDA, "%s: %zu bytes: %s", who, m.off, cudaGetErrorString(e));
  }
  Arena a(sb.mem, m.off, false);
  carve(a);
  return VTTS_OK;
}

// the rejections every push and push_host share, before anything else is looked at
inline int stream_args(vtts_ctx* ctx, const char* who, const StreamBase* sb, bool pointers_ok) {
  if (!sb || sb->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: the stream belongs to another context", who);
  if (!pointers_ok) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  return VTTS_OK;
}

template <class Stream>
int stream_destroy(vtts_ctx* ctx, const char* who, Stream* sb) {
  if (!ctx) return VTTS_ERR_BAD_ARG;
  if (!sb) return VTTS_OK;
  if (sb->ctx != ctx) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: the stream belongs to another context", who);
  VTTS_CUDA(cudaSetDevice(ctx->device));
  VTTS_CUDA(cudaDeviceSynchronize());   // a push may still be running on the caller's stream
  delete sb;
  return VTTS_OK;
}

// ---- host staging ------------------------------------------------------------------------------------------------
// The *_host entry points run the device call on the context's own stream with their buffers staged at the same
// offsets in the pinned host buffer (ctx->hpin) and the device staging buffer (ctx->dstage): inputs first, then
// outputs, then device-only scratch, each block 256 B aligned.  Declare every block, then upload(): it sizes the
// buffers, packs the inputs and queues one H2D of the input span.  From then on the stream is synchronised on every
// exit, so no copy from or into the pinned buffer outlives the call (the next call rewrites it).
class HostStage {
 public:
  explicit HostStage(vtts_ctx* c) : ctx(c), st(c->own_stream) {}
  ~HostStage() {
    if (queued) cudaStreamSynchronize(st);
  }
  HostStage(const HostStage&) = delete;
  HostStage& operator=(const HostStage&) = delete;

  // an input block of `bytes`, packed from `src` (null: left unset)
  size_t in(const void* src, size_t bytes) {
    const size_t o = take(bytes);
    ins.push_back({o, src, bytes});
    in_end = off;
    return o;
  }
  size_t out(size_t bytes) {
    const size_t o = take(bytes);
    host_end = off;
    return o;
  }
  size_t scratch(size_t bytes) { return take(bytes); }

  int upload() {
    int rc = ctx->ensure_staging(std::max(in_end, host_end), off);
    if (rc) return rc;
    char* hp = (char*)ctx->hpin;
    for (const In& i : ins)
      if (i.src) memcpy(hp + i.o, i.src, i.bytes);
    queued = true;
    if (in_end) VTTS_CUDA(cudaMemcpyAsync(ctx->dstage, hp, in_end, cudaMemcpyHostToDevice, st));
    return VTTS_OK;
  }

  template <class T>
  T* dev(size_t o) const { return reinterpret_cast<T*>((char*)ctx->dstage + o); }

  // queues the D2H of `bytes` at output offset o into dst: straight into it when `direct` (page-locked caller memory),
  // else through the pinned buffer, copied out by finish()
  int fetch(size_t o, void* dst, size_t bytes, bool direct = false) {
    VTTS_CUDA(cudaMemcpyAsync(direct ? dst : (char*)ctx->hpin + o, (char*)ctx->dstage + o, bytes, cudaMemcpyDeviceToHost, st));
    if (!direct) outs.push_back({o, dst, bytes});
    return VTTS_OK;
  }
  int finish() {
    VTTS_CUDA(cudaStreamSynchronize(st));
    queued = false;
    for (const Out& u : outs) memcpy(u.dst, (char*)ctx->hpin + u.o, u.bytes);
    return VTTS_OK;
  }

  vtts_ctx* const ctx;
  const cudaStream_t st;

 private:
  struct In { size_t o; const void* src; size_t bytes; };
  struct Out { size_t o; void* dst; size_t bytes; };
  size_t take(size_t bytes) {
    off = (off + 255) & ~size_t(255);
    const size_t o = off;
    off += bytes;
    return o;
  }
  size_t off = 0, in_end = 0, host_end = 0;
  bool queued = false;
  std::vector<In> ins;
  std::vector<Out> outs;
};

// push_host of a stream: the x_bytes of host input x are staged, push(x_dev, y_dev, stream) runs the stream's device
// push on the staged buffers, and the y_bytes of its output come back to host memory y
template <class Push>
int stream_push_host(vtts_ctx* ctx, const float* x, size_t x_bytes, float* y, size_t y_bytes, Push&& push) {
  VTTS_CUDA(cudaSetDevice(ctx->device));
  HostStage hs(ctx);
  const size_t o_x = hs.in(x, x_bytes), o_y = hs.out(y_bytes);
  int rc = hs.upload();
  if (!rc) rc = push(hs.dev<const float>(o_x), hs.dev<float>(o_y), hs.st);
  if (!rc) rc = hs.fetch(o_y, y, y_bytes);
  return rc ? rc : hs.finish();
}
