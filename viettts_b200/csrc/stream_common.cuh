// Host-side pieces shared by the per-slot streams and the *_host entry points: the slot protocol of a push, the device
// memory of a stream, the window and push tables of a sample stream, and the staging of host buffers.
#pragma once
#include <climits>
#include <memory>
#include <tuple>

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

// ---- sample streams ----------------------------------------------------------------------------------------------
// What a stream of samples adds: its window, per slot the K samples carried from earlier pushes and then the push's new
// ones ([S][cap]), and its per-push tables, one host image and its device copy laid out as Rows [S] for each row type in
// turn, then the int [S][2] window step table of vtts_stream_window_prep.  A push fills rows<I>() and then upload()s.
template <class... Rows>
struct SampleStream : StreamBase {
  template <int I>
  using Row = std::tuple_element_t<I, std::tuple<Rows...>>;

  const int K, cap;
  float* win = nullptr;

  SampleStream(vtts_ctx* c, int s, int f, int k)
      : StreamBase(c, s, f), K(k), cap(k + f), tbl((size_t)s * (offset(sizeof...(Rows)) + 2 * sizeof(int)), 0) {}

  // stream_alloc: the window comes first and the device tables last, around the stream's own buffers
  void carve_window(Arena& a) { win = a.take<float>((size_t)S * cap); }
  void carve_tables(Arena& a) { d_tbl = a.take<char>(tbl.size()); }

  template <int I>
  Row<I>* rows() { return reinterpret_cast<Row<I>*>(tbl.data() + (size_t)S * offset(I)); }
  template <int I>
  const Row<I>* d_rows() const { return reinterpret_cast<const Row<I>*>(d_tbl + (size_t)S * offset(I)); }

  // after the rows are filled, on the caller's stream: the window step table, the push's one table copy (from pageable
  // memory: the call returns once it is staged, so the next push may rewrite the image) and the window step of x
  int upload(const int32_t* n_new, const uint8_t* flags, const float* x, cudaStream_t st) {
    const size_t steps = (size_t)S * offset(sizeof...(Rows));
    slots.prep(n_new, flags, reinterpret_cast<int*>(tbl.data() + steps));
    VTTS_CUDA(cudaMemcpyAsync(d_tbl, tbl.data(), tbl.size(), cudaMemcpyHostToDevice, st));
    return vtts_stream_window_prep(ctx, win, cap, K, reinterpret_cast<const int*>(d_tbl + steps), x, F, S, st);
  }

  // a stream that reads each push's inputs where they are (K = 0, no window carved): only the push's one table copy
  int upload_rows(cudaStream_t st) {
    VTTS_CUDA(cudaMemcpyAsync(d_tbl, tbl.data(), (size_t)S * offset(sizeof...(Rows)), cudaMemcpyHostToDevice, st));
    return VTTS_OK;
  }

 private:
  // bytes per slot of the row types before the n-th
  static constexpr size_t offset(int n) {
    constexpr size_t sz[] = {sizeof(Rows)...};
    size_t b = 0;
    for (int i = 0; i < n; ++i) b += sz[i];
    return b;
  }
  std::vector<char> tbl;
  char* d_tbl = nullptr;
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

// the rejections every stream create shares: a null handle or other pointer the create needs (pointers_ok false), then
// the slot count and the largest chunk; *out is null on every failure
template <class Stream>
int create_check(vtts_ctx* ctx, const char* who, Stream** out, bool pointers_ok, int max_streams, int max_chunk, int chunk_max = 1 << 22,
                 const char* chunk = "max_chunk_samples", int streams_max = 65535) {
  if (!out || !pointers_ok) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
  *out = nullptr;
  if (max_streams < 1 || max_streams > streams_max || max_chunk < 1 || max_chunk > chunk_max)
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: max_streams=%d %s=%d (1..%d, 1..%d)", who, max_streams, chunk, max_chunk, streams_max, chunk_max);
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

// ---- batch shape -------------------------------------------------------------------------------------------------
// The one-shot audio entry points take B rows of S samples.  B rides on a grid's y dimension (at most 65535).  S runs
// from S_min (1, or 0 where an empty row has a meaning) to the stage's S_max, given by the stage beside its reason.
constexpr long long S_ANY = INT_MAX;   // no ceiling beyond an int sample count

inline int batch_check(vtts_ctx* ctx, const char* who, int B, int S, long long S_max, int S_min = 1) {
  if (B < 1 || B > 65535 || S < S_min || S > S_max)
    return ctx->fail(VTTS_ERR_BAD_ARG, "%s: B=%d S=%d (B in 1..65535, S in %d..%lld)", who, B, S, S_min, S_max);
  return VTTS_OK;
}

// ---- host staging ------------------------------------------------------------------------------------------------
// The *_host entry points run the device call on the context's own stream with their buffers staged at the same
// offsets in the pinned host buffer (ctx->hpin) and the device staging buffer (ctx->dstage): inputs first, then
// outputs, then device-only scratch, each block 256 B aligned.  Declare every block, then run(launch): it sizes the
// buffers, packs the inputs, queues one H2D of the input span, launch(stream), the D2H of every output that has a host
// destination, and waits.  From upload() on the stream is synchronised on every exit, so no copy from or into the
// pinned buffer outlives the call (the next call rewrites it).  A HostStage is the call's CallOrder scope on the own
// stream, from its construction, before the first copy, to its destruction, after the last wait.
class HostStage {
 public:
  explicit HostStage(vtts_ctx* c) : ctx(c), st(c->own_stream), order(c, c->own_stream) {}
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
  // an output block of `bytes`, fetched into `dst` by run() (null: not fetched)
  size_t out(size_t bytes, void* dst = nullptr) {
    const size_t o = take(bytes);
    host_end = off;
    if (dst) fetched.push_back({o, dst, bytes});
    return o;
  }
  size_t scratch(size_t bytes) { return take(bytes); }

  // the batch x [B][S] of `elem`-byte samples and its row lengths n [B] (null: every row full) of host entry point
  // `who`, staged as the first inputs: a null x with samples to stage, any other null pointer the call needs
  // (pointers_ok false) and any n[b] outside [0, S] are rejected
  int rows(const char* who, const void* x, const int32_t* n, int B, int S, bool pointers_ok = true, size_t elem = 4) {
    if ((!x && S) || !pointers_ok) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: null pointer", who);
    if (n)
      for (int b = 0; b < B; ++b)
        if (n[b] < 0 || n[b] > S) return ctx->fail(VTTS_ERR_BAD_ARG, "%s: n[%d]=%d outside [0, %d]", who, b, n[b], S);
    o_x = in(x, (size_t)B * S * elem);
    o_n = n ? in(n, (size_t)B * 4) : SIZE_MAX;
    return VTTS_OK;
  }
  // the staged batch and lengths (null when the call has none)
  template <class T = float>
  const T* x() const { return dev<const T>(o_x); }
  const int32_t* n() const { return o_n == SIZE_MAX ? nullptr : dev<const int32_t>(o_n); }

  template <class T>
  T* dev(size_t o) const { return reinterpret_cast<T*>((char*)ctx->dstage + o); }

  template <class Launch>
  int run(Launch&& launch) {
    VTTS_CUDA(cudaSetDevice(ctx->device));
    int rc = upload();
    if (!rc) rc = launch(st);
    for (const Out& u : fetched)
      if (!rc) rc = fetch(u.o, u.dst, u.bytes);
    return rc ? rc : finish();
  }

  // the explicit steps, for calls that wait or fetch between launches (fetch and finish may follow run, for outputs
  // whose size the launch decides)
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
  // queues the D2H of `bytes` at output offset o into dst: straight into it when `direct` (page-locked caller memory),
  // else through the pinned buffer, copied out by finish()
  int fetch(size_t o, void* dst, size_t bytes, bool direct = false) {
    VTTS_CUDA(cudaMemcpyAsync(direct ? dst : (char*)ctx->hpin + o, (char*)ctx->dstage + o, bytes, cudaMemcpyDeviceToHost, st));
    queued = true;
    if (!direct) outs.push_back({o, dst, bytes});
    return VTTS_OK;
  }
  int finish() {
    VTTS_CUDA(cudaStreamSynchronize(st));
    queued = false;
    for (const Out& u : outs) memcpy(u.dst, (char*)ctx->hpin + u.o, u.bytes);
    outs.clear();
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
  const CallOrder order;
  size_t off = 0, in_end = 0, host_end = 0, o_x = 0, o_n = SIZE_MAX;
  bool queued = false;
  std::vector<In> ins;
  std::vector<Out> fetched, outs;   // declared by out(), queued by fetch()
};
