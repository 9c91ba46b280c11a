// Host side of libaf2b200.so: TMA descriptor construction, kernel launches and the per-module
// orchestration behind the C ABI declared in include/af2b200.h.
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>
#include <nvtx3/nvToolsExt.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/af2b200.h"
#include "attention_proj.cuh"
#include "attention_tc.cuh"
#include "attention_fwd.cuh"
#include "chan2tok_tma.cuh"
#include "contract_tail.cuh"
#include "ff_fused.cuh"
#include "gemm_tc.cuh"
#include "simt_kernels.cuh"
#include "strict_kernels.cuh"
#include "glue_kernels.cuh"
#include "template_attn.cuh"
#include "heads.cuh"
#include "structure.cuh"
#include "geometry.cuh"
#include "metrics.cuh"
#include "distogram_loss.cuh"
#include "angle_loss.cuh"

using namespace af2;

namespace {

thread_local char g_err[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

#define CUDA_OK(expr)                                                                            \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return fail(AF2_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)
#define AF2_TRY(expr)            \
  do {                           \
    int _r = (expr);             \
    if (_r != AF2_OK) return _r; \
  } while (0)

// Per-device state: the dynamic-shared-memory opt-in, the SM count and the cluster occupancy are properties of a
// device, and one process may drive several (ops.py keeps per-device workspaces), so every cache is indexed by ordinal.
constexpr int MAX_DEVICES = 64;
int cur_dev() {
  int dev = 0;
  cudaGetDevice(&dev);
  return (dev >= 0 && dev < MAX_DEVICES) ? dev : 0;
}
int sm_count() {
  static int n[MAX_DEVICES] = {0};
  const int dev = cur_dev();
  if (n[dev] == 0) {
    cudaDeviceGetAttribute(&n[dev], cudaDevAttrMultiProcessorCount, dev);
    if (n[dev] <= 0) n[dev] = 132;
  }
  return n[dev];
}

// Programmatic dependent launch (common.cuh)
template <class... KArgs, class... Args>
cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

struct NvtxRange {   // one NVTX range per C-ABI call (sub-op granularity for nsys / ncu --nvtx)
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// ---------------------------------------------------------------------------------------------
// launch accounting + optional per-kernel-class CUDA-event profiling (bench.py roofline numbers)
// ---------------------------------------------------------------------------------------------
enum KClass { KC_GEMM_LINEAR = 0, KC_GEMM_CHANNEL = 1, KC_ATTENTION = 2, KC_LAYERNORM = 3, KC_CHAN2TOK = 4, KC_MISC = 5, KC_COUNT = 6 };
struct ProfRec { cudaEvent_t a, b; int cls; double flops, bytes; };
unsigned long long g_launches = 0;
bool g_prof = false;
std::vector<ProfRec> g_recs;
std::vector<cudaEvent_t> g_pool;

cudaEvent_t prof_event() {
  if (!g_pool.empty()) { cudaEvent_t e = g_pool.back(); g_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
struct ProfScope {
  cudaStream_t s; bool on; ProfRec r;
  ProfScope(cudaStream_t st, int cls, double flops, double bytes) : s(st), on(g_prof) {
    ++g_launches;
    if (on) { r.a = prof_event(); r.b = prof_event(); r.cls = cls; r.flops = flops; r.bytes = bytes; cudaEventRecord(r.a, s); }
  }
  ~ProfScope() { if (on) { cudaEventRecord(r.b, s); g_recs.push_back(r); } }
};

PFN_cuTensorMapEncodeTiled_v12000 encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// bf16 tensor map. dims[0] is the contiguous dimension; strides_bytes[i] is the stride of dims[i+1].
int make_tmap(CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
              const unsigned long long* strides_bytes, const unsigned* box, CUtensorMapSwizzle swz,
              CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16,
              CUtensorMapL2promotion promo = CU_TENSOR_MAP_L2_PROMOTION_L2_256B) {
  auto fn = encode_fn();
  if (!fn) return fail(AF2_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  if (reinterpret_cast<uintptr_t>(base) & 15) return fail(AF2_ERR_BAD_ARG, "TMA base pointer not 16-byte aligned");
  for (int i = 0; i + 1 < rank; ++i)
    if (gstr[i] & 15) return fail(AF2_ERR_BAD_ARG, "TMA stride %d (%llu B) not a multiple of 16", i, (unsigned long long)gstr[i]);
  CUresult r = fn(m, dt, rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, promo,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(AF2_ERR_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return AF2_OK;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline long long align_up(long long v, long long a) { return (v + a - 1) / a * a; }

// bump allocator over the caller's workspace
struct Arena {
  char* base;
  long long size, off;
  bool ok;
  Arena(void* b, long long s) : base(static_cast<char*>(b)), size(s), off(0), ok(true) {}
  template <class T>
  T* take(long long count) {
    long long bytes = align_up(count * (long long)sizeof(T), 256);
    if (off + bytes > size) {
      ok = false;
      return nullptr;
    }
    T* p = reinterpret_cast<T*>(base + off);
    off += bytes;
    return p;
  }
};

// -------------------------------------------------------------------------------------------------
// GEMM launch
// -------------------------------------------------------------------------------------------------
struct GemmCall {
  const void* A; long long lda; long long a_batch;
  const void* Bm; long long ldb; long long b_batch;
  int M, N, K, batch;
  bool mn_major;
  int bn;                 // 64 / 128 / 256
  // epilogue
  int mode, act, layout, use_rowscale;
  void* out; long long ld_out; long long out_batch;
  const float* bias; const float* rowscale; const float* resid; long long ld_resid;
  int cm_inner, cm_pitch;
  int out_cols;           // 0: N (N/2 for GATED); else explicit number of valid output columns
  // split-bf16 operands (strict precision, GemmParams::nseg): nseg = SPL_NSEG (3 planes); a_half / b_half = element stride between planes
  int nseg; long long a_half, b_half;
  // gathered operands (GemmParams::a_pr / b_pr): rows (K-major) or columns (MN-major) per piece, element stride between pieces
  int a_pr, b_pr; long long a_piece, b_piece;
};

template <int BN, int STAGES, bool MN, int EK>
int launch_gemm_inst(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const CUtensorMap& tr,
                     const GemmParams& p, cudaStream_t s) {
  using L = GemmSmem<BN, STAGES>;
  static bool configured[MAX_DEVICES] = {false};
  auto kern = gemm_tc_kernel<BN, STAGES, MN, EK>;
  if (!configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured[cur_dev()] = true;
  }
  const int m_tiles = (p.M + GEMM_BM - 1) / GEMM_BM;
  const long long total = (long long)p.batch * m_tiles * p.num_ntiles;
  if (total <= 0) return AF2_OK;
  const int grid = (int)(total < sm_count() ? total : sm_count());
  const double flops = 2.0 * p.batch * (double)p.M * p.N * p.K;    // algorithmic (a split-operand launch issues 3x this)
  const double obytes = (p.tile.mode == EPI_STORE_BF16 ? 2.0 : (p.tile.mode == EPI_GATED_BF16 ? 1.0 : (p.tile.mode == EPI_RESID_F32 ? 8.0 : 4.0)));
  const double bytes = p.batch * ((double)p.M * p.K * 2 + (p.batch > 1 ? (double)p.N * p.K * 2 : 0) + (double)p.M * p.N * obytes) +
                       (p.batch > 1 ? 0 : (double)p.N * p.K * 2);
  ProfScope ps(s, p.batch > 1 ? KC_GEMM_CHANNEL : KC_GEMM_LINEAR, flops, bytes);
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), L::TOTAL, s, ta, tb, tc, tr, p));
  return AF2_OK;
}

// Whether the call's output (and residual) can go through TMA: 16-byte aligned bases and pitches, and for the channel-major
// layout whole 64-row boxes inside each cm_inner block.  Otherwise the epilogue stores from registers.  A token-major row
// must also end on a 16-byte boundary: a TMA store clipped inside a 16-byte segment writes the rest of the segment.
bool gemm_epi_tma_ok(const GemmCall& c, int out_cols) {
  const bool f32 = c.mode == EPI_RESID_F32 || c.mode == EPI_STORE_F32;
  const long long es = f32 ? 4 : 2;
  if (!aligned16(c.out) || (c.batch > 1 && (c.out_batch * es) % 16)) return false;
  if (c.layout == LAYOUT_CHANNEL) {
    if (f32 || c.cm_inner <= 0 || c.cm_inner % GEMM_BM || c.M % c.cm_inner || (c.cm_pitch * 2) % 16 || (c.ld_out * 2) % 16) return false;
  } else if ((c.ld_out * es) % 16 || (out_cols * es) % 16) {
    return false;
  }
  if (c.mode == EPI_RESID_F32 && (!aligned16(c.resid) || (c.ld_resid * 4) % 16)) return false;
  return true;
}

int launch_gemm(const GemmCall& c, cudaStream_t s) {
  if (c.M <= 0 || c.N <= 0 || c.K <= 0 || c.batch <= 0) return AF2_OK;
  // the residual is read at [row][col] of batch 0 whatever the batch index: a batched residual GEMM would add the wrong rows
  if (c.mode == EPI_RESID_F32 && c.batch > 1) return fail(AF2_ERR_BAD_ARG, "gemm: residual epilogue with batch %d (needs 1)", c.batch);
  CUtensorMap ta, tb;
  const int BN = c.bn;
  if (c.nseg > 1) {
    // rank-4 maps (k | mn, row | k, plane, batch) over the SPL planes of split-bf16 operands
    if (c.nseg != SPL_NSEG) return fail(AF2_ERR_BAD_ARG, "gemm: %d split passes (needs %d)", c.nseg, SPL_NSEG);
    const unsigned long long npl = SPL;
    const unsigned long long ab = (unsigned long long)(c.batch > 1 ? c.a_batch : 0) * 2, bb_ = (unsigned long long)(c.batch > 1 ? c.b_batch : 0) * 2;
    if (!c.mn_major) {
      unsigned long long da[4] = {(unsigned long long)c.K, (unsigned long long)c.M, npl, (unsigned long long)c.batch};
      unsigned long long sa[3] = {(unsigned long long)c.lda * 2, (unsigned long long)c.a_half * 2, ab ? ab : (unsigned long long)c.a_half * 8};
      unsigned ba[4] = {64, GEMM_BM, 1, 1};
      AF2_TRY(make_tmap(&ta, c.A, 4, da, sa, ba, CU_TENSOR_MAP_SWIZZLE_128B));
      unsigned long long db[4] = {(unsigned long long)c.K, (unsigned long long)c.N, npl, (unsigned long long)c.batch};
      unsigned long long sb[3] = {(unsigned long long)c.ldb * 2, (unsigned long long)c.b_half * 2, bb_ ? bb_ : (unsigned long long)c.b_half * 8};
      unsigned bx[4] = {64, (unsigned)BN, 1, 1};
      AF2_TRY(make_tmap(&tb, c.Bm, 4, db, sb, bx, CU_TENSOR_MAP_SWIZZLE_128B));
    } else {
      unsigned long long da[4] = {(unsigned long long)c.M, (unsigned long long)c.K, npl, (unsigned long long)c.batch};
      unsigned long long sa[3] = {(unsigned long long)c.lda * 2, (unsigned long long)c.a_half * 2, ab ? ab : (unsigned long long)c.a_half * 8};
      unsigned bx[4] = {64, 64, 1, 1};
      AF2_TRY(make_tmap(&ta, c.A, 4, da, sa, bx, CU_TENSOR_MAP_SWIZZLE_128B));
      unsigned long long db[4] = {(unsigned long long)c.N, (unsigned long long)c.K, npl, (unsigned long long)c.batch};
      unsigned long long sb[3] = {(unsigned long long)c.ldb * 2, (unsigned long long)c.b_half * 2, bb_ ? bb_ : (unsigned long long)c.b_half * 8};
      AF2_TRY(make_tmap(&tb, c.Bm, 4, db, sb, bx, CU_TENSOR_MAP_SWIZZLE_128B));
    }
  } else if (!c.mn_major) {
    unsigned long long da[3] = {(unsigned long long)c.K, (unsigned long long)c.M, (unsigned long long)c.batch};
    unsigned long long sa[2] = {(unsigned long long)c.lda * 2, (unsigned long long)(c.batch > 1 ? c.a_batch : c.lda * c.M) * 2};
    unsigned ba[3] = {64, GEMM_BM, 1};
    AF2_TRY(make_tmap(&ta, c.A, 3, da, sa, ba, CU_TENSOR_MAP_SWIZZLE_128B));
    unsigned long long db[3] = {(unsigned long long)c.K, (unsigned long long)c.N, (unsigned long long)c.batch};
    unsigned long long sb[2] = {(unsigned long long)c.ldb * 2, (unsigned long long)(c.batch > 1 && c.b_batch ? c.b_batch : c.ldb * c.N) * 2};
    unsigned bb[3] = {64, (unsigned)BN, 1};
    AF2_TRY(make_tmap(&tb, c.Bm, 3, db, sb, bb, CU_TENSOR_MAP_SWIZZLE_128B));
  } else {
    unsigned long long da[3] = {(unsigned long long)c.M, (unsigned long long)c.K, (unsigned long long)c.batch};
    unsigned long long sa[2] = {(unsigned long long)c.lda * 2, (unsigned long long)(c.batch > 1 ? c.a_batch : c.lda * c.K) * 2};
    unsigned bx[3] = {64, 64, 1};
    AF2_TRY(make_tmap(&ta, c.A, 3, da, sa, bx, CU_TENSOR_MAP_SWIZZLE_128B));
    unsigned long long db[3] = {(unsigned long long)c.N, (unsigned long long)c.K, (unsigned long long)c.batch};
    unsigned long long sb[2] = {(unsigned long long)c.ldb * 2, (unsigned long long)(c.batch > 1 ? c.b_batch : c.ldb * c.K) * 2};
    AF2_TRY(make_tmap(&tb, c.Bm, 3, db, sb, bx, CU_TENSOR_MAP_SWIZZLE_128B));
  }
  // gathered ("pieces") operands: replace the plain map by a rank-4 map (k | mn, row | k, piece, batch)
  if (c.nseg <= 1 && (c.a_pr > 0 || c.b_pr > 0)) {
    const unsigned long long bsa = (unsigned long long)(c.batch > 1 ? c.a_batch : c.lda) * 2, bsb = (unsigned long long)(c.batch > 1 ? c.b_batch : c.ldb) * 2;
    if (!c.mn_major) {
      if (c.a_pr > 0) {
        if (c.a_pr % 128 != 0) return fail(AF2_ERR_BAD_ARG, "gemm: gathered A pieces of %d rows (need a multiple of 128)", c.a_pr);
        unsigned long long da[4] = {(unsigned long long)c.K, (unsigned long long)c.a_pr, (unsigned long long)((c.M + c.a_pr - 1) / c.a_pr), (unsigned long long)c.batch};
        unsigned long long sa[3] = {(unsigned long long)c.lda * 2, (unsigned long long)c.a_piece * 2, bsa};
        unsigned ba[4] = {64, GEMM_BM, 1, 1};
        AF2_TRY(make_tmap(&ta, c.A, 4, da, sa, ba, CU_TENSOR_MAP_SWIZZLE_128B));
      }
      if (c.b_pr > 0) {
        if (!((c.b_pr % BN) == 0 || (BN % c.b_pr) == 0) || c.b_pr % 8) return fail(AF2_ERR_BAD_ARG, "gemm: gathered B pieces of %d rows do not tile BN=%d", c.b_pr, BN);
        unsigned long long db[4] = {(unsigned long long)c.K, (unsigned long long)c.b_pr, (unsigned long long)((c.N + c.b_pr - 1) / c.b_pr), (unsigned long long)c.batch};
        unsigned long long sb[3] = {(unsigned long long)c.ldb * 2, (unsigned long long)c.b_piece * 2, bsb};
        unsigned bb[4] = {64, (unsigned)(c.b_pr >= BN ? BN : c.b_pr), (unsigned)(c.b_pr >= BN ? 1 : BN / c.b_pr), 1};
        AF2_TRY(make_tmap(&tb, c.Bm, 4, db, sb, bb, CU_TENSOR_MAP_SWIZZLE_128B));
      }
    } else {
      unsigned bx[4] = {64, 64, 1, 1};
      if (c.a_pr > 0) {
        if (c.a_pr % 64) return fail(AF2_ERR_BAD_ARG, "gemm: gathered MN-major A pieces of %d columns (need a multiple of 64)", c.a_pr);
        unsigned long long da[4] = {(unsigned long long)c.a_pr, (unsigned long long)c.K, (unsigned long long)((c.M + c.a_pr - 1) / c.a_pr), (unsigned long long)c.batch};
        unsigned long long sa[3] = {(unsigned long long)c.lda * 2, (unsigned long long)c.a_piece * 2, bsa};
        AF2_TRY(make_tmap(&ta, c.A, 4, da, sa, bx, CU_TENSOR_MAP_SWIZZLE_128B));
      }
      if (c.b_pr > 0) {
        if (c.b_pr % 64) return fail(AF2_ERR_BAD_ARG, "gemm: gathered MN-major B pieces of %d columns (need a multiple of 64)", c.b_pr);
        unsigned long long db[4] = {(unsigned long long)c.b_pr, (unsigned long long)c.K, (unsigned long long)((c.N + c.b_pr - 1) / c.b_pr), (unsigned long long)c.batch};
        unsigned long long sb[3] = {(unsigned long long)c.ldb * 2, (unsigned long long)c.b_piece * 2, bsb};
        AF2_TRY(make_tmap(&tb, c.Bm, 4, db, sb, bx, CU_TENSOR_MAP_SWIZZLE_128B));
      }
    }
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = c.M; p.N = c.N; p.K = c.K; p.batch = c.batch; p.nseg = c.nseg > 1 ? c.nseg : 1;
  if (c.nseg <= 1) { p.a_pr = c.a_pr; p.b_pr = c.b_pr; }
  p.num_ntiles = (c.N + BN - 1) / BN;
  p.out_cols = c.out_cols > 0 ? c.out_cols : ((c.mode == EPI_GATED_BF16) ? c.N / 2 : c.N);
  p.rowscale = c.rowscale; p.resid = c.resid; p.ld_resid = c.ld_resid;
  p.out_batch_stride = c.out_batch;
  p.cm_inner = c.cm_inner > 0 ? c.cm_inner : 1; p.cm_pitch = c.cm_pitch > 0 ? c.cm_pitch : 1;
  p.tile.mode = c.mode; p.tile.act = c.act; p.tile.layout = c.layout; p.tile.use_rowscale = c.use_rowscale;
  p.tile.out = c.out; p.tile.bias = c.bias; p.tile.ld = c.ld_out;
  // compile-time epilogue specialisation for the big-tile instantiation
  int ek = EK_GENERIC;
  if (BN == 256) {
    if (c.mode == EPI_STORE_BF16 && c.layout == LAYOUT_TOKEN && c.act == ACT_NONE && !c.use_rowscale) ek = EK_STORE_TOK;
    else if (c.mode == EPI_STORE_BF16 && c.layout == LAYOUT_TOKEN && c.act == ACT_SIGMOID && !c.use_rowscale) ek = EK_STORE_TOK_SIG;
    else if (c.mode == EPI_STORE_BF16 && c.layout == LAYOUT_CHANNEL && c.act == ACT_NONE) ek = EK_STORE_CH;
    else if (c.mode == EPI_GATED_BF16 && c.layout == LAYOUT_TOKEN && c.act == ACT_GELU && !c.use_rowscale) ek = EK_GATED_TOK_GELU;
    else if (c.mode == EPI_GATED_BF16 && c.layout == LAYOUT_CHANNEL && c.act == ACT_SIGMOID) ek = EK_GATED_CH_SIG;
    else if (c.mode == EPI_RESID_F32 && !c.use_rowscale) ek = EK_RESID_F32;
    else if (c.mode == EPI_STORE_F32) ek = EK_STORE_F32;
  }
  if (c.mn_major && ek != EK_STORE_F32) ek = EK_GENERIC;
  // output (and residual) tensor maps of the TMA epilogue; the register epilogue needs none
  CUtensorMap tc = ta, tr = ta;
  p.epi_tma = ek != EK_GENERIC && gemm_epi_tma_ok(c, p.out_cols) ? 1 : 0;
  if (p.epi_tma) {
    const bool f32 = c.mode == EPI_RESID_F32 || c.mode == EPI_STORE_F32;
    const unsigned long long es = f32 ? 4 : 2;
    // batch 1: the batch stride is never stepped, but TMA still needs it below 2^40 B; the span of one batch element (for
    // the channel-major layout ld_out is the channel stride: ld_out * M overflowed from N_res = 1024 on)
    const unsigned long long bstride =
        (unsigned long long)(c.batch > 1 ? c.out_batch : (c.layout == LAYOUT_CHANNEL ? c.ld_out * p.out_cols : c.ld_out * c.M)) * es;
    if (c.layout == LAYOUT_CHANNEL) {
      // [batch][col][row block][row in block]: 64-row x 64-column boxes written from a [col][row] stage
      unsigned long long dc[4] = {(unsigned long long)p.cm_inner, (unsigned long long)(c.M / p.cm_inner), (unsigned long long)p.out_cols, (unsigned long long)c.batch};
      unsigned long long sc[3] = {(unsigned long long)p.cm_pitch * 2, (unsigned long long)c.ld_out * 2, bstride};
      unsigned bc[4] = {64, 1, 64, 1};
      AF2_TRY(make_tmap(&tc, c.out, 4, dc, sc, bc, CU_TENSOR_MAP_SWIZZLE_128B));
    } else {
      unsigned long long dc[3] = {(unsigned long long)p.out_cols, (unsigned long long)c.M, (unsigned long long)c.batch};
      unsigned long long sc[2] = {(unsigned long long)c.ld_out * es, bstride};
      unsigned bc[3] = {f32 ? 32u : 64u, (unsigned)GEMM_BM, 1};
      AF2_TRY(make_tmap(&tc, c.out, 3, dc, sc, bc, CU_TENSOR_MAP_SWIZZLE_128B,
                        f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16));
    }
    if (c.mode == EPI_RESID_F32) {
      unsigned long long dr[2] = {(unsigned long long)p.out_cols, (unsigned long long)c.M};
      unsigned long long sr[1] = {(unsigned long long)c.ld_resid * 4};
      unsigned br[2] = {32, (unsigned)GEMM_BM};
      AF2_TRY(make_tmap(&tr, c.resid, 2, dr, sr, br, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_DATA_TYPE_FLOAT32));
    }
  }
  if (c.mn_major) {
    if (BN == 256) {
      if (ek == EK_STORE_F32) return launch_gemm_inst<256, 4, true, EK_STORE_F32>(ta, tb, tc, tr, p, s);
      return launch_gemm_inst<256, 4, true, EK_GENERIC>(ta, tb, tc, tr, p, s);
    }
    if (BN == 128) return launch_gemm_inst<128, 6, true, EK_GENERIC>(ta, tb, tc, tr, p, s);
    return launch_gemm_inst<64, 8, true, EK_GENERIC>(ta, tb, tc, tr, p, s);
  }
  if (BN == 256) {
    switch (ek) {
      case EK_STORE_TOK: return launch_gemm_inst<256, 4, false, EK_STORE_TOK>(ta, tb, tc, tr, p, s);
      case EK_STORE_TOK_SIG: return launch_gemm_inst<256, 4, false, EK_STORE_TOK_SIG>(ta, tb, tc, tr, p, s);
      case EK_STORE_CH: return launch_gemm_inst<256, 4, false, EK_STORE_CH>(ta, tb, tc, tr, p, s);
      case EK_GATED_TOK_GELU: return launch_gemm_inst<256, 4, false, EK_GATED_TOK_GELU>(ta, tb, tc, tr, p, s);
      case EK_GATED_CH_SIG: return launch_gemm_inst<256, 4, false, EK_GATED_CH_SIG>(ta, tb, tc, tr, p, s);
      case EK_RESID_F32: return launch_gemm_inst<256, 4, false, EK_RESID_F32>(ta, tb, tc, tr, p, s);
      case EK_STORE_F32: return launch_gemm_inst<256, 4, false, EK_STORE_F32>(ta, tb, tc, tr, p, s);
      default: return launch_gemm_inst<256, 4, false, EK_GENERIC>(ta, tb, tc, tr, p, s);
    }
  }
  if (BN == 128) return launch_gemm_inst<128, 6, false, EK_GENERIC>(ta, tb, tc, tr, p, s);
  return launch_gemm_inst<64, 8, false, EK_GENERIC>(ta, tb, tc, tr, p, s);
}

int pick_bn(int n) { return n > 128 ? 256 : (n > 64 ? 128 : 64); }

GemmCall linear_call(const void* A, long long lda, const void* W, long long ldw, int M, int N, int K) {
  GemmCall c;
  memset(&c, 0, sizeof(c));
  c.A = A; c.lda = lda; c.Bm = W; c.ldb = ldw; c.M = M; c.N = N; c.K = K; c.batch = 1;
  c.mn_major = false; c.bn = pick_bn(N);
  return c;
}

// -------------------------------------------------------------------------------------------------
// Fused GEGLU feed-forward launch (ff_fused.cuh)
// -------------------------------------------------------------------------------------------------
// The fused kernel reads W1 packed with 256-row tiles ([128 value | 128 gate] rows, ops.pack_gated), W2 in HC-column
// chunks and everything through TMA or 8-byte vector accesses; other shapes take the two-GEMM path.
bool ff_fused_ok(const af2_ff_weights* w, const float* x, const void* xn, int d, int hidden) {
  return (d == 128 || d == 256) && hidden % 128 == 0 && w->bn == 256 && w->b1 && w->b2 && aligned16(x) && aligned16(xn) &&
         aligned16(w->w1) && aligned16(w->w2) && aligned16(w->b1) && aligned16(w->b2);
}

template <int D, int HC>
int launch_ff_fused(const af2_ff_weights* w, float* x, const __nv_bfloat16* xn, long long T, int hidden, cudaStream_t s) {
  using L = FfSmem<D, HC>;
  static bool configured[MAX_DEVICES] = {false};
  auto kern = ff_fused_kernel<D, HC>;
  if (!configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured[cur_dev()] = true;
  }
  if (T <= 0) return AF2_OK;
  CUtensorMap tx, t1, t2;
  const unsigned long long dx[2] = {(unsigned long long)D, (unsigned long long)T}, sx[1] = {(unsigned long long)D * 2};
  const unsigned long long d1[2] = {(unsigned long long)D, 2ull * hidden}, s1[1] = {(unsigned long long)D * 2};
  const unsigned long long d2[2] = {(unsigned long long)hidden, (unsigned long long)D}, s2[1] = {(unsigned long long)hidden * 2};
  const unsigned b64[2] = {64, 64}, bw1[2] = {64, (unsigned)HC}, bw2[2] = {(unsigned)HC, (unsigned)D};
  AF2_TRY(make_tmap(&tx, xn, 2, dx, sx, b64, CU_TENSOR_MAP_SWIZZLE_128B));
  AF2_TRY(make_tmap(&t1, w->w1, 2, d1, s1, bw1, CU_TENSOR_MAP_SWIZZLE_128B));
  AF2_TRY(make_tmap(&t2, w->w2, 2, d2, s2, bw2, HC == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B));
  FfParams p;
  p.x = x; p.b1 = w->b1; p.b2 = w->b2; p.T = (int)T; p.hidden = hidden;
  const long long tiles = (T + FF_BM - 1) / FF_BM;
  const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
  const double flops = 2.0 * T * (2.0 * D * hidden + (double)hidden * D);
  const double bytes = (double)T * D * 2 + 3.0 * D * hidden * 2 + (double)T * D * 8;   // xn, W1 and W2 once, x read + written
  ProfScope ps(s, KC_GEMM_LINEAR, flops, bytes);
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(FF_THREADS), L::TOTAL, s, tx, t1, t2, p));
  return AF2_OK;
}

// -------------------------------------------------------------------------------------------------
// LayerNorm launch
// -------------------------------------------------------------------------------------------------
int launch_layernorm(const LnParams& p, cudaStream_t s) {
  if (p.T <= 0) return AF2_OK;
  if (p.d % 4 != 0 || p.d > 1024) return fail(AF2_ERR_BAD_ARG, "LayerNorm: dim %d must be a multiple of 4 and <= 1024", p.d);
  const long long blocks_needed = (p.T + 7) / 8;
  const long long cap = (long long)sm_count() * 16;
  const int grid = (int)(blocks_needed < cap ? blocks_needed : cap);
  ProfScope ps(s, KC_LAYERNORM, 0.0, (double)p.T * p.d * (p.y ? 6.0 : 4.0) + (p.wb ? (double)p.T * p.heads * 2 : 0));
  if (p.d <= 128) layernorm_rows_kernel<1><<<grid, 256, 0, s>>>(p);
  else if (p.d <= 256) layernorm_rows_kernel<2><<<grid, 256, 0, s>>>(p);
  else if (p.d <= 512) layernorm_rows_kernel<4><<<grid, 256, 0, s>>>(p);
  else layernorm_rows_kernel<8><<<grid, 256, 0, s>>>(p);
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

// pair bias <x_raw, w_edge> of T tokens (d % 32 == 0, d <= 256, heads <= 8), else the LayerNorm kernel's bias path
bool pair_bias_fast_ok(int d, int heads) { return d % 32 == 0 && d >= 32 && d <= 256 && heads <= 8; }
int launch_pair_bias(const float* x, long long T, int d, const float* wb, __nv_bfloat16* bias_out, int heads, long long bias_hs,
                     int n_inner, int pitch, cudaStream_t s, int transpose = 0) {
  if (T <= 0) return AF2_OK;
  PairBiasParams p;
  p.x = x; p.T = T; p.d = d; p.wb = wb; p.bias_out = bias_out; p.heads = heads; p.bias_hs = bias_hs; p.n_inner = n_inner; p.pitch = pitch;
  p.transpose = transpose;
  if (T > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "pair_bias: too many tokens");
  const bool mma = (d == 256 || d == 128);
  const long long need = mma ? (T + 127) / 128 : (T + 31) / 32;   // 8 warps x 16 (tensor-core kernel) / 4 tokens per block iteration
  const long long cap = (long long)sm_count() * 3;     // persistent: 3 resident blocks per SM
  const int grid = (int)(need < cap ? need : cap);
  ProfScope ps(s, KC_LAYERNORM, 0.0, (double)T * d * 4 + (double)T * heads * 2);
  if (mma && d == 256) CUDA_OK(launch_pdl(pair_bias_mma_kernel<16>, dim3(grid), dim3(256), 0, s, p));
  else if (mma) CUDA_OK(launch_pdl(pair_bias_mma_kernel<8>, dim3(grid), dim3(256), 0, s, p));
  else {
    switch (d / 32) {
      case 7: pair_bias_kernel<7><<<grid, 256, 0, s>>>(p); break;
      case 6: pair_bias_kernel<6><<<grid, 256, 0, s>>>(p); break;
      case 5: pair_bias_kernel<5><<<grid, 256, 0, s>>>(p); break;
      case 3: pair_bias_kernel<3><<<grid, 256, 0, s>>>(p); break;
      case 2: pair_bias_kernel<2><<<grid, 256, 0, s>>>(p); break;
      default: pair_bias_kernel<1><<<grid, 256, 0, s>>>(p); break;
    }
  }
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

template <int D>
int launch_chan_to_token_tma(const ChanLnParams& p, long long T, cudaStream_t s) {
  using L = Chan2TokSmem<D>;
  static bool configured[MAX_DEVICES] = {false};
  auto kern = chan_to_token_tma_kernel<D>;
  if (!configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured[cur_dev()] = true;
  }
  CUtensorMap tx, tg, ty;
  {
    unsigned long long dx[2] = {(unsigned long long)T, (unsigned long long)D};
    unsigned long long sx[1] = {(unsigned long long)p.chan_stride * 4};
    unsigned bx[2] = {C2T_TOK, (unsigned)D};
    AF2_TRY(make_tmap(&tx, p.src, 2, dx, sx, bx, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_DATA_TYPE_FLOAT32));
    unsigned long long dy[2] = {(unsigned long long)D, (unsigned long long)T};
    unsigned long long sy[1] = {(unsigned long long)D * 2};
    unsigned by[2] = {64, C2T_TOK};
    AF2_TRY(make_tmap(&ty, p.y, 2, dy, sy, by, CU_TENSOR_MAP_SWIZZLE_128B));
    if (p.mode == 0) AF2_TRY(make_tmap(&tg, p.gate, 2, dy, sy, by, CU_TENSOR_MAP_SWIZZLE_128B));
    else tg = ty;
  }
  Chan2TokParams q;
  q.T = T; q.mode = p.mode; q.gamma = p.gamma; q.beta = p.beta; q.scale = p.scale; q.scale_const = p.scale_const; q.eps = p.eps;
  const long long tiles = (T + C2T_TOK - 1) / C2T_TOK;
  const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
  ProfScope ps(s, KC_CHAN2TOK, 0.0, (double)T * D * (p.mode == 0 ? 8.0 : 6.0));
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(L::THREADS), L::TOTAL, s, tx, tg, ty, q));
  return AF2_OK;
}

// channel -> token kernels (af2_chan_to_token numbers them the same way)
enum C2tVariant { C2T_AUTO = 0, C2T_SIMT = 1, C2T_TILE = 2, C2T_TMA = 3 };

// What each kernel needs of the call.  Both dense-grid kernels read src[c][t] at t = row * n + j, so the rows must be
// unpadded (pitch == n).  TMA: 16-byte aligned bases and a 16-byte channel stride for the tensor maps, int token
// coordinates.  Tile: 16-byte loads of src (at c * chan_stride) and stores of y, in mode 0 also of gate, gamma and beta,
// and whole float4 token groups (T % 4 == 0).  SIMT: one block row per token row (grid.y), d * 33 floats of shared memory.
bool c2t_variant_ok(const ChanLnParams& p, int v) {
  const long long T = (long long)p.rows * p.n;
  switch (v) {
    case C2T_TMA:
      return p.pitch == p.n && (p.d == 256 || p.d == 128) && (p.chan_stride % 4) == 0 && T > 0 && T < (1ll << 31) &&
             aligned16(p.src) && aligned16(p.y) && (p.mode != 0 || aligned16(p.gate));
    case C2T_TILE:
      return p.pitch == p.n && p.d % 64 == 0 && p.d <= 256 && (T % 4) == 0 && (p.chan_stride % 4) == 0 &&
             aligned16(p.src) && aligned16(p.y) && (p.mode != 0 || (aligned16(p.gate) && aligned16(p.gamma) && aligned16(p.beta)));
    case C2T_SIMT:
      return p.rows <= 65535 && p.d > 0 && (size_t)p.d * 33 * sizeof(float) <= 227 * 1024;
    default:
      return false;
  }
}

// the kernel launch_chan_to_token runs for this call: the TMA kernel where it applies, else the tile kernel, else the SIMT
// kernel; 0 if none can take it
int c2t_select(const ChanLnParams& p) {
  if (c2t_variant_ok(p, C2T_TMA)) return C2T_TMA;
  if (c2t_variant_ok(p, C2T_TILE)) return C2T_TILE;
  return c2t_variant_ok(p, C2T_SIMT) ? C2T_SIMT : 0;
}

// variant: C2T_AUTO (c2t_select) or a forced kernel, which must satisfy c2t_variant_ok; *ran <- the kernel launched (0: none)
int launch_chan_to_token(const ChanLnParams& p, cudaStream_t s, int variant = C2T_AUTO, int* ran = nullptr) {
  if (ran) *ran = 0;
  const long long T = (long long)p.rows * p.n;
  if (T <= 0) return AF2_OK;
  const int v = variant == C2T_AUTO ? c2t_select(p) : variant;
  if (v == 0 || !c2t_variant_ok(p, v))
    return fail(AF2_ERR_BAD_ARG, "chan_to_token: variant %d cannot run d=%d rows=%d n=%d pitch=%d chan_stride=%lld mode=%d",
                variant, p.d, p.rows, p.n, p.pitch, p.chan_stride, p.mode);
  if (ran) *ran = v;
  if (v == C2T_TMA) {
    // dense token grid: persistent TMA-pipelined kernel
    return p.d == 256 ? launch_chan_to_token_tma<256>(p, T, s) : launch_chan_to_token_tma<128>(p, T, s);
  }
  if (v == C2T_TILE) {
    // dense token grid: 64-token tiles, fully coalesced
    const size_t smem = (size_t)p.d * 64 * sizeof(float) + 8 * 64 * 2 * sizeof(float);
    static bool configured[MAX_DEVICES] = {false};
    if (!configured[cur_dev()]) {
      CUDA_OK(cudaFuncSetAttribute(chan_to_token_tile_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 64 * 4 + 4096));
      CUDA_OK(cudaFuncSetAttribute(chan_to_token_tile_kernel<24>, cudaFuncAttributeMaxDynamicSharedMemorySize, 192 * 64 * 4 + 4096));
      configured[cur_dev()] = true;
    }
    ProfScope ps(s, KC_CHAN2TOK, 0.0, (double)T * p.d * (p.mode == 0 ? 8.0 : 6.0));
    const unsigned grid = (unsigned)((T + 63) / 64);
    switch (p.d / 64) {
      case 4: chan_to_token_tile_kernel<32><<<grid, 512, smem, s>>>(p, T); break;
      case 3: chan_to_token_tile_kernel<24><<<grid, 512, smem, s>>>(p, T); break;
      case 2: chan_to_token_tile_kernel<16><<<grid, 512, smem, s>>>(p, T); break;
      default: chan_to_token_tile_kernel<8><<<grid, 512, smem, s>>>(p, T); break;
    }
    CUDA_OK(cudaGetLastError());
    return AF2_OK;
  }
  const size_t smem = (size_t)p.d * 33 * sizeof(float);
  static size_t configured[MAX_DEVICES] = {0};
  if (smem > 48 * 1024 && smem > configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(chan_to_token_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured[cur_dev()] = smem;
  }
  dim3 grid((p.n + 31) / 32, p.rows);
  ProfScope ps(s, KC_CHAN2TOK, 0.0, (double)p.rows * p.n * p.d * (p.mode == 0 ? 8.0 : 6.0));
  chan_to_token_kernel<<<grid, 256, smem, s>>>(p);
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

// -------------------------------------------------------------------------------------------------
// attention launch (one folded batch group)
// -------------------------------------------------------------------------------------------------
// head widths of the bf16 tensor-core attention kernel (strict mode takes any multiple of 4)
static bool attention_dim_head_ok(int dh) { return dh == 16 || dh == 32 || dh == 64 || dh == 128; }
#define DIM_HEAD_UNSUPPORTED \
  "dim_head %d unsupported (16, 32, 64 or 128 in bf16 mode; strict mode takes any multiple of 4)"

template <int DH>
int launch_attention_inst(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const CUtensorMap& tg,
                          const AttnParams& p, cudaStream_t s) {
  using L = AttnSmem<DH>;
  static int configured[MAX_DEVICES] = {0};
  auto kern = attention_tc_kernel<DH>;
  const int smem = L::bytes(p.n);
  if (smem > 232448) return fail(AF2_ERR_BAD_ARG, "attention: sequence length %d too long", p.n);
  if (smem > configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured[cur_dev()] = smem;
  }
  const int nqb = (p.n + 127) / 128;
  const long long items = (long long)nqb * p.heads * p.nbatch;
  if (items <= 0) return AF2_OK;
  const int grid = (int)(items < sm_count() ? items : sm_count());   // persistent: one CTA per SM, items strided over them
  if (items > 0x7fffffffLL - grid) return fail(AF2_ERR_BAD_ARG, "attention: too many work items");
  const double tokens = (double)p.n * p.nbatch;
  ProfScope ps(s, KC_ATTENTION, 4.0 * tokens * p.n * p.heads * DH,
               tokens * p.heads * DH * 2.0 * 5 + (p.has_bias ? (double)p.heads * p.n * p.n * 2 : 0));
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(ATTN_THREADS), smem, s, tq, tk, tv, tg, p));
  return AF2_OK;
}

// qkv: bf16 [tokens, 3I] (q | k | v), gate: bf16 [tokens, I], token(b', i) = b' * tok_sb + i * tok_si
int launch_attention(const __nv_bfloat16* qkv, int heads, int dh, int n, int nbatch, long long tok_sb, long long tok_si,
                     const __nv_bfloat16* bias, int npad, const uint8_t* mask, const __nv_bfloat16* gate,
                     __nv_bfloat16* out, cudaStream_t s) {
  if (!attention_dim_head_ok(dh)) return fail(AF2_ERR_BAD_ARG, "attention: " DIM_HEAD_UNSUPPORTED, dh);
  const long long I = (long long)heads * dh;
  const long long ld = 3 * I;
  CUtensorMap tq, tk, tv, tg;
  unsigned long long dims[4] = {(unsigned long long)dh, (unsigned long long)n, (unsigned long long)heads, (unsigned long long)nbatch};
  unsigned long long str[3] = {(unsigned long long)(tok_si * ld * 2), (unsigned long long)(dh * 2), (unsigned long long)(tok_sb * ld * 2)};
  unsigned long long gstr[3] = {(unsigned long long)(tok_si * I * 2), (unsigned long long)(dh * 2), (unsigned long long)(tok_sb * I * 2)};
  // a 128B-swizzled box row holds at most 64 channels: DH 128 tiles are loaded as two 64-channel boxes
  unsigned box[4] = {(unsigned)(dh < 64 ? dh : 64), 128, 1, 1};
  const CUtensorMapSwizzle swz = dh >= 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                 : dh == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
  // A box row is ONE head's slice of a token (dh * 2 bytes); the CTAs resident together read all heads of the same tokens
  // (head-innermost item order).  256B promotion measured no faster than promotion to the row size under that order (one
  // H100, C2 shapes, tools/time_attention.py), so the L2 fill stays at the row size: 64 B (the least promotion) at DH 16
  // and 32, 128 B at 64, 256 B at 128.
  const CUtensorMapL2promotion promo = dh == 128 ? CU_TENSOR_MAP_L2_PROMOTION_L2_256B
                                       : dh == 64 ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_64B;
  const CUtensorMapDataType bf = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  AF2_TRY(make_tmap(&tq, qkv, 4, dims, str, box, swz, bf, promo));
  AF2_TRY(make_tmap(&tk, qkv + I, 4, dims, str, box, swz, bf, promo));
  AF2_TRY(make_tmap(&tv, qkv + 2 * I, 4, dims, str, box, swz, bf, promo));
  AF2_TRY(make_tmap(&tg, gate, 4, dims, gstr, box, swz, bf, promo));
  if (bias && npad % 2 != 0) return fail(AF2_ERR_BAD_ARG, "attention: bias pitch %d must be even", npad);
  AttnParams p;
  memset(&p, 0, sizeof(p));
  p.n = n; p.heads = heads; p.nbatch = nbatch; p.has_bias = bias != nullptr; p.bias = bias; p.npad = npad;
  p.mask = mask; p.mask_sb = tok_sb; p.mask_si = tok_si;
  p.out = out; p.tok_sb = tok_sb; p.tok_si = tok_si; p.ld_out = I; p.gate = gate;
  switch (dh) {
    case 16: return launch_attention_inst<16>(tq, tk, tv, tg, p, s);
    case 32: return launch_attention_inst<32>(tq, tk, tv, tg, p, s);
    case 64: return launch_attention_inst<64>(tq, tk, tv, tg, p, s);
    default: return launch_attention_inst<128>(tq, tk, tv, tg, p, s);
  }
}

// -------------------------------------------------------------------------------------------------
// attention with the projections inside (attention_proj.cuh), one folded batch group
// -------------------------------------------------------------------------------------------------
// the longest sequence attention_proj_kernel<dh> keeps resident (0: no such kernel for this head width)
int attn_proj_max_n(int dh) {
  int best = 0;
  for (int n = APROJ_KB; n <= 4096; n += APROJ_KB) {
    const int st = dh == 64 ? AttnProjSmem<64>::stages_for(n) : (dh == 32 ? AttnProjSmem<32>::stages_for(n) : 0);
    if (st) best = n;
  }
  return best;
}

// Whether an attention call can take the fused kernel: head width 32 or 64, every key resident in shared memory, and the
// TMA operands 16-byte aligned.  The rest (and the tied-query and strict paths, which never ask) run the projection GEMMs
// and attention_tc_kernel.
bool attn_proj_ok(int dh, int n, const void* xn, const void* w_qkv, const void* w_gate) {
  return (dh == 32 || dh == 64) && n >= 1 && n <= attn_proj_max_n(dh) && aligned16(xn) && aligned16(w_qkv) && aligned16(w_gate);
}

template <int DH>
int launch_attention_proj_inst(const CUtensorMap& tx, const CUtensorMap& tw, const CUtensorMap& tg, AttnProjParams p,
                               cudaStream_t s) {
  using L = AttnProjSmem<DH>;
  static int configured[MAX_DEVICES] = {0};
  auto kern = attention_proj_kernel<DH>;
  p.stages = L::stages_for(p.n);
  if (p.stages == 0) return fail(AF2_ERR_BAD_ARG, "attention_proj: sequence length %d too long", p.n);
  const int smem = L::bytes(p.n, p.stages);
  if (smem > configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured[cur_dev()] = smem;
  }
  const long long items = (long long)p.heads * p.nbatch;
  if (items <= 0) return AF2_OK;
  const int grid = (int)(items < sm_count() ? items : sm_count());
  if (items > 0x7fffffffLL - grid) return fail(AF2_ERR_BAD_ARG, "attention_proj: too many work items");
  // algorithmic: the four projections (q, k, v, gate) plus QK^T and PV; xn read once, og written once, the bias once
  const double tokens = (double)p.n * p.nbatch, I = (double)p.heads * DH;
  ProfScope ps(s, KC_ATTENTION, 2.0 * tokens * p.d * 4.0 * I + 4.0 * tokens * p.n * I,
               tokens * p.d * 2.0 + tokens * I * 2.0 + 4.0 * I * p.d * 2.0 + (p.has_bias ? (double)p.heads * p.n * p.n * 2 : 0));
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(APROJ_THREADS), smem, s, tx, tw, tg, p));
  return AF2_OK;
}

// xn: bf16 [tokens, d] (the LayerNorm output), token(b', i) = b' * tok_sb + i * tok_si; w_qkv bf16 [3I, d] (q rows pre-scaled),
// w_gate bf16 [I, d], b_gate fp32 [I] or null; out bf16 [tokens, I].  The caller checks attn_proj_ok.
int launch_attention_proj(const __nv_bfloat16* xn, int d, const __nv_bfloat16* w_qkv, const __nv_bfloat16* w_gate,
                          const float* b_gate, int heads, int dh, int n, int nbatch, long long tok_sb, long long tok_si,
                          const __nv_bfloat16* bias, int npad, const uint8_t* mask, __nv_bfloat16* out, cudaStream_t s) {
  const long long I = (long long)heads * dh;
  CUtensorMap tx, tw, tg;
  const unsigned long long dx[3] = {(unsigned long long)d, (unsigned long long)n, (unsigned long long)nbatch};
  const unsigned long long sx[2] = {(unsigned long long)(tok_si * d * 2), (unsigned long long)(tok_sb * d * 2)};
  const unsigned bx[3] = {64, APROJ_TOK, 1};
  AF2_TRY(make_tmap(&tx, xn, 3, dx, sx, bx, CU_TENSOR_MAP_SWIZZLE_128B));
  const unsigned long long dw[2] = {(unsigned long long)d, (unsigned long long)(3 * I)}, dg[2] = {(unsigned long long)d, (unsigned long long)I};
  const unsigned long long sw[1] = {(unsigned long long)d * 2};
  const unsigned bw[2] = {64, (unsigned)dh};
  AF2_TRY(make_tmap(&tw, w_qkv, 2, dw, sw, bw, CU_TENSOR_MAP_SWIZZLE_128B));
  AF2_TRY(make_tmap(&tg, w_gate, 2, dg, sw, bw, CU_TENSOR_MAP_SWIZZLE_128B));
  if (bias && npad % 2 != 0) return fail(AF2_ERR_BAD_ARG, "attention_proj: bias pitch %d must be even", npad);
  AttnProjParams p;
  memset(&p, 0, sizeof(p));
  p.n = n; p.heads = heads; p.nbatch = nbatch; p.d = d; p.has_bias = bias != nullptr; p.bias = bias; p.npad = npad;
  p.mask = mask; p.mask_sb = tok_sb; p.mask_si = tok_si; p.b_gate = b_gate;
  p.out = out; p.tok_sb = tok_sb; p.tok_si = tok_si; p.ld_out = I;
  return dh == 64 ? launch_attention_proj_inst<64>(tx, tw, tg, p, s) : launch_attention_proj_inst<32>(tx, tw, tg, p, s);
}

// OuterMean normaliser of pair rows [row0, row0 + rows) of one batch element (quirk Q3): bit-packed kernel when the packed
// mask fits in shared memory, else the byte-loop kernel
// variant: 0 the choice above, 1 the byte-loop kernel, 2 the bit-packed pair (needs `words` and the shared-memory fit);
// *ran <- the variant launched (0: none)
int launch_outer_scale(const uint8_t* mask, float* scale, uint32_t* words, int row0, int rows, int S, int N, float eps, cudaStream_t s,
                       int variant = 0, int* ran = nullptr);

int ew_grid(long long n) {
  long long b = (n + 255) / 256;
  long long cap = (long long)sm_count() * 8;
  return (int)(b < cap ? (b > 0 ? b : 1) : cap);
}

// tied queries (alphafold2.py:142-151): q <- mean over the nbatch folded rows / columns, in place in the projection
// buf [tokens][ld] (its first `cols` columns); T = bf16 (default path) or float (strict mode)
template <class T>
int tie_queries(T* buf, long long ld, int cols, int n, int nbatch, long long tok_sb, long long tok_si, cudaStream_t s) {
  ProfScope ps(s, KC_MISC, 0.0, 0.0);
  tie_queries_kernel<T><<<ew_grid((long long)n * cols), 256, 0, s>>>(buf, ld, cols, n, nbatch, tok_sb, tok_si);
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

int launch_outer_scale(const uint8_t* mask, float* scale, uint32_t* words, int row0, int rows, int S, int N, float eps, cudaStream_t s,
                       int variant, int* ran) {
  if (ran) *ran = 0;
  const long long T = (long long)rows * N;
  if (T <= 0) return AF2_OK;
  const int nw = (S + 31) / 32;
  const size_t smem = (size_t)nw * N * 4;
  const bool bits_ok = words && smem <= 160 * 1024;
  if (variant == 2 && !bits_ok)
    return fail(AF2_ERR_BAD_ARG, "outer_scale: bit-packed kernel needs the words workspace and %zu <= %d bytes of shared memory", smem, 160 * 1024);
  const bool bits = variant == 2 || (variant == 0 && bits_ok);
  if (ran) *ran = bits ? 2 : 1;
  ProfScope ps(s, KC_MISC, 0.0, 0.0);
  if (bits) {
    static size_t configured[MAX_DEVICES] = {0};
    if (smem > 48 * 1024 && smem > configured[cur_dev()]) {
      CUDA_OK(cudaFuncSetAttribute(outer_scale_bits_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured[cur_dev()] = smem;
    }
    mask_pack_bits_kernel<<<ew_grid((long long)nw * N), 256, 0, s>>>(mask, words, S, N);
    CUDA_OK(cudaGetLastError());
    const long long need = (T + 255) / 256;
    const int grid = (int)(need < sm_count() ? need : sm_count());
    outer_scale_bits_kernel<<<grid, 256, smem, s>>>(words, scale, row0, rows, S, N, eps);
  } else {
    outer_scale_rows_kernel<<<ew_grid(T), 256, 0, s>>>(mask, scale, row0, rows, S, N, eps);
  }
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

// -------------------------------------------------------------------------------------------------
// module stages shared by the whole-module and the stage-level entry points
// -------------------------------------------------------------------------------------------------
// TriangleMultiply front of `tokens` tokens of x (a grid of rows x inner): LN(x) -> xn; left / right = (proj + b) * mask *
// sigmoid(gate + b) -> channel-major Lc, Rc [c][chan_stride] (token t at (t / inner) * pitch + t % inner, pad columns zeroed);
// sigmoid(out_gate) -> gate [tokens][d].  xn [tokens][d] and maskf [tokens] are workspace.
// gate = bf16(sigmoid(xn w_ogate^T + b_ogate)) [tokens][d]: the triangle out gate (EK_STORE_TOK_SIG)
int launch_out_gate(const void* xn, const void* w_ogate, const float* b_ogate, long long tokens, int d, void* gate, cudaStream_t s) {
  GemmCall cg = linear_call(xn, d, w_ogate, d, (int)tokens, d, d);
  cg.mode = EPI_STORE_BF16; cg.act = ACT_SIGMOID; cg.layout = LAYOUT_TOKEN; cg.out = gate; cg.ld_out = d; cg.bias = b_ogate;
  return launch_gemm(cg, s);
}

// out_gate = false: the out gate is left to the tail (contract_tail with a TailGateProj), which projects it from xn itself
int triangle_front(const af2_trimul_weights* w, const float* x, const unsigned char* mask, long long tokens, int inner, int pitch,
                   int d, __nv_bfloat16* xn, float* maskf, void* Lc, void* Rc, long long chan_stride, void* gate, cudaStream_t s,
                   bool out_gate = true) {
  LnParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.x = x; lp.gamma = w->ln_gamma; lp.beta = w->ln_beta; lp.y = xn; lp.T = tokens; lp.d = d; lp.eps = 1e-5f;
  AF2_TRY(launch_layernorm(lp, s));
  if (mask) {
    { ProfScope ps(s, KC_MISC, 0.0, 0.0); mask_to_float_kernel<<<ew_grid(tokens), 256, 0, s>>>(mask, maskf, tokens); }
    CUDA_OK(cudaGetLastError());
  }
  if (pitch != inner) {   // pad columns of the channel-major operands are read by TMA as K / MN padding: keep them zero
    const long long span = tokens / inner * pitch;   // this call's rows of one channel
    if (chan_stride == span) {
      CUDA_OK(cudaMemsetAsync(Lc, 0, (size_t)d * chan_stride * 2, s));
      CUDA_OK(cudaMemsetAsync(Rc, 0, (size_t)d * chan_stride * 2, s));
    } else {                // a band of rows inside larger operands: only its own rows, other bands' rows stay as they are
      CUDA_OK(cudaMemset2DAsync(Lc, (size_t)chan_stride * 2, 0, (size_t)span * 2, (size_t)d, s));
      CUDA_OK(cudaMemset2DAsync(Rc, (size_t)chan_stride * 2, 0, (size_t)span * 2, (size_t)d, s));
    }
  }
  const int half = w->bn / 2;
  const int npk = (d + half - 1) / half * w->bn;
  for (int side = 0; side < 2; ++side) {
    GemmCall c = linear_call(xn, d, side ? w->w_right : w->w_left, d, (int)tokens, npk, d);
    c.bn = w->bn; c.mode = EPI_GATED_BF16; c.act = ACT_SIGMOID; c.layout = LAYOUT_CHANNEL;
    c.out = side ? Rc : Lc; c.ld_out = chan_stride; c.bias = side ? w->b_right : w->b_left;
    c.use_rowscale = mask != nullptr; c.rowscale = maskf; c.cm_inner = inner; c.cm_pitch = pitch; c.out_cols = d;
    AF2_TRY(launch_gemm(c, s));
  }
  return out_gate ? launch_out_gate(xn, w->w_ogate, w->b_ogate, tokens, d, gate, s) : AF2_OK;
}

// OuterMean front of `tokens` MSA tokens of m (a grid of rows x inner): [left | right] = (LN(m) W^T + b) * mask ->
// channel-major LRc [2d][chan_stride] (layout as in triangle_front).  mn [tokens][d] and maskf [tokens] are workspace.
int outer_front(const af2_outer_weights* w, const float* m, const unsigned char* msa_mask, long long tokens, int inner, int pitch,
                int d, __nv_bfloat16* mn, float* maskf, void* LRc, long long chan_stride, cudaStream_t s) {
  LnParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.x = m; lp.gamma = w->ln_gamma; lp.beta = w->ln_beta; lp.y = mn; lp.T = tokens; lp.d = d; lp.eps = 1e-5f;
  AF2_TRY(launch_layernorm(lp, s));
  if (msa_mask) {
    { ProfScope ps(s, KC_MISC, 0.0, 0.0); mask_to_float_kernel<<<ew_grid(tokens), 256, 0, s>>>(msa_mask, maskf, tokens); }
    CUDA_OK(cudaGetLastError());
  }
  if (pitch != inner) {   // pad columns are read by TMA as MN padding of the contraction: keep them zero
    const long long span = tokens / inner * pitch;   // this call's MSA rows of one channel
    if (chan_stride == span) {
      CUDA_OK(cudaMemsetAsync(LRc, 0, (size_t)2 * d * chan_stride * 2, s));
    } else {                // a chunk of MSA rows inside a larger operand: only its own rows, other chunks' rows stay as they are
      CUDA_OK(cudaMemset2DAsync(LRc, (size_t)chan_stride * 2, 0, (size_t)span * 2, (size_t)2 * d, s));
    }
  }
  GemmCall c = linear_call(mn, d, w->w_lr, d, (int)tokens, 2 * d, d);
  c.mode = EPI_STORE_BF16; c.layout = LAYOUT_CHANNEL; c.out = LRc; c.ld_out = chan_stride; c.bias = w->b_lr;
  c.use_rowscale = msa_mask != nullptr; c.rowscale = maskf; c.cm_inner = inner; c.cm_pitch = pitch;
  return launch_gemm(c, s);
}

ChanLnParams chan_ln_params(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode,
                            const float* gamma, const float* beta, const void* gate, const float* scale,
                            float scale_const, float eps, void* y) {
  ChanLnParams p;
  memset(&p, 0, sizeof(p));
  p.src = src; p.chan_stride = chan_stride; p.pitch = pitch; p.rows = rows; p.n = n; p.d = d; p.mode = mode;
  p.gamma = gamma; p.beta = beta; p.gate = static_cast<const __nv_bfloat16*>(gate); p.scale = scale;
  p.scale_const = scale_const; p.eps = eps; p.y = static_cast<__nv_bfloat16*>(y);
  return p;
}

// The out gate of a whole-module triangle multiply, projected by the tail from the front's LayerNorm output:
// gate = bf16(sigmoid(xn w^T + b)).  The unfused tail launches that GEMM into cp.gate first.
struct TailGateProj {
  const void* xn;     // [tokens][d] bf16
  const void* w;      // [d][d] bf16
  const float* b;     // [d] or nullptr
};

template <int D, int V>
int launch_contract_tail(const ChanLnParams& cp, const TailGateProj* gp, const void* w_out, const float* b_out, float* x,
                         long long T, cudaStream_t s) {
  using L = CtailSmem<D>;
  static bool configured[MAX_DEVICES] = {false};
  auto kern = contract_tail_kernel<D, V>;
  if (!configured[cur_dev()]) {
    CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::TOTAL));
    configured[cur_dev()] = true;
  }
  const void* g = V == CT_GATE_PROJECT ? gp->xn : (V == CT_GATE_LOAD ? static_cast<const void*>(cp.gate) : nullptr);
  CUtensorMap to, tg, twg, two;
  {
    const unsigned long long dO[2] = {(unsigned long long)T, (unsigned long long)D}, sO[1] = {(unsigned long long)cp.chan_stride * 4};
    const unsigned bO[2] = {CT_TOK, (unsigned)D};
    AF2_TRY(make_tmap(&to, cp.src, 2, dO, sO, bO, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_DATA_TYPE_FLOAT32));
    const unsigned long long dW[2] = {(unsigned long long)D, (unsigned long long)D}, sW[1] = {(unsigned long long)D * 2};
    const unsigned bW[2] = {64, (unsigned)D};
    AF2_TRY(make_tmap(&two, w_out, 2, dW, sW, bW, CU_TENSOR_MAP_SWIZZLE_128B));
    if (V == CT_GATE_PROJECT) AF2_TRY(make_tmap(&twg, gp->w, 2, dW, sW, bW, CU_TENSOR_MAP_SWIZZLE_128B));
    else twg = two;
    if (g) {
      const unsigned long long dG[2] = {(unsigned long long)D, (unsigned long long)T}, sG[1] = {(unsigned long long)D * 2};
      const unsigned bG[2] = {64, CT_TOK};
      AF2_TRY(make_tmap(&tg, g, 2, dG, sG, bG, CU_TENSOR_MAP_SWIZZLE_128B));
    } else {
      tg = to;
    }
  }
  CtailParams q;
  q.x = x; q.b_ogate = V == CT_GATE_PROJECT ? gp->b : nullptr; q.b_out = b_out; q.gamma = cp.gamma; q.beta = cp.beta;
  q.scale = cp.scale; q.scale_const = cp.scale_const; q.eps = cp.eps; q.T = (int)T;
  const long long tiles = (T + CT_TOK - 1) / CT_TOK;
  const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
  const int ngemm = V == CT_GATE_PROJECT ? 2 : 1;
  const double flops = 2.0 * ngemm * T * D * (double)D;
  // O, xn / gate, x read + written, the weights once
  const double bytes = (double)T * D * (4.0 + (V == CT_SCALE ? 0.0 : 2.0) + 8.0) + ngemm * (double)D * D * 2;
  ProfScope ps(s, KC_GEMM_LINEAR, flops, bytes);
  CUDA_OK(launch_pdl(kern, dim3(grid), dim3(CT_THREADS), L::TOTAL, s, to, tg, twg, two, q));
  return AF2_OK;
}

// The fused tail runs exactly where launch_chan_to_token would take the TMA kernel and the weights, x and (projected
// gate) xn are TMA-addressable; every other call keeps the chan_to_token + to_out GEMM launches.
bool contract_tail_fused_ok(const ChanLnParams& cp, const void* w_out, const float* x, const TailGateProj* gp) {
  return c2t_variant_ok(cp, C2T_TMA) && aligned16(w_out) && aligned16(x) && (!gp || (aligned16(gp->xn) && aligned16(gp->w)));
}

enum CtailPath { CTAIL_AUTO = 0, CTAIL_UNFUSED = 1, CTAIL_FUSED = 2 };

// tail of the triangle / outer-product contractions: x [rows * n][d] += tail(O) w_out^T + b_out, tail(O) as
// launch_chan_to_token makes it (with the out gate projected from gp->xn first when gp is given).  Fused: one
// contract_tail_kernel launch; unfused: [out-gate GEMM,] chan_to_token into cp.y, to_out GEMM.  *ran <- the path taken.
int contract_tail(const ChanLnParams& cp, const void* w_out, const float* b_out, float* x, cudaStream_t s,
                  const TailGateProj* gp = nullptr, int path = CTAIL_AUTO, int* ran = nullptr) {
  if (ran) *ran = 0;
  const long long T = (long long)cp.rows * cp.n;
  const bool fused_ok = contract_tail_fused_ok(cp, w_out, x, gp);
  if (path == CTAIL_FUSED && !fused_ok)
    return fail(AF2_ERR_BAD_ARG, "contract_tail: the fused tail cannot run d=%d rows=%d n=%d pitch=%d chan_stride=%lld", cp.d,
                cp.rows, cp.n, cp.pitch, cp.chan_stride);
  if (gp && cp.mode != 0) return fail(AF2_ERR_BAD_ARG, "contract_tail: a projected gate needs mode 0");
  const int d = cp.d;
  if (path != CTAIL_UNFUSED && fused_ok) {
    if (ran) *ran = CTAIL_FUSED;
    if (T <= 0) return AF2_OK;
    if (cp.mode == 1)
      return d == 256 ? launch_contract_tail<256, CT_SCALE>(cp, gp, w_out, b_out, x, T, s)
                      : launch_contract_tail<128, CT_SCALE>(cp, gp, w_out, b_out, x, T, s);
    if (gp)
      return d == 256 ? launch_contract_tail<256, CT_GATE_PROJECT>(cp, gp, w_out, b_out, x, T, s)
                      : launch_contract_tail<128, CT_GATE_PROJECT>(cp, gp, w_out, b_out, x, T, s);
    return d == 256 ? launch_contract_tail<256, CT_GATE_LOAD>(cp, gp, w_out, b_out, x, T, s)
                    : launch_contract_tail<128, CT_GATE_LOAD>(cp, gp, w_out, b_out, x, T, s);
  }
  if (ran) *ran = CTAIL_UNFUSED;
  if (gp) AF2_TRY(launch_out_gate(gp->xn, gp->w, gp->b, T, d, const_cast<__nv_bfloat16*>(cp.gate), s));
  AF2_TRY(launch_chan_to_token(cp, s));
  GemmCall co = linear_call(cp.y, d, w_out, d, (int)T, d, d);
  co.mode = EPI_RESID_F32; co.out = x; co.ld_out = d; co.bias = b_out; co.resid = x; co.ld_resid = d;
  return launch_gemm(co, s);
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

const char* af2_last_error(void) { return g_err; }
int af2_abi_version(void) { return 5; }

unsigned long long af2_launch_count(void) { return g_launches; }

void af2_profile_enable(int on) {
  g_prof = on != 0;
  if (g_prof) {
    for (auto& r : g_recs) { g_pool.push_back(r.a); g_pool.push_back(r.b); }
    g_recs.clear();
  }
}

// Sums the recorded launches of kernel class `cls` (synchronises the device). Returns the launch count.
long long af2_profile_read(int cls, double* ms, double* flops, double* bytes) {
  cudaDeviceSynchronize();
  double t = 0, f = 0, b = 0;
  long long n = 0;
  for (auto& r : g_recs) {
    if (r.cls != cls) continue;
    float e = 0.f;
    if (cudaEventElapsedTime(&e, r.a, r.b) == cudaSuccess) t += e;
    f += r.flops; b += r.bytes; ++n;
  }
  if (ms) *ms = t;
  if (flops) *flops = f;
  if (bytes) *bytes = b;
  return n;
}

int af2_check_device(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(AF2_ERR_CUDA, "no CUDA device");
  int major = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  int minor = 0;
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0)
    return fail(AF2_ERR_UNSUPPORTED_DEVICE, "libaf2b200 is built for sm_90a only; device has compute capability %d.%d", major, minor);
  return AF2_OK;
}

// ------------------------------------------------------------------------------------------------
long long af2_feed_forward_workspace(long long tokens, int d, int hidden) {
  return align_up(tokens * d * 2, 256) + align_up(tokens * hidden * 2, 256) + 1024;
}

int af2_feed_forward(const af2_ff_weights* w, float* x, long long tokens, int d, int hidden, void* workspace,
                     long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_feed_forward");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x) return fail(AF2_ERR_BAD_ARG, "feed_forward: null argument");
  if (d % 8 || hidden % 8) return fail(AF2_ERR_BAD_ARG, "feed_forward: d=%d and hidden=%d must be multiples of 8", d, hidden);
  if (tokens > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "feed_forward: too many tokens");
  Arena ar(workspace, workspace_bytes);
  __nv_bfloat16* xn = ar.take<__nv_bfloat16>(tokens * d);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "feed_forward: workspace too small");
  LnParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.x = x; lp.gamma = w->ln_gamma; lp.beta = w->ln_beta; lp.y = xn; lp.T = tokens; lp.d = d; lp.eps = 1e-5f;
  if (ff_fused_ok(w, x, xn, d, hidden)) {
    AF2_TRY(launch_layernorm(lp, s));
    // 64 hidden units per chunk: 32 measured slower (n64 GEMM1 tiles read more shared memory per FLOP)
    return d == 256 ? launch_ff_fused<256, 64>(w, x, xn, tokens, hidden, s) : launch_ff_fused<128, 64>(w, x, xn, tokens, hidden, s);
  }
  __nv_bfloat16* hbuf = ar.take<__nv_bfloat16>(tokens * hidden);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "feed_forward: workspace too small");
  // h = a * gelu(g)
  const int half = w->bn / 2;
  const int n1p = (hidden + half - 1) / half * w->bn;   // packed accumulator columns
  AF2_TRY(launch_layernorm(lp, s));
  GemmCall c1 = linear_call(xn, d, w->w1, d, (int)tokens, n1p, d);
  c1.bn = w->bn; c1.mode = EPI_GATED_BF16; c1.act = ACT_GELU; c1.layout = LAYOUT_TOKEN;
  c1.out = hbuf; c1.ld_out = hidden; c1.bias = w->b1; c1.out_cols = hidden;
  AF2_TRY(launch_gemm(c1, s));
  GemmCall c2 = linear_call(hbuf, hidden, w->w2, hidden, (int)tokens, d, hidden);
  c2.mode = EPI_RESID_F32; c2.out = x; c2.ld_out = d; c2.bias = w->b2; c2.resid = x; c2.ld_resid = d;
  AF2_TRY(launch_gemm(c2, s));
  return AF2_OK;
}

// ------------------------------------------------------------------------------------------------
long long af2_axial_attention_workspace(int B, int h, int wdim, int d, int heads, int dim_head, int row_attn) {
  const long long T = (long long)B * h * wdim, I = (long long)heads * dim_head;
  const int n = row_attn ? wdim : h;
  const long long npad = align_up(n, 8);
  return align_up(T * d * 2, 256) + align_up(T * 3 * I * 2, 256) + 2 * align_up(T * I * 2, 256) +
         align_up((long long)B * heads * n * npad * 2, 256) + 1024;
}

// One axial attention call: its shape and its workspace carve-up (af2_axial_attention_workspace).  The whole-call entry points
// run axial_project and axial_attend on one plan; the tied-query pair af2_axial_attention_tied_begin / _end runs them in two
// calls on the same workspace, with the cross-shard query mean between them.
struct AxialPlan {
  long long T, I;
  int n, nb, npad;
  bool has_bias;
  bool fused;   // attention_proj_kernel projects q, k, v and the gate: the q|k|v and gate slices stay unused
  __nv_bfloat16 *xn, *qkv, *gate, *og, *bias;
};

static int axial_plan(AxialPlan& p, const af2_attn_weights* w, const float* x, const float* edges, const void* pre_bias, int B,
                      int h, int wdim, int d, int heads, int dim_head, int row_attn, void* workspace, long long workspace_bytes) {
  if (!w || !x) return fail(AF2_ERR_BAD_ARG, "axial_attention: null argument");
  if (!attention_dim_head_ok(dim_head)) return fail(AF2_ERR_BAD_ARG, "axial_attention: " DIM_HEAD_UNSUPPORTED, dim_head);
  if (d % 8) return fail(AF2_ERR_BAD_ARG, "axial_attention: dim %d must be a multiple of 8", d);
  p.T = (long long)B * h * wdim; p.I = (long long)heads * dim_head;
  if (p.T > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "axial_attention: too many tokens");
  p.n = row_attn ? wdim : h;
  p.nb = row_attn ? h : wdim;
  p.npad = (int)align_up(p.n, 8);
  p.has_bias = pre_bias != nullptr || (edges != nullptr && w->w_edge != nullptr);
  p.fused = false;
  Arena ar(workspace, workspace_bytes);
  p.xn = ar.take<__nv_bfloat16>(p.T * d);
  p.qkv = ar.take<__nv_bfloat16>(p.T * 3 * p.I);
  p.gate = ar.take<__nv_bfloat16>(p.T * p.I);
  p.og = ar.take<__nv_bfloat16>(p.T * p.I);
  p.bias = ar.take<__nv_bfloat16>((long long)B * heads * p.n * p.npad);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "axial_attention: workspace too small");
  if (pre_bias) p.bias = const_cast<__nv_bfloat16*>(static_cast<const __nv_bfloat16*>(pre_bias));   // [B][H][n][npad], zero padded
  return AF2_OK;
}

// 1. LayerNorm (+ pair bias from the raw edges) and 2. the q|k|v and gate projections into the plan's workspace
static int axial_project(const AxialPlan& p, const af2_attn_weights* w, float* x, const float* edges, const void* pre_bias,
                         int B, int d, int heads, cudaStream_t s) {
  const long long T = p.T, I = p.I;
  const int n = p.n, npad = p.npad;
  const bool has_bias = p.has_bias;
  __nv_bfloat16 *xn = p.xn, *qkv = p.qkv, *gate = p.gate, *bias = p.bias;
  // 1. LayerNorm (+ pair bias from the RAW edges; fused when the edges are x itself)
  LnParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.x = x; lp.gamma = w->ln_gamma; lp.beta = w->ln_beta; lp.y = xn; lp.T = T; lp.d = d; lp.eps = 1e-5f;
  const bool fuse_bias = has_bias && !pre_bias && edges == x && B == 1;
  // pad key columns of the bias rows are never read, but keep them finite (zero)
  if (has_bias && !pre_bias && npad != n) CUDA_OK(cudaMemsetAsync(bias, 0, (size_t)B * heads * n * npad * 2, s));
  if (fuse_bias && pair_bias_fast_ok(d, heads)) {
    // pair bias from the raw x by the dedicated kernel (the one the sharded schedule uses), LayerNorm without it
    AF2_TRY(launch_pair_bias(x, T, d, w->w_edge, bias, heads, (long long)n * npad, n, npad, s));
  } else if (fuse_bias) {
    lp.wb = w->w_edge; lp.bias_out = bias; lp.heads = heads; lp.bias_hs = (long long)n * npad; lp.n_inner = n; lp.pitch = npad;
  }
  AF2_TRY(launch_layernorm(lp, s));
  if (has_bias && !fuse_bias && !pre_bias && pair_bias_fast_ok(d, heads)) {
    for (int b = 0; b < B; ++b)
      AF2_TRY(launch_pair_bias(edges + (long long)b * n * n * d, (long long)n * n, d, w->w_edge, bias + (long long)b * heads * n * npad,
                               heads, (long long)n * npad, n, npad, s));
  } else if (has_bias && !fuse_bias && !pre_bias) {
    for (int b = 0; b < B; ++b) {
      LnParams bp;
      memset(&bp, 0, sizeof(bp));
      bp.x = edges + (long long)b * n * n * d; bp.T = (long long)n * n; bp.d = d; bp.eps = 1e-5f;
      bp.wb = w->w_edge; bp.bias_out = bias + (long long)b * heads * n * npad; bp.heads = heads;
      bp.bias_hs = (long long)n * npad; bp.n_inner = n; bp.pitch = npad;
      AF2_TRY(launch_layernorm(bp, s));
    }
  }
  // 2. projections (the fused attention kernel makes its own)
  if (p.fused) return AF2_OK;
  GemmCall cq = linear_call(xn, d, w->w_qkv, d, (int)T, (int)(3 * I), d);
  cq.mode = EPI_STORE_BF16; cq.layout = LAYOUT_TOKEN; cq.out = qkv; cq.ld_out = 3 * I;
  AF2_TRY(launch_gemm(cq, s));
  GemmCall cg = linear_call(xn, d, w->w_gate, d, (int)T, (int)I, d);
  cg.mode = EPI_STORE_BF16; cg.act = ACT_SIGMOID; cg.layout = LAYOUT_TOKEN; cg.out = gate; cg.ld_out = I; cg.bias = w->b_gate;
  return launch_gemm(cg, s);
}

// 3. attention per batch element (queries tied first when `tied`; projected inside the kernel when the plan is fused) and
// 4. to_out + bias + residual into x
static int axial_attend(const AxialPlan& p, const af2_attn_weights* w, float* x, const unsigned char* mask, int B, int h,
                        int wdim, int d, int heads, int dim_head, int row_attn, int tied, cudaStream_t s) {
  const long long T = p.T, I = p.I;
  const int n = p.n, nb = p.nb, npad = p.npad;
  const long long tok_sb = row_attn ? wdim : 1, tok_si = row_attn ? 1 : wdim;
  for (int b = 0; b < B; ++b) {
    const long long t0 = (long long)b * h * wdim;
    // MSAColumnGlobalAttention-style tied queries (alphafold2.py:142-151): q <- mean over the folded batch
    if (p.fused) {
      AF2_TRY(launch_attention_proj(p.xn + t0 * d, d, static_cast<const __nv_bfloat16*>(w->w_qkv),
                                    static_cast<const __nv_bfloat16*>(w->w_gate), w->b_gate, heads, dim_head, n, nb, tok_sb, tok_si,
                                    p.has_bias ? p.bias + (long long)b * heads * n * npad : nullptr, npad, mask ? mask + t0 : nullptr,
                                    p.og + t0 * I, s));
      continue;
    }
    if (tied) AF2_TRY(tie_queries<__nv_bfloat16>(p.qkv + t0 * 3 * I, 3 * I, (int)I, n, nb, tok_sb, tok_si, s));
    AF2_TRY(launch_attention(p.qkv + t0 * 3 * I, heads, dim_head, n, nb, tok_sb, tok_si,
                             p.has_bias ? p.bias + (long long)b * heads * n * npad : nullptr, npad,
                             mask ? mask + t0 : nullptr, p.gate + t0 * I, p.og + t0 * I, s));
  }
  // 4. to_out + bias + residual
  GemmCall co = linear_call(p.og, I, w->w_out, I, (int)T, d, (int)I);
  co.mode = EPI_RESID_F32; co.out = x; co.ld_out = d; co.bias = w->b_out; co.resid = x; co.ld_resid = d;
  AF2_TRY(launch_gemm(co, s));
  return AF2_OK;
}

static int axial_attention_impl(const af2_attn_weights* w, float* x, const float* edges, const void* pre_bias,
                                const unsigned char* mask, int B, int h, int wdim, int d, int heads, int dim_head,
                                int row_attn, void* workspace, long long workspace_bytes, af2_stream_t stream, int tied = 0) {
  NvtxRange nvtx_(row_attn ? "af2_axial_attention(row)" : "af2_axial_attention(col)");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AxialPlan p;
  AF2_TRY(axial_plan(p, w, x, edges, pre_bias, B, h, wdim, d, heads, dim_head, row_attn, workspace, workspace_bytes));
  p.fused = !tied && attn_proj_ok(dim_head, p.n, p.xn, w->w_qkv, w->w_gate);
  AF2_TRY(axial_project(p, w, x, edges, pre_bias, B, d, heads, s));
  return axial_attend(p, w, x, mask, B, h, wdim, d, heads, dim_head, row_attn, tied, s);
}

// the sharded tied-query column attention: the checks shared by af2_axial_attention_tied_begin and _end
static int tied_args_ok(const af2_attn_weights* w, const float* x, const void* sums, const void* workspace, int h, int wdim) {
  if (!w || !x || !sums || !workspace) return fail(AF2_ERR_BAD_ARG, "axial_attention_tied: null argument");
  if (h < 1 || wdim < 1) return fail(AF2_ERR_BAD_ARG, "axial_attention_tied: empty shard h=%d wdim=%d", h, wdim);
  return AF2_OK;
}

// ------------------------------------------------------------------------------------------------
// per-channel contractions of the triangle multiplications and the outer mean
// ------------------------------------------------------------------------------------------------
// The contraction's fp32 product Oc [d][rows][pitch] (pitch = align4(cols), channel stride cs) and the tail's bf16 tokens
// tn [rows * cols][d], taken from the workspace in this order.
struct ContractOut {
  float* Oc; __nv_bfloat16* tn; int pitch; long long cs;
};

static ContractOut take_contract_out(Arena& ar, int rows, int cols, int d) {
  ContractOut o;
  o.pitch = (int)align_up(cols, 4);
  o.cs = (long long)rows * o.pitch;
  o.Oc = ar.take<float>(d * o.cs);
  o.tn = ar.take<__nv_bfloat16>((long long)rows * cols * d);
  return o;
}

// O_c = A_c B_c^T for every channel c < d into Oc [c][M][ld_o] (channel stride cs_o), one batched GEMM over the channels.
//   K-major (mn_major = 0): A [c][M][lda], B [c][N][ldb], k < K;   MN-major: A [c][K][lda] (i < M), B [c][K][ldb] (j < N).
// Channel c of A (B) starts cs_a (cs_b) elements after channel c - 1.  A (gather_a) or B may be `pieces` gathered shards,
// piece_stride elements apart, each holding M / pieces rows (A) or N / pieces columns (B) of O with the pitch lda (ldb).
// One launch addresses all pieces through rank-4 tensor maps when a piece tiles the kernel's boxes (MN-major pieces of whole
// 64-wide boxes, K-major B pieces of a multiple of 8 rows that tile BN); otherwise each piece is its own launch.
static int launch_contract(const void* A, long long lda, long long cs_a, const void* B, long long ldb, long long cs_b,
                           bool mn_major, int M, int N, int K, int d, int pieces, bool gather_a, long long piece_stride,
                           float* Oc, int ld_o, long long cs_o, cudaStream_t s) {
  GemmCall c;
  memset(&c, 0, sizeof(c));
  c.A = A; c.lda = lda; c.a_batch = cs_a; c.Bm = B; c.ldb = ldb; c.b_batch = cs_b; c.mn_major = mn_major;
  c.M = M; c.N = N; c.K = K; c.batch = d; c.bn = pick_bn(N);
  c.mode = EPI_STORE_F32; c.layout = LAYOUT_TOKEN; c.out = Oc; c.ld_out = ld_o; c.out_batch = cs_o;
  const int pw = (gather_a ? M : N) / pieces;
  if (pieces > 1 && (mn_major ? pw % 64 == 0 : !gather_a && pw % 8 == 0 && (pw % c.bn == 0 || c.bn % pw == 0))) {
    if (gather_a) { c.a_pr = pw; c.a_piece = piece_stride; }
    else { c.b_pr = pw; c.b_piece = piece_stride; }
    return launch_gemm(c, s);
  }
  const __nv_bfloat16* g = static_cast<const __nv_bfloat16*>(gather_a ? A : B);
  for (int p = 0; p < pieces; ++p) {
    if (gather_a) { c.A = g + p * piece_stride; c.M = pw; c.out = Oc + (long long)p * pw * ld_o; }
    else { c.Bm = g + p * piece_stride; c.N = pw; c.bn = pick_bn(pw); c.out = Oc + (long long)p * pw; }
    AF2_TRY(launch_gemm(c, s));
  }
  return AF2_OK;
}

long long af2_triangle_multiply_workspace(int B, int N, int d) {
  const long long T = (long long)B * N * N;
  const long long np8 = align_up(N, 8), np4 = align_up(N, 4);
  return 3 * align_up(T * d * 2, 256)                               // xn, gate, tn
         + 2 * align_up((long long)d * B * N * np8 * 2, 256)          // Lc, Rc
         + align_up((long long)d * B * N * np4 * 4, 256)              // Oc
         + align_up(T * 4, 256) + 1024;                               // mask as float
}

int af2_triangle_multiply(const af2_trimul_weights* w, float* x, const unsigned char* mask, int B, int N, int d,
                          int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_triangle_multiply");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x) return fail(AF2_ERR_BAD_ARG, "triangle_multiply: null argument");
  if (d % 32) return fail(AF2_ERR_BAD_ARG, "triangle_multiply: dim %d must be a multiple of 32", d);
  const long long T = (long long)B * N * N;
  if (T > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "triangle_multiply: too many tokens");
  const int np8 = (int)align_up(N, 8);
  const long long cs_lr = (long long)B * N * np8;   // channel stride of Lc / Rc
  Arena ar(workspace, workspace_bytes);
  __nv_bfloat16* xn = ar.take<__nv_bfloat16>(T * d);
  __nv_bfloat16* gate = ar.take<__nv_bfloat16>(T * d);
  __nv_bfloat16* Lc = ar.take<__nv_bfloat16>(d * cs_lr);
  __nv_bfloat16* Rc = ar.take<__nv_bfloat16>(d * cs_lr);
  const ContractOut o = take_contract_out(ar, B * N, N, d);
  float* maskf = ar.take<float>(T);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "triangle_multiply: workspace too small");

  // the tail projects the out gate itself when it runs fused: decided here, before the front, with the tail's own predicate
  const ChanLnParams cp = chan_ln_params(o.Oc, o.cs, o.pitch, B * N, N, d, 0, w->on_gamma, w->on_beta, gate, nullptr, 0.f, 1e-5f, o.tn);
  const TailGateProj gp = {xn, w->w_ogate, w->b_ogate};
  const bool project = contract_tail_fused_ok(cp, w->w_out, x, &gp);
  AF2_TRY(triangle_front(w, x, mask, T, N, np8, d, xn, maskf, Lc, Rc, cs_lr, gate, s, !project));
  // outgoing: O_c = L_c R_c^T, both K-major;  ingoing: O_c[i][j] = sum_k R_c[k][i] L_c[k][j], both MN-major
  for (int b = 0; b < B; ++b) {
    const long long boff = (long long)b * N * np8;
    AF2_TRY(launch_contract((ingoing ? Rc : Lc) + boff, np8, cs_lr, (ingoing ? Lc : Rc) + boff, np8, cs_lr, ingoing, N, N, N, d, 1,
                            false, 0, o.Oc + (long long)b * N * o.pitch, o.pitch, o.cs, s));
  }
  // LN over channels * out_gate -> to_out + residual
  return contract_tail(cp, w->w_out, w->b_out, x, s, project ? &gp : nullptr, project ? CTAIL_FUSED : CTAIL_AUTO);
}

// ------------------------------------------------------------------------------------------------
long long af2_outer_mean_workspace(int B, int S, int N, int d) {
  const long long Tm = (long long)B * S * N, Tx = (long long)B * N * N;
  const long long np8 = align_up(N, 8), np4 = align_up(N, 4);
  return align_up(Tm * d * 2, 256) + align_up((long long)2 * d * B * S * np8 * 2, 256) +
         align_up((long long)d * B * N * np4 * 4, 256) + align_up(Tx * d * 2, 256) + align_up(Tm * 4, 256) +
         align_up(Tx * 4, 256) + align_up((long long)((S + 31) / 32) * N * 4, 256) + 1024;
}

int af2_outer_mean(const af2_outer_weights* w, float* x, const float* m, const unsigned char* msa_mask, int B, int S,
                   int N, int d, float eps, void* workspace, long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_outer_mean");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x || !m) return fail(AF2_ERR_BAD_ARG, "outer_mean: null argument");
  if (d % 32) return fail(AF2_ERR_BAD_ARG, "outer_mean: dim %d must be a multiple of 32", d);
  const long long Tm = (long long)B * S * N, Tx = (long long)B * N * N;
  if (Tm > 0x7fffffffLL || Tx > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "outer_mean: too many tokens");
  const int np8 = (int)align_up(N, 8);
  const long long cs_lr = (long long)B * S * np8;
  Arena ar(workspace, workspace_bytes);
  __nv_bfloat16* mn = ar.take<__nv_bfloat16>(Tm * d);
  __nv_bfloat16* LRc = ar.take<__nv_bfloat16>(2LL * d * cs_lr);
  const ContractOut o = take_contract_out(ar, B * N, N, d);
  float* maskf = ar.take<float>(Tm);
  float* scale = ar.take<float>(Tx);
  uint32_t* mwords = ar.take<uint32_t>((long long)((S + 31) / 32) * N);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "outer_mean: workspace too small");

  // the normaliser goes first: launched between the two GEMMs, its kernels would keep the contraction from starting under
  // the projection's tail (programmatic dependent launch)
  if (msa_mask)
    for (int b = 0; b < B; ++b)
      AF2_TRY(launch_outer_scale(msa_mask + (long long)b * S * N, scale + (long long)b * N * N, mwords, 0, N, S, N, eps, s));
  AF2_TRY(outer_front(w, m, msa_mask, Tm, N, np8, d, mn, maskf, LRc, cs_lr, s));
  // O_c[i][j] = sum_s L_c[s][i] R_c[s][j]  (MN-major operands, K = S)
  for (int b = 0; b < B; ++b) {
    const __nv_bfloat16* Lb = LRc + (long long)b * S * np8;
    AF2_TRY(launch_contract(Lb, np8, cs_lr, Lb + (long long)d * cs_lr, np8, cs_lr, true, N, N, S, d, 1, false, 0,
                            o.Oc + (long long)b * N * o.pitch, o.pitch, o.cs, s));
  }
  return contract_tail(chan_ln_params(o.Oc, o.cs, o.pitch, B * N, N, d, 1, nullptr, nullptr, nullptr, msa_mask ? scale : nullptr,
                                      1.0f / (float)S, 0.f, o.tn),
                       w->w_out, w->b_out, x, s);
}


int af2_axial_attention(const af2_attn_weights* w, float* x, const float* edges, const unsigned char* mask, int B,
                        int h, int wdim, int d, int heads, int dim_head, int row_attn, void* workspace,
                        long long workspace_bytes, af2_stream_t stream) {
  return axial_attention_impl(w, x, edges, nullptr, mask, B, h, wdim, d, heads, dim_head, row_attn, workspace,
                              workspace_bytes, stream);
}

// same with flags: bit 0 = tied queries (global_query_attn of the extra-MSA stack, alphafold2.py:142-151, 250)
int af2_axial_attention_ex(const af2_attn_weights* w, float* x, const float* edges, const unsigned char* mask, int B,
                           int h, int wdim, int d, int heads, int dim_head, int row_attn, int flags, void* workspace,
                           long long workspace_bytes, af2_stream_t stream) {
  return axial_attention_impl(w, x, edges, nullptr, mask, B, h, wdim, d, heads, dim_head, row_attn, workspace,
                              workspace_bytes, stream, flags & 1);
}

int af2_axial_attention_prebias(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask,
                                int B, int h, int wdim, int d, int heads, int dim_head, int row_attn, void* workspace,
                                long long workspace_bytes, af2_stream_t stream) {
  return axial_attention_impl(w, x, nullptr, bias_bf16, mask, B, h, wdim, d, heads, dim_head, row_attn, workspace,
                              workspace_bytes, stream);
}

// tied-query column attention of a column shard x [h][wdim][d] (batch 1), in two calls around the caller's collective
int af2_axial_attention_tied_begin(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask, int h,
                                   int wdim, int d, int heads, int dim_head, float* qsum_out, void* workspace,
                                   long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_axial_attention_tied_begin");
  (void)mask;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AF2_TRY(tied_args_ok(w, x, qsum_out, workspace, h, wdim));
  AxialPlan p;
  AF2_TRY(axial_plan(p, w, x, nullptr, bias_bf16, 1, h, wdim, d, heads, dim_head, 0, workspace, workspace_bytes));
  AF2_TRY(axial_project(p, w, x, nullptr, bias_bf16, 1, d, heads, s));
  ProfScope ps(s, KC_MISC, 0.0, 0.0);
  tie_queries_sum_kernel<<<ew_grid((long long)h * p.I), 256, 0, s>>>(p.qkv, 3 * p.I, (int)p.I, h, wdim, 1, wdim, qsum_out);
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

int af2_axial_attention_tied_end(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask, int h,
                                 int wdim, int d, int heads, int dim_head, const float* parts, int nparts, int ncols_total,
                                 void* workspace, long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_axial_attention_tied_end");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  AF2_TRY(tied_args_ok(w, x, parts, workspace, h, wdim));
  if (nparts < 1) return fail(AF2_ERR_BAD_ARG, "axial_attention_tied_end: nparts %d < 1", nparts);
  if (ncols_total < wdim) return fail(AF2_ERR_BAD_ARG, "axial_attention_tied_end: ncols_total %d < wdim %d", ncols_total, wdim);
  AxialPlan p;
  AF2_TRY(axial_plan(p, w, x, nullptr, bias_bf16, 1, h, wdim, d, heads, dim_head, 0, workspace, workspace_bytes));
  {
    ProfScope ps(s, KC_MISC, 0.0, 0.0);
    tie_queries_parts_kernel<<<ew_grid((long long)h * p.I), 256, 0, s>>>(p.qkv, 3 * p.I, (int)p.I, h, wdim, 1, wdim, parts, nparts,
                                                                          ncols_total);
    CUDA_OK(cudaGetLastError());
  }
  return axial_attend(p, w, x, mask, 1, h, wdim, d, heads, dim_head, 0, 0, s);
}

// bias rows of a shard of the pair tensor: out[h][r][j] (pitch npad, caller zero-fills the pad) = <x[r, j, :], w_edge[h, :]>
int af2_pair_bias(const float* x_rows, const float* w_edge, void* bias_out, int rows, int n, int d, int heads,
                  af2_stream_t stream) {
  NvtxRange nvtx_("af2_pair_bias");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!x_rows || !w_edge || !bias_out) return fail(AF2_ERR_BAD_ARG, "pair_bias: null argument");
  const int npad = (int)align_up(n, 8);
  if (pair_bias_fast_ok(d, heads))
    return launch_pair_bias(x_rows, (long long)rows * n, d, w_edge, static_cast<__nv_bfloat16*>(bias_out), heads, (long long)rows * npad,
                            n, npad, s);
  LnParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.x = x_rows; bp.T = (long long)rows * n; bp.d = d; bp.eps = 1e-5f;
  bp.wb = w_edge; bp.bias_out = static_cast<__nv_bfloat16*>(bias_out); bp.heads = heads;
  bp.bias_hs = (long long)rows * npad; bp.n_inner = n; bp.pitch = npad;
  return launch_layernorm(bp, s);
}

// ------------------------------------------------------------------------------------------------
// stage-level triangle multiply (used by the sharded path; pieces = number of gathered operand shards)
// ------------------------------------------------------------------------------------------------
long long af2_triangle_project_workspace(long long tokens, int d) {
  return align_up(tokens * d * 2, 256) + align_up(tokens * 4, 256) + 1024;
}

int af2_triangle_project(const af2_trimul_weights* w, const float* x, const unsigned char* mask, long long tokens,
                         int inner, int d, void* Lc, void* Rc, long long chan_stride, void* gate, void* workspace,
                         long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_triangle_project");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x || !Lc || !Rc || !gate) return fail(AF2_ERR_BAD_ARG, "triangle_project: null argument");
  if (d % 32) return fail(AF2_ERR_BAD_ARG, "triangle_project: dim %d must be a multiple of 32", d);
  if (tokens % inner) return fail(AF2_ERR_BAD_ARG, "triangle_project: tokens must be a multiple of inner");
  const int pitch = (int)align_up(inner, 8);
  Arena ar(workspace, workspace_bytes);
  __nv_bfloat16* xn = ar.take<__nv_bfloat16>(tokens * d);
  float* maskf = ar.take<float>(tokens);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "triangle_project: workspace too small");
  return triangle_front(w, x, mask, tokens, inner, pitch, d, xn, maskf, Lc, Rc, chan_stride, gate, s);
}

long long af2_triangle_contract_workspace(int rows, int cols, int d) {
  return align_up((long long)d * rows * align_up(cols, 4) * 4, 256) + align_up((long long)rows * cols * d * 2, 256) + 1024;
}

// x [rows, cols, d] (local shard, updated in place) += to_out(LN_c(O) * gate) with
//   outgoing: O[i][j] = sum_k L[i][k] R[j][k]; L = Lc [c][rows][ld_l], piece p of Rg = [c][cols/pieces][ld_r]
//   ingoing : O[i][j] = sum_k R[k][i] L[k][j]; L = Lc [c][K][ld_l],    piece p of Rg = [c][K][ld_r] (i < rows/pieces)
// Either operand may be a window into a larger channel-major tensor (the banded schedule's column window R[c][k][i0 .. i0 + rows)).
int af2_triangle_contract(const af2_trimul_weights* w, float* x, const void* Lc, long long cs_l, long long ld_l, const void* Rg,
                          long long cs_r, long long ld_r, long long piece_stride, int pieces, const void* gate, int rows,
                          int cols, int K, int d, int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream) {
  NvtxRange nvtx_("af2_triangle_contract");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x || !Lc || !Rg || !gate || pieces < 1) return fail(AF2_ERR_BAD_ARG, "triangle_contract: bad argument");
  if (rows <= 0 || cols <= 0 || K <= 0 || d % 32) return fail(AF2_ERR_BAD_ARG, "triangle_contract: rows %d cols %d K %d d %d", rows, cols, K, d);
  if ((!ingoing && cols % pieces) || (ingoing && rows % pieces)) return fail(AF2_ERR_BAD_ARG, "triangle_contract: pieces must divide the gathered axis");
  if (ld_l % 8 || ld_r % 8 || cs_l % 8 || cs_r % 8)
    return fail(AF2_ERR_BAD_ARG, "triangle_contract: pitches and channel strides must be multiples of 8 elements");
  const long long mn_l = ingoing ? cols : K, mn_r = ingoing ? rows / pieces : K;   // elements used along each operand's pitch
  if (ld_l < mn_l || ld_r < mn_r) return fail(AF2_ERR_BAD_ARG, "triangle_contract: pitch shorter than the operand row");
  Arena ar(workspace, workspace_bytes);
  const ContractOut o = take_contract_out(ar, rows, cols, d);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "triangle_contract: workspace too small");
  if (!ingoing)   // O_c = L_c R_c^T, both K-major, R gathered along j
    AF2_TRY(launch_contract(Lc, ld_l, cs_l, Rg, ld_r, cs_r, false, rows, cols, K, d, pieces, false, piece_stride, o.Oc, o.pitch, o.cs, s));
  else            // O_c[i][j] = sum_k R_c[k][i] L_c[k][j], both MN-major, R gathered along i
    AF2_TRY(launch_contract(Rg, ld_r, cs_r, Lc, ld_l, cs_l, true, rows, cols, K, d, pieces, true, piece_stride, o.Oc, o.pitch, o.cs, s));
  return contract_tail(chan_ln_params(o.Oc, o.cs, o.pitch, rows, cols, d, 0, w->on_gamma, w->on_beta, gate, nullptr, 0.f, 1e-5f, o.tn),
                       w->w_out, w->b_out, x, s);
}

// ------------------------------------------------------------------------------------------------
// stage-level outer mean
// ------------------------------------------------------------------------------------------------
long long af2_outer_project_workspace(long long tokens, int d) {
  return align_up(tokens * d * 2, 256) + align_up(tokens * 4, 256) + 1024;
}

// m [S, inner, d] local columns -> LRc bf16 [2d][S*pitch(inner)]: channels [0,d) = left, [d,2d) = right
int af2_outer_project(const af2_outer_weights* w, const float* m, const unsigned char* msa_mask, long long tokens,
                      int inner, int d, void* LRc, long long chan_stride, void* workspace, long long workspace_bytes,
                      af2_stream_t stream) {
  NvtxRange nvtx_("af2_outer_project");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !m || !LRc) return fail(AF2_ERR_BAD_ARG, "outer_project: null argument");
  if (d % 32) return fail(AF2_ERR_BAD_ARG, "outer_project: dim %d must be a multiple of 32", d);
  if (inner <= 0 || tokens % inner || tokens > 0x7fffffffLL)
    return fail(AF2_ERR_BAD_ARG, "outer_project: %lld tokens must be a multiple of inner %d and at most 2^31 - 1", tokens, inner);
  const int pitch = (int)align_up(inner, 8);
  if (chan_stride < tokens / inner * pitch) return fail(AF2_ERR_BAD_ARG, "outer_project: channel stride shorter than the rows written");
  Arena ar(workspace, workspace_bytes);
  __nv_bfloat16* mn = ar.take<__nv_bfloat16>(tokens * d);
  float* maskf = ar.take<float>(tokens);
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "outer_project: workspace too small");
  return outer_front(w, m, msa_mask, tokens, inner, pitch, d, mn, maskf, LRc, chan_stride, s);
}

long long af2_outer_contract_workspace(int rows, int N, int d) {
  return align_up((long long)d * rows * align_up(N, 4) * 4, 256) + align_up((long long)rows * N * d * 2, 256) +
         align_up((long long)rows * N * 4, 256) + align_up((long long)N * 4096 / 8, 256) + 1024;    // + packed mask bits (S <= 4096)
}

// x [rows, N, d] (pair rows row0..row0+rows, updated in place) += proj_out( sum_s L[s][i] R[s][j] * scale[i][j] )
//   L = Lc [c][S][pitch(rows)] (local columns), piece p of Rg = [c][S][pitch(N/pieces)]
int af2_outer_contract(const af2_outer_weights* w, float* x, const void* Lc, long long cs_l, const void* Rg,
                       long long cs_r, long long piece_stride, int pieces, const unsigned char* msa_mask_full,
                       int row0, int rows, int N, int S, int d, float eps, void* workspace, long long workspace_bytes,
                       af2_stream_t stream) {
  NvtxRange nvtx_("af2_outer_contract");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!w || !x || !Lc || !Rg || pieces < 1 || N % pieces) return fail(AF2_ERR_BAD_ARG, "outer_contract: bad argument");
  Arena ar(workspace, workspace_bytes);
  const ContractOut o = take_contract_out(ar, rows, N, d);
  float* scale = ar.take<float>((long long)rows * N);
  uint32_t* mwords = (S <= 4096) ? ar.take<uint32_t>((long long)((S + 31) / 32) * N) : nullptr;
  if (!ar.ok) return fail(AF2_ERR_WORKSPACE, "outer_contract: workspace too small");
  if (msa_mask_full) AF2_TRY(launch_outer_scale(msa_mask_full, scale, mwords, row0, rows, S, N, eps, s));
  // both MN-major, R gathered along j
  AF2_TRY(launch_contract(Lc, align_up(rows, 8), cs_l, Rg, align_up(N / pieces, 8), cs_r, true, rows, N, S, d, pieces, false,
                          piece_stride, o.Oc, o.pitch, o.cs, s));
  return contract_tail(chan_ln_params(o.Oc, o.cs, o.pitch, rows, N, d, 1, nullptr, nullptr, nullptr, msa_mask_full ? scale : nullptr,
                                      1.0f / (float)S, 0.f, o.tn),
                       w->w_out, w->b_out, x, s);
}

// ------------------------------------------------------------------------------------------------
int af2_rotary(const float* x, const float* sin_, const float* cos_, float* y, int b, int h, int n, int dh, int rot,
               int sincos_batch, af2_stream_t stream) {
  NvtxRange nvtx_("af2_rotary");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (dh % 2 || rot % 2 || rot > dh) return fail(AF2_ERR_BAD_ARG, "rotary: dh=%d rot=%d must be even, rot <= dh", dh, rot);
  const long long pairs = (long long)b * h * n * (dh / 2);
  if (pairs == 0) return AF2_OK;
  { ProfScope ps(s, KC_MISC, 0.0, 0.0); rotary_kernel<<<ew_grid(pairs), 256, 0, s>>>(x, sin_, cos_, y, b, h, n, dh, rot, sincos_batch); }
  CUDA_OK(cudaGetLastError());
  return AF2_OK;
}

int af2_layernorm_bf16(const float* x, const float* gamma, const float* beta, void* y_bf16, long long T, int d,
                       float eps, af2_stream_t stream) {
  LnParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.x = x; lp.gamma = gamma; lp.beta = beta; lp.y = static_cast<__nv_bfloat16*>(y_bf16); lp.T = T; lp.d = d; lp.eps = eps;
  return launch_layernorm(lp, static_cast<cudaStream_t>(stream));
}

int af2_gemm_bf16_epilogue(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb, long long b_batch,
                           int M, int N, int K, int batch, int mn_major, const af2_gemm_epilogue* epi, af2_stream_t stream) {
  if (!A || !Bm || !epi || !epi->out) return fail(AF2_ERR_BAD_ARG, "gemm: null argument");
  if (epi->bn != 64 && epi->bn != 128 && epi->bn != 256) return fail(AF2_ERR_BAD_ARG, "gemm: bn %d (64, 128 or 256)", epi->bn);
  if (epi->mode < EPI_STORE_BF16 || epi->mode > EPI_STORE_F32 || epi->act < ACT_NONE || epi->act > ACT_GELU ||
      epi->layout < LAYOUT_TOKEN || epi->layout > LAYOUT_CHANNEL)
    return fail(AF2_ERR_BAD_ARG, "gemm: epilogue mode %d / act %d / layout %d", epi->mode, epi->act, epi->layout);
  const bool f32 = epi->mode == EPI_RESID_F32 || epi->mode == EPI_STORE_F32;
  if (f32 && (epi->layout != LAYOUT_TOKEN || epi->use_rowscale))
    return fail(AF2_ERR_BAD_ARG, "gemm: fp32 epilogues store token-major without a row scale");
  if (epi->use_rowscale && !epi->rowscale) return fail(AF2_ERR_BAD_ARG, "gemm: use_rowscale without rowscale");
  if (epi->mode == EPI_RESID_F32 && !epi->resid) return fail(AF2_ERR_BAD_ARG, "gemm: residual epilogue without resid");
  if (epi->mode == EPI_GATED_BF16 && N % epi->bn) return fail(AF2_ERR_BAD_ARG, "gemm: gated N %d not a multiple of bn %d", N, epi->bn);
  GemmCall c;
  memset(&c, 0, sizeof(c));
  c.A = A; c.lda = lda; c.a_batch = a_batch; c.Bm = Bm; c.ldb = ldb; c.b_batch = b_batch;
  c.M = M; c.N = N; c.K = K; c.batch = batch; c.mn_major = mn_major != 0; c.bn = epi->bn;
  c.mode = epi->mode; c.act = epi->act; c.layout = epi->layout; c.use_rowscale = epi->use_rowscale;
  c.bias = epi->bias; c.rowscale = epi->rowscale; c.resid = epi->resid; c.ld_resid = epi->ld_resid;
  c.out = epi->out; c.ld_out = epi->ld_out; c.out_batch = epi->out_batch;
  c.cm_inner = epi->cm_inner; c.cm_pitch = epi->cm_pitch; c.out_cols = epi->out_cols;
  return launch_gemm(c, static_cast<cudaStream_t>(stream));
}

int af2_gemm_bf16_f32(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb, long long b_batch,
                      float* C, long long ldc, long long c_batch, int M, int N, int K, int batch, int mn_major,
                      af2_stream_t stream) {
  af2_gemm_epilogue e;
  memset(&e, 0, sizeof(e));
  e.bn = pick_bn(N); e.mode = EPI_STORE_F32; e.layout = LAYOUT_TOKEN; e.out = C; e.ld_out = ldc; e.out_batch = c_batch;
  return af2_gemm_bf16_epilogue(A, lda, a_batch, Bm, ldb, b_batch, M, N, K, batch, mn_major, &e, stream);
}

int af2_attention_bf16(const void* qkv, const void* gate, const void* bias, const unsigned char* mask, void* out, int n,
                       int nbatch, int heads, int dim_head, long long tok_sb, long long tok_si, af2_stream_t stream) {
  if (!qkv || !gate || !out) return fail(AF2_ERR_BAD_ARG, "attention: null argument");
  if (n <= 0 || nbatch <= 0 || heads <= 0) return AF2_OK;
  return launch_attention(static_cast<const __nv_bfloat16*>(qkv), heads, dim_head, n, nbatch, tok_sb, tok_si,
                          static_cast<const __nv_bfloat16*>(bias), (int)align_up(n, 8), mask,
                          static_cast<const __nv_bfloat16*>(gate), static_cast<__nv_bfloat16*>(out),
                          static_cast<cudaStream_t>(stream));
}

int af2_attention_proj_max_n(int dim_head) { return attn_proj_max_n(dim_head); }

int af2_attention_proj_bf16(const void* xn, int d, const void* w_qkv, const void* w_gate, const float* b_gate, const void* bias,
                            const unsigned char* mask, void* out, int n, int nbatch, int heads, int dim_head, long long tok_sb,
                            long long tok_si, af2_stream_t stream) {
  if (!xn || !w_qkv || !w_gate || !out) return fail(AF2_ERR_BAD_ARG, "attention_proj: null argument");
  if (d < 8 || d % 8) return fail(AF2_ERR_BAD_ARG, "attention_proj: dim %d must be a positive multiple of 8", d);
  if (n <= 0 || nbatch <= 0 || heads <= 0) return AF2_OK;
  if (!attn_proj_ok(dim_head, n, xn, w_qkv, w_gate))
    return fail(AF2_ERR_BAD_ARG, "attention_proj: dim_head %d, n %d (at most %d) or a misaligned operand", dim_head, n,
                attn_proj_max_n(dim_head));
  return launch_attention_proj(static_cast<const __nv_bfloat16*>(xn), d, static_cast<const __nv_bfloat16*>(w_qkv),
                               static_cast<const __nv_bfloat16*>(w_gate), b_gate, heads, dim_head, n, nbatch, tok_sb, tok_si,
                               static_cast<const __nv_bfloat16*>(bias), (int)align_up(n, 8), mask, static_cast<__nv_bfloat16*>(out),
                               static_cast<cudaStream_t>(stream));
}

int af2_gemm_bf16_f32_gathered(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb, long long b_batch,
                               float* C, long long ldc, long long c_batch, int M, int N, int K, int batch, int mn_major, int bn,
                               int a_pr, long long a_piece, int b_pr, long long b_piece, af2_stream_t stream) {
  if (!A || !Bm || !C) return fail(AF2_ERR_BAD_ARG, "gemm: null argument");
  if (bn != 64 && bn != 128 && bn != 256) return fail(AF2_ERR_BAD_ARG, "gemm: bn %d (64, 128 or 256)", bn);
  if (a_pr < 0 || b_pr < 0) return fail(AF2_ERR_BAD_ARG, "gemm: negative piece size");
  GemmCall c;
  memset(&c, 0, sizeof(c));
  c.A = A; c.lda = lda; c.a_batch = a_batch; c.Bm = Bm; c.ldb = ldb; c.b_batch = b_batch;
  c.M = M; c.N = N; c.K = K; c.batch = batch; c.mn_major = mn_major != 0; c.bn = bn;
  c.mode = EPI_STORE_F32; c.layout = LAYOUT_TOKEN; c.out = C; c.ld_out = ldc; c.out_batch = c_batch;
  c.a_pr = a_pr; c.a_piece = a_piece; c.b_pr = b_pr; c.b_piece = b_piece;
  return launch_gemm(c, static_cast<cudaStream_t>(stream));
}

static int chan_ln_check(const ChanLnParams& p) {
  if (!p.src || !p.y || (p.mode == 0 && (!p.gamma || !p.beta || !p.gate))) return fail(AF2_ERR_BAD_ARG, "chan_to_token: null argument");
  if (p.mode != 0 && p.mode != 1) return fail(AF2_ERR_BAD_ARG, "chan_to_token: mode %d (0 or 1)", p.mode);
  if (p.rows < 0 || p.n < 0 || p.d <= 0 || p.pitch < p.n || p.chan_stride < (long long)p.rows * p.pitch)
    return fail(AF2_ERR_BAD_ARG, "chan_to_token: rows=%d n=%d pitch=%d d=%d chan_stride=%lld", p.rows, p.n, p.pitch, p.d, p.chan_stride);
  return AF2_OK;
}

int af2_chan_to_token_select(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode,
                             const float* gamma, const float* beta, const void* gate, const float* scale, float scale_const,
                             float eps, void* y) {
  const ChanLnParams p = chan_ln_params(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y);
  AF2_TRY(chan_ln_check(p));
  const int v = c2t_select(p);
  return v ? v : fail(AF2_ERR_BAD_ARG, "chan_to_token: no kernel takes d=%d rows=%d", d, rows);
}

int af2_chan_to_token(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode, const float* gamma,
                      const float* beta, const void* gate, const float* scale, float scale_const, float eps, void* y, int variant,
                      int* ran, af2_stream_t stream) {
  if (ran) *ran = 0;
  const ChanLnParams p = chan_ln_params(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y);
  AF2_TRY(chan_ln_check(p));
  if (variant < C2T_AUTO || variant > C2T_TMA) return fail(AF2_ERR_BAD_ARG, "chan_to_token: variant %d (0..3)", variant);
  return launch_chan_to_token(p, static_cast<cudaStream_t>(stream), variant, ran);
}

int af2_outer_scale(const unsigned char* mask, float* scale, void* words, int row0, int rows, int S, int N, float eps, int variant,
                    int* ran, af2_stream_t stream) {
  if (ran) *ran = 0;
  if (!mask || !scale) return fail(AF2_ERR_BAD_ARG, "outer_scale: null argument");
  if (S < 1 || N < 1 || row0 < 0 || rows < 0 || row0 + rows > N)
    return fail(AF2_ERR_BAD_ARG, "outer_scale: S=%d N=%d rows [%d, %d)", S, N, row0, row0 + rows);
  if (variant < 0 || variant > 2) return fail(AF2_ERR_BAD_ARG, "outer_scale: variant %d (0..2)", variant);
  return launch_outer_scale(mask, scale, static_cast<uint32_t*>(words), row0, rows, S, N, eps, static_cast<cudaStream_t>(stream),
                            variant, ran);
}

// The tail of the triangle / outer-product contractions on its own (see include/af2b200.h)
int af2_contract_tail(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode, const float* gamma,
                      const float* beta, const void* gate, const float* scale, float scale_const, float eps, const void* xn,
                      const void* w_ogate, const float* b_ogate, const void* w_out, const float* b_out, float* x, void* y,
                      int variant, int* ran, af2_stream_t stream) {
  if (ran) *ran = 0;
  const ChanLnParams p = chan_ln_params(src, chan_stride, pitch, rows, n, d, mode, gamma, beta, gate, scale, scale_const, eps, y);
  AF2_TRY(chan_ln_check(p));
  if (!w_out || !x) return fail(AF2_ERR_BAD_ARG, "contract_tail: null argument");
  if ((xn != nullptr) != (w_ogate != nullptr)) return fail(AF2_ERR_BAD_ARG, "contract_tail: xn and w_ogate go together");
  if (d % 8) return fail(AF2_ERR_BAD_ARG, "contract_tail: dim %d must be a multiple of 8", d);
  if ((long long)rows * n > 0x7fffffffLL) return fail(AF2_ERR_BAD_ARG, "contract_tail: too many tokens");
  if (variant < CTAIL_AUTO || variant > CTAIL_FUSED) return fail(AF2_ERR_BAD_ARG, "contract_tail: variant %d (0..2)", variant);
  const TailGateProj gp = {xn, w_ogate, b_ogate};
  return contract_tail(p, w_out, b_out, x, static_cast<cudaStream_t>(stream), xn ? &gp : nullptr, variant, ran);
}

}  // extern "C"

#include "strict_api.inl"
#include "peer_api.inl"
#include "template_api.inl"
#include "attention_api.inl"
#include "heads_api.inl"
#include "structure_api.inl"
#include "geometry_api.inl"
#include "metrics_api.inl"
#include "distogram_loss_api.inl"
#include "angle_loss_api.inl"
