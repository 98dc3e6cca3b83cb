// libgitb200.so -- C ABI + host-side engine of the H100-native (sm_90a) GIT captioning hot path.
// See include/gitb200.h for the contract of every entry point and the reference function it replaces.
//
// Device data layout (all engine-owned, HBM resident):
//   weights      : GEMM operands bf16 [out, in] (the nn.Linear layout is already K-major), biases /
//                  LayerNorm / embeddings fp32; decoder q,k,v fused to one [2304, 768] matrix; patch kernel
//                  flattened to [d, 3*p*p] zero-padded to a multiple of 64 columns.
//   encoder      : residual stream x fp32 [NI*L, d]; GEMM A operands (LN output, attention context, MLP
//                  hidden) bf16 row-major; packed qkv bf16 [NI*L, 3d].
//   image K/V    : bf16 [layer][k|v][B][M][768]  (token-major rows: a decode-step reader streams contiguous
//                  1536-byte rows; written once by the prefill QKV GEMM epilogue, shared by all beams).
//                  Ragged batches (gitb200_set_image_sizes): M = L_max, image b's first L_b rows are valid and its
//                  padding rows hold finite values that no valid row reads.
//   text K/V     : bf16 [layer][k|v][rows][T_alloc][768] + int32 src_row[rows][T_alloc] indirection for beams.
//   decode step  : fp32 row state [rows, 768], bf16 copy for the GEMMs, fp32 qkv / logits.
//   scoring      : the text rows of N captions x T positions as [N * T, 768] row blocks (one layer's text K/V at a time);
//                  no logits: LM-head statistics [N * T][2 * column tiles] float4 (gemm.cuh EPI_LSE).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <set>
#include <string>
#include <utility>
#include <vector>

#include "../../include/gitb200.h"
#include "attention.cuh"
#include "constrained.cuh"
#include "decode_mega.cuh"
#include "gemm.cuh"
#include "preproc.cuh"
#include "ptx.cuh"
#include "rowops.cuh"
#include "search.cuh"

using namespace gitb200;
typedef __nv_bfloat16 bf16;

#define GITB200_ABI_VERSION 12

// ------------------------------------------------------------------------------------------------
// errors
// ------------------------------------------------------------------------------------------------
static thread_local std::string g_create_error;

struct DevBuf {
  static inline std::atomic<unsigned long long> moves{0};   // bumped whenever a buffer's address changes (step_graph)
  void* p = nullptr;
  size_t cap = 0;
  bool owned = true;   // false: borrowed from another engine (gitb200_share_weights)
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (!owned) return cudaErrorInvalidValue;   // a borrowed buffer is never re-allocated
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    ++moves;
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  void release() {
    if (p) ++moves;
    if (p && owned) cudaFree(p);
    p = nullptr;
    cap = 0;
    owned = true;
  }
  void borrow(const DevBuf& o) {
    release();
    ++moves;
    p = o.p;
    cap = o.cap;
    owned = false;
  }
  template <typename T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

struct EncLayer {
  DevBuf wqkv, bqkv, wo, bo, ln1g, ln1b, ln2g, ln2b, w1, b1, w2, b2;
};
struct DecLayer {
  DevBuf wqkv, bqkv, wo, bo, lnag, lnab, w1, b1, w2, b2, lnog, lnob;
  DevBuf m_wqkv, m_wo, m_w1, m_w2;   // fragment-packed 8-feature tiles for decode_mega_kernel (built by finalize_weights)
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

struct TmapKey {
  const void* ptr;
  long long rows, cols, ld;
  int box_rows;   // negative: un-swizzled box (decode attention K/V slices)
  bool operator<(const TmapKey& o) const {
    if (ptr != o.ptr) return ptr < o.ptr;
    if (rows != o.rows) return rows < o.rows;
    if (cols != o.cols) return cols < o.cols;
    if (ld != o.ld) return ld < o.ld;
    return box_rows < o.box_rows;
  }
};

// The images of one call as the encoder reads them (image_batch), built at the call's entry from its batch and frames and
// either the sizes set for it (gitb200_set_image_sizes) or the sticky input size (gitb200_set_input_size).
struct ImageBatch {
  std::vector<RaggedImg> imgs;   // every encoded image, NI = B * frames of them in the encoder's order f * B + b
  int B = 0, frames = 1;         // frames after the temporal-embedding truncation of list inputs
  int L_max = 0;                 // slot length: tokens of the largest image
  std::vector<int> lens;         // a ragged batch: L of each image (rg_lens), else empty
  int pos_rows = 0;              // rows of the call's positional table in pos_interp (0: the stored table serves)
  size_t bytes = 0;              // pixel bytes the call passes (every frame, before the truncation)
  bool list_input = false;       // frames >= 1 were passed: temporal embeddings apply
  bool ragged = false;           // the sizes were given per image
};

// Geometry of decode_attn_kernel (dec_attn_geometry).
struct DecAttnGeom {
  int chunk_rows, box_rows;   // DecAttnParams::chunk_rows / box_rows
  size_t smem;                // dynamic shared memory per CTA
  int grid;                   // CTAs the engine launches
};

struct gitb200_engine {
  gitb200_config cfg;
  int device = 0;
  int num_sms = 132;
  std::string err;
  int64_t launches = 0;
  bool use_graph = true;
  bool use_pdl = true;
  // fp32-grade parity mode: every GEMM operand is a (hi, lo) bf16 pair and each GEMM computes a_hi w_hi + a_lo w_hi +
  // a_hi w_lo in ONE pass of the same wgmma kernel (activations stored [hi | lo | hi], weights [hi | hi | lo] along K);
  // attention, K/V caches and q/k/v stay fp32; exact QuickGELU.  ~3x the GEMM work: a verification mode (the north star's
  // "logits within 1e-3" against the fp32 reference), not a serving mode.  Weights must be (re-)uploaded after switching.
  bool use_mega = true;   // greedy decode steps of <= 64 sequences through the persistent decode_mega_kernel
  bool mega_ready = false;
  int debug_layers = -1;  // debugging: run only the first n decoder layers in the decode step (both step paths); -1 = all
  bool parity = false;
  int ks() const { return parity ? 3 : 1; }                  // K multiplier of every GEMM operand
  size_t kvb() const { return parity ? 4 : 2; }              // bytes per K/V cache element
  const gitb200_engine* weights_from = nullptr;   // non-null: weight buffers are borrowed from that engine

  // derived geometry
  int g = 0, L = 0, Kpatch = 0, Kp = 0, d = 0, D = 0, F = 0, V = 0;
  // input size of the next encodes (gitb200_set_input_size; default image_size x image_size); differs from the model's
  // for MinMaxResizeForTest inputs (reference inference.py:29-64)
  int in_h = 0, in_w = 0;
  // the images of the last encode (cur_img.ragged: their sizes were given per image) and, on the device, its RaggedImg
  // table and, for a ragged batch, each image's valid key count L_b; what the last upload wrote to each, so that a call
  // with the same images copies nothing
  ImageBatch cur_img;
  DevBuf rg_tab, rg_lens;
  std::string rg_tab_up, rg_lens_up;

  // weights
  DevBuf w_patch, cls, pos_emb, lnpre_g, lnpre_b, lnpost_g, lnpost_b;
  std::vector<EncLayer> enc;
  DevBuf w_vp, b_vp, lnvp_g, lnvp_b, words_f32, words_bf16, positions, lnemb_g, lnemb_b, out_bias, temb;
  DevBuf m_lm;                                              // packed LM-head tiles (decode_mega_kernel)
  std::vector<DecLayer> dec;
  std::set<std::string> seen;
  bool finalized = false;

  // workspaces
  DevBuf x, h, qkv, ctx, u, feats, feats_f32, pos_interp;   // encoder
  DevBuf pt, pxd, phd, pq, pctx, pu;                        // decoder-layer pass (image rows, caption rows)
  DevBuf img_kv, txt_kv, src_row[2];                        // caches
  size_t txt_kv_eb = 0;                                     // element size (kvb()) the text cache was last zeroed for
  DevBuf xd_t, hd_t, qkv_t, ctx_t, t_t, u_t, logits;        // decode step
  DevBuf y_t, qb_t, mega_bar;                               // decode_mega_kernel: pre-LN sums, bf16 q, grid-barrier counters
  DevBuf state, next_token, logprob_sum, tokens_i64, stage_img, stage_tok, stage_lp, prefix_dev;
  DevBuf beam_ws;                                           // beam-search bookkeeping (search.cuh)
  BeamState beam_s{};                                       // ... as the last beam generate carved it (gitb200_debug_read)
  int beam_B = 0, beam_max_steps = 0;                       // 0: the last prefill was not a beam generate
  int beam_cand = 0;                                        // row stride of beam_s's candidate arrays (beam_cand_capacity)
  DevBuf sc_kv, sc_tgt, sc_part, sc_loss, sc_valid, sc_index;   // caption scoring: one layer's text K/V, LM-head targets /
                                                               // statistics, per-row losses, op image_index
  DevBuf sel_ws;                                            // greedy selection partials
  DevBuf chain;                                             // decode-step kernel chain completion counters [64]
  DecAttnGeom attn_geom{};                                  // decode_attn_kernel geometry of the last prefill
  int cur_B = 0, cur_frames = 0, cur_M = 0, cur_beam = 1, T_alloc = 0, cur_rows = 0, cur_src = 0;
  int cur_seqs = 1;                                         // sequences per image of the last prefill (rows = B * seqs * beam)

  EncodeTiledFn encode_tiled = nullptr;
  std::map<TmapKey, CUtensorMap> tmaps;

  // decode-step graph cache
  // (keyed by everything the captured launches bake in, see step_graph; several shapes alternate when batches are
  //  coalesced into launches of different sizes, so a handful of instantiated graphs are kept)
  struct StepGraph { cudaGraphExec_t exec = nullptr; int64_t launches = 0; unsigned long long last_use = 0; };
  std::map<std::string, StepGraph> step_graphs;
  unsigned long long step_graph_clock = 0;
  int last_gemm_grid = 0;
  cudaStream_t own_stream = nullptr;
  cudaEvent_t own_event = nullptr;
  // asynchronous generate: enqueue now, read the loop state back in gitb200_generate_finish
  StepState* host_state = nullptr;   // pinned
  bool pending = false;
  int pend_max_steps = 0;
  int pend_rows = 0;                               // rows of the call in flight (beam: B * beam)
  bool pend_beam = false;
  cudaStream_t pend_stream = nullptr;
  cudaEvent_t chunk_ev[2] = {nullptr, nullptr};   // decode-loop chunks (generate_impl)
  cudaEvent_t dec_ev[2] = {nullptr, nullptr};     // around the decode loop of the last generate (gitb200_last_decode_ms)
  int dec_steps = 0;                               // step launches between them
  bool dec_mega = false;                           // ... each of which was one decode_mega_kernel launch
  // vocabulary trie (gitb200_set_trie; sticky)
  DevBuf trie_begin, trie_token, trie_child, trie_cursor;
  int trie_nodes = 0;
  // inputs of the next call only, taken by it at entry (take_next_call)
  struct NextCall {
    std::vector<int> image_hw;           // (height, width) of every image (gitb200_set_image_sizes)
    const long long* prefix_tok = nullptr;  // per-row prefixes (gitb200_set_row_prefixes)
    const int32_t* prefix_lens = nullptr;
    int prefix_rows = 0, prefix_stride = 0;
    const float* uniforms = nullptr;      // sampling (gitb200_set_sampling)
    int sample_steps = 0, sample_rows = 0;
    float temperature = 1.0f;
    const float* beam_uniforms = nullptr; // sampled beam search (gitb200_set_beam_sampling)
    int beam_sample_steps = 0, beam_sample_rows = 0;
    float beam_temperature = 1.0f, beam_top_p = 1.0f;
    int beam_top_k = 0;
    int seqs_per_image = 1;               // gitb200_set_sequences_per_image
  } next;
};

// The inputs set for the next call that the calling one takes (include/gitb200.h, gitb200_set_image_sizes).
static gitb200_engine::NextCall take_next_call(gitb200_engine* h, bool generate) {
  gitb200_engine::NextCall c;
  if (generate) std::swap(c, h->next);
  else c.image_hw.swap(h->next.image_hw);
  return c;
}

static void drop_step_graphs(gitb200_engine* h) {
  for (auto& kv : h->step_graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
  h->step_graphs.clear();
}

static int fail(gitb200_engine* h, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  if (h) h->err = buf; else g_create_error = buf;
  return 1;
}

#define CK(call)                                                                                     \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess) return fail(h, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
  } while (0)
#define CKL(h_, what)                                                                                \
  do {                                                                                               \
    cudaError_t e_ = cudaGetLastError();                                                             \
    if (e_ != cudaSuccess) return fail(h_, "launch %s failed: %s", what, cudaGetErrorString(e_));    \
    (h_)->launches++;                                                                                \
  } while (0)
#define TRY(expr)                 \
  do {                            \
    int rc_ = (expr);             \
    if (rc_ != 0) return rc_;     \
  } while (0)

// Kernel launch with optional programmatic dependent launch (the decode step chains ~45 small kernels; PDL lets
// each one's prologue / weight prefetch overlap its predecessor's tail, also inside a captured CUDA graph).
template <typename... KArgs, typename... Args>
static cudaError_t launch_k(bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                            Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}

// ------------------------------------------------------------------------------------------------
// TMA descriptors
// ------------------------------------------------------------------------------------------------
static int load_encode_fn(gitb200_engine* h) {
  if (h->encode_tiled) return 0;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr)
    return fail(h, "cuTensorMapEncodeTiled not available from the driver: %s", cudaGetErrorString(e));
  h->encode_tiled = reinterpret_cast<EncodeTiledFn>(fn);
  return 0;
}

// bf16 matrix [rows, cols] with leading dimension ld (elements); box = [box_rows x 64], 128B-swizzled (GEMM
// operands) or plain row-major (swizzle == false: decode-attention K/V slices).
static int get_tmap(gitb200_engine* h, const void* ptr, long long rows, long long cols, long long ld, int box_rows,
                    CUtensorMap* out, bool swizzle = true) {
  TmapKey key{ptr, rows, cols, ld, swizzle ? box_rows : -box_rows};
  auto it = h->tmaps.find(key);
  if (it != h->tmaps.end()) {
    *out = it->second;
    return 0;
  }
  TRY(load_encode_fn(h));
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0)
    return fail(h, "TMA operand must be 16-byte aligned with a 16-byte multiple row pitch (ptr=%p ld=%lld)", ptr, ld);
  CUtensorMap m;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = h->encode_tiled(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(h, "cuTensorMapEncodeTiled failed with CUresult %d (rows=%lld cols=%lld ld=%lld box=%d)",
                                     static_cast<int>(r), rows, cols, ld, box_rows);
  if (h->tmaps.size() > 4096) h->tmaps.clear();
  h->tmaps[key] = m;
  *out = m;
  return 0;
}

// Raises `kernel`'s dynamic shared-memory limit to smem bytes on the engine's device; the attribute is set once per kernel,
// device and larger size (the parity and decode attention kernels size their shared memory per call).
static int set_dyn_smem(gitb200_engine* h, const void* kernel, size_t smem) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> done;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = done[{kernel, h->device}];
  if (have < smem) {
    CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    have = smem;
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// GEMM launcher
// ------------------------------------------------------------------------------------------------
struct GemmCall {
  const bf16* A = nullptr;  // [M, K] (kernel operand A: 128-row tiles)
  long long lda = 0;
  const bf16* B = nullptr;  // [N, K] (kernel operand B: BN-row tiles)
  long long ldb = 0;
  GemmParams p{};
  int bn = 0;               // 0 = heuristic
};

template <int BN, int EPI>
static int launch_gemm_inst(gitb200_engine* h, const GemmCall& c, cudaStream_t st) {
  using C = GemmCfg<BN>;
  TRY(set_dyn_smem(h, reinterpret_cast<const void*>(gemm_bf16_wgmma<BN, EPI>), C::SMEM_BYTES));
  CUtensorMap ta, tb;
  TRY(get_tmap(h, c.A, c.p.M, c.p.K, c.lda, 128, &ta));
  TRY(get_tmap(h, c.B, c.p.N, c.p.K, c.ldb, BN, &tb));
  const int m_tiles = (c.p.M + 127) / 128;
  const int n_tiles = (c.p.N + BN - 1) / BN;
  const int tiles = m_tiles * n_tiles * c.p.k_splits;
  const int grid = tiles < h->num_sms ? tiles : h->num_sms;
  h->last_gemm_grid = grid;
  CK(launch_k(c.p.pdl != 0, gemm_bf16_wgmma<BN, EPI>, dim3(grid), dim3(C::THREADS), C::SMEM_BYTES, st, ta, tb, c.p));
  CKL(h, "gemm_bf16_wgmma");
  return 0;
}

template <int BN>
static int launch_gemm_bn(gitb200_engine* h, const GemmCall& c, cudaStream_t st) {
  const GemmParams& p = c.p;
  if constexpr (BN == 256) {   // caption scoring's LM head: statistics only (see EPI_LSE)
    if (p.lse_target != nullptr) return launch_gemm_inst<BN, EPI_LSE>(h, c, st);
  }
  if (p.lse_target != nullptr) return fail(h, "gemm: the LM-head statistics epilogue runs with 256-column tiles only");
  const int code = epi_code(p.transposed != 0, p.out_bf16 != 0, p.resid != nullptr, p.partial != 0, p.act) | (p.split3 ? EPI_SPLIT3 : 0);
  if constexpr (BN == 256) {   // parity mode: bf16 outputs that feed another GEMM leave as [hi | lo | hi]
    switch (code) {
      case epi_code(false, true, false, false, ACT_QUICKGELU_EXACT) | EPI_SPLIT3: return launch_gemm_inst<BN, epi_code(false, true, false, false, ACT_QUICKGELU_EXACT) | EPI_SPLIT3>(h, c, st);
      case epi_code(false, true, false, false, ACT_GELU_ERF) | EPI_SPLIT3: return launch_gemm_inst<BN, epi_code(false, true, false, false, ACT_GELU_ERF) | EPI_SPLIT3>(h, c, st);
      default: break;
    }
  }
  if constexpr (BN == 64 || BN == 128 || BN == 256) {
    if (code == (epi_code(true, true, false, false, ACT_GELU_ERF) | EPI_SPLIT3))
      return launch_gemm_inst<BN, epi_code(true, true, false, false, ACT_GELU_ERF) | EPI_SPLIT3>(h, c, st);
  }
  if constexpr (BN == 192 || BN == 256 || BN == 128) {
    switch (code) {
      case epi_code(false, true, false, false, ACT_NONE): return launch_gemm_inst<BN, epi_code(false, true, false, false, ACT_NONE)>(h, c, st);
      case epi_code(false, false, true, false, ACT_NONE): return launch_gemm_inst<BN, epi_code(false, false, true, false, ACT_NONE)>(h, c, st);
      case epi_code(false, false, false, false, ACT_NONE): return launch_gemm_inst<BN, epi_code(false, false, false, false, ACT_NONE)>(h, c, st);
      case epi_code(false, true, false, false, ACT_QUICKGELU): return launch_gemm_inst<BN, epi_code(false, true, false, false, ACT_QUICKGELU)>(h, c, st);
      case epi_code(false, true, false, false, ACT_GELU_ERF): return launch_gemm_inst<BN, epi_code(false, true, false, false, ACT_GELU_ERF)>(h, c, st);
      default: break;
    }
  }
  if constexpr (BN == 64 || BN == 128 || BN == 256) {
    switch (code) {
      case epi_code(true, false, false, true, ACT_NONE): return launch_gemm_inst<BN, epi_code(true, false, false, true, ACT_NONE)>(h, c, st);
      case epi_code(true, false, false, false, ACT_NONE): return launch_gemm_inst<BN, epi_code(true, false, false, false, ACT_NONE)>(h, c, st);
      case epi_code(true, true, false, false, ACT_GELU_ERF): return launch_gemm_inst<BN, epi_code(true, true, false, false, ACT_GELU_ERF)>(h, c, st);
      default: break;
    }
  }
  return fail(h, "gemm: epilogue combination not instantiated (transposed=%d bf16=%d resid=%d partial=%d act=%d bn=%d)",
              p.transposed, p.out_bf16, p.resid != nullptr, p.partial, p.act, BN);
}

static int pick_bn(const gitb200_engine* h, int M, int N, bool transposed) {
  if (transposed) return N <= 64 ? 64 : (N <= 128 ? 128 : 256);
  // Wide outputs (N = 2304 / 3072) take 128x256 tiles (fewest operand bytes per FLOP through L2 / shared memory); N = 768
  // takes 128x192 tiles (4 column tiles: less wave quantisation than 3 x 256 at 99 row tiles over 132 SMs).
  (void)h; (void)M;
  if (N % 256 == 0 && N >= 1024) return 256;
  if (N % 192 == 0) return 192;
  if (N % 256 == 0) return 256;
  if (N % 128 == 0) return 128;
  return N > 192 ? 256 : (N > 128 ? 192 : 128);
}

// Splits launch_gemm runs for `requested` over K: every split takes ceil(k-blocks / requested) 64-wide k-blocks, and the
// splits that would be left without one are dropped (8 requested over 12 k-blocks -> 6).
static int effective_k_splits(int K, int requested) {
  const int kb_total = (K + 63) / 64;
  const int splits = std::max(1, std::min(requested, kb_total));
  const int kb_per = (kb_total + splits - 1) / splits;
  return (kb_total + kb_per - 1) / kb_per;
}

static int launch_gemm(gitb200_engine* h, GemmCall c, cudaStream_t st) {
  GemmParams& p = c.p;
  p.k_splits = effective_k_splits(p.K, p.k_splits);
  if (p.seg_n <= 0) p.seg_n = p.N;
  if (p.rows_per_batch <= 0) {
    p.rows_per_batch = p.M;
    p.batch_stride = p.M;
  }
  if (!p.transposed && p.lse_target == nullptr && (p.N % 32 != 0 || p.seg_n % 32 != 0))
    return fail(h, "gemm: N and segment width must be multiples of 32 (N=%d seg=%d)", p.N, p.seg_n);
  if (p.partial && !p.transposed) return fail(h, "gemm: split-K partial buffers are only implemented for the transposed epilogue");
  if (p.k_splits > 1 && !p.partial) return fail(h, "gemm: k_splits > 1 needs the partial-sum epilogue");
  if (p.partial && p.split_stride < static_cast<long long>(p.N) * p.ldo) return fail(h, "gemm: split_stride smaller than one partial buffer");
  int bn = c.bn > 0 ? c.bn : pick_bn(h, p.M, p.N, p.transposed != 0);
  if ((p.split3 || p.lse_target != nullptr) && !p.transposed) bn = 256;
  switch (bn) {
    case 64: return launch_gemm_bn<64>(h, c, st);
    case 128: return launch_gemm_bn<128>(h, c, st);
    case 192: return launch_gemm_bn<192>(h, c, st);
    case 256: return launch_gemm_bn<256>(h, c, st);
    default: return fail(h, "gemm: unsupported tile width %d", bn);
  }
}

// Plain C = A W^T (+bias)(+act)(+resid) -> out (fp32 or bf16), identity row map.
static GemmCall gemm_plain(const bf16* A, long long lda, const bf16* W, long long ldw, int M, int N, int K,
                           const float* bias, int act, const float* resid, void* out, bool out_bf16) {
  GemmCall c;
  c.A = A; c.lda = lda; c.B = W; c.ldb = ldw;
  c.p.M = M; c.p.N = N; c.p.K = K; c.p.k_splits = 1;
  c.p.bias = bias; c.p.act = act; c.p.resid = resid; c.p.ld_resid = N;
  c.p.out[0] = out; c.p.ldo = N; c.p.out_bf16 = out_bf16 ? 1 : 0;
  c.p.seg_n = N;
  return c;
}
// Output of a row-pass GEMM (encoder, decoder-layer pass, LM heads) in the engine's precision mode:
//   F32      fp32 [M, N] (+ resid, which may alias out);
//   OPERAND  the A operand of the next GEMM: bf16 [M, N], or [hi | lo | hi] rows of 3 N columns in parity mode;
//   QKV      attention inputs: bf16, or fp32 in parity mode.
enum class RowOut { F32, OPERAND, QKV };
// gemm_plain over the logical reduction length K: parity mode stores every operand at 3 K (activations [hi | lo | hi],
// weights [hi | hi | lo]) and computes QuickGELU exactly.
static GemmCall gemm_rows(const gitb200_engine* h, RowOut kind, const bf16* A, const bf16* W, int M, int N, int K,
                          const float* bias, int act, const float* resid, void* out) {
  const int ks = h->ks();
  const bool bf16_out = kind == RowOut::OPERAND || (kind == RowOut::QKV && !h->parity);
  GemmCall c = gemm_plain(A, static_cast<long long>(K) * ks, W, static_cast<long long>(K) * ks, M, N, K * ks, bias,
                          (h->parity && act == ACT_QUICKGELU) ? ACT_QUICKGELU_EXACT : act, resid, out, bf16_out);
  if (kind == RowOut::OPERAND && h->parity) {
    c.p.split3 = 1;
    c.p.ldo = 3LL * N;
  }
  return c;
}
// Skinny decode-step GEMM: out[r][f] = sum_k X[r][k] W[f][k] (+bias[f]) (+act) -- swap-AB, transposed epilogue.
// k_splits > 1: split s writes its partial sums to out + s * rows * ldo (fp32); the consumer adds them in split order.
static GemmCall gemm_skinny(const bf16* X, long long ldx, const bf16* W, long long ldw, int rows, int feats, int K,
                            const float* bias, int act, void* out, long long ldo, bool out_bf16, int k_splits,
                            const int* skip, bool pdl = false) {
  GemmCall c;
  c.A = W; c.lda = ldw; c.B = X; c.ldb = ldx;
  c.p.M = feats; c.p.N = rows; c.p.K = K; c.p.k_splits = k_splits;
  c.p.transposed = 1; c.p.partial = k_splits > 1 ? 1 : 0;
  c.p.split_stride = static_cast<long long>(rows) * ldo;
  c.p.bias = bias; c.p.act = act;
  c.p.out[0] = out; c.p.ldo = ldo; c.p.out_bf16 = out_bf16 ? 1 : 0;
  c.p.skip = skip;
  c.p.pdl = pdl ? 1 : 0;
  return c;
}

// ------------------------------------------------------------------------------------------------
// other launch helpers
// ------------------------------------------------------------------------------------------------
static int launch_ln(gitb200_engine* h, const LnParams& p, int D, cudaStream_t st, bool pdl = false) {
  const int grid = (p.rows + 7) / 8;
  if (D == 768 && pdl) CK(launch_k(true, layernorm_kernel<768, true>, dim3(grid), dim3(256), 0, st, p));
  else if (D == 768) CK(launch_k(false, layernorm_kernel<768, false>, dim3(grid), dim3(256), 0, st, p));
  else if (D == 1024) CK(launch_k(pdl, layernorm_kernel<1024, false>, dim3(grid), dim3(256), 0, st, p));
  else return fail(h, "layernorm: unsupported width %d", D);
  CKL(h, "layernorm_kernel");
  return 0;
}
static LnParams ln_params(const float* x, const float* bias, const float* resid, const float* g, const float* b,
                          float eps, float* of32, bf16* obf16, int rows) {
  LnParams p{};
  p.x = x; p.bias = bias; p.resid = resid; p.gamma = g; p.beta = b; p.eps = eps;
  p.out_f32 = of32; p.out_bf16 = obf16; p.rows = rows;
  return p;
}
// ln_params whose bf16 output is the next GEMM's A operand: [hi | lo | hi] rows in parity mode.
static LnParams ln_operand(const gitb200_engine* h, const float* x, const float* g, const float* b, float eps, float* of32,
                           bf16* obf16, int rows) {
  LnParams p = ln_params(x, nullptr, nullptr, g, b, eps, of32, obf16, rows);
  p.split3 = h->parity ? 1 : 0;
  return p;
}

// Self attention (attention.cuh): non-causal, B batches of S rows.  q / k / v rows q_rs / kv_rs elements apart and batches
// q_bs / kv_bs apart; out rows o_rs apart and batches o_bs apart.  bf16: flash_attn_wgmma_kernel, which reads whole
// batches by TMA (batches back to back, 16-byte aligned bases and pitches: get_tmap checks).  fp32 (parity mode):
// attn_f32_kernel, fp32 q / k / v and out rows in the [hi | lo | hi] format of 3 * H * 64 columns.
struct SelfAttn {
  const void* q;
  const void* k;
  const void* v;
  bf16* out;
  int B, S, H;
  long long q_rs, kv_rs, q_bs, kv_bs, o_rs, o_bs;
  const int* seq_lens;   // null, or [B] valid rows of each batch
};
static int launch_self_attention(gitb200_engine* h, const SelfAttn& a, bool fp32, cudaStream_t st) {
  if (fp32) {
    AttnF32Params p{};
    p.q = static_cast<const float*>(a.q); p.k = static_cast<const float*>(a.k); p.v = static_cast<const float*>(a.v);
    p.out = a.out;
    p.B = a.B; p.S = a.S; p.H = a.H; p.d_model = a.H * 64;
    p.q_rs = a.q_rs; p.kv_rs = a.kv_rs; p.q_bs = a.q_bs; p.kv_bs = a.kv_bs; p.o_bs = a.o_bs;
    p.seq_lens = a.seq_lens;
    const size_t smem = static_cast<size_t>(4) * (64 + p.S) * sizeof(float);
    if (smem > 200 * 1024) return fail(h, "parity attention: %d keys do not fit in shared memory", p.S);
    TRY(set_dyn_smem(h, reinterpret_cast<const void*>(attn_f32_kernel), smem));
    const long long items = static_cast<long long>(p.B) * p.H * p.S;
    attn_f32_kernel<<<static_cast<unsigned int>((items + 3) / 4), 128, smem, st>>>(p);
    CKL(h, "attn_f32_kernel");
    return 0;
  }
  if (a.q_bs != static_cast<long long>(a.S) * a.q_rs || a.kv_bs != static_cast<long long>(a.S) * a.kv_rs)
    return fail(h, "attention: batches must be stored back to back (batch stride = S * row stride)");
  AttnParams p{};
  p.q = static_cast<const bf16*>(a.q); p.k = static_cast<const bf16*>(a.k); p.v = static_cast<const bf16*>(a.v);
  p.out = a.out;
  p.B = a.B; p.S = a.S; p.H = a.H;
  p.q_rs = a.q_rs; p.kv_rs = a.kv_rs; p.q_bs = a.q_bs; p.kv_bs = a.kv_bs; p.o_rs = a.o_rs; p.o_bs = a.o_bs;
  p.scale_log2 = 0.125f * 1.44269504088896340736f;
  p.seq_lens = a.seq_lens;
  const long long rows = static_cast<long long>(a.B) * a.S;
  CUtensorMap tq, tk, tv;
  TRY(get_tmap(h, a.q, rows, a.H * 64, a.q_rs, kAttnWgRows, &tq));
  TRY(get_tmap(h, a.k, rows, a.H * 64, a.kv_rs, kAttnWgRows, &tk));
  TRY(get_tmap(h, a.v, rows, a.H * 64, a.kv_rs, kAttnWgRows, &tv));
  const dim3 grid((a.S + kAttnWgRows - 1) / kAttnWgRows, a.H, a.B);
  if (a.seq_lens != nullptr) flash_attn_wgmma_kernel<true><<<grid, 128, kAttnWgSmem, st>>>(tq, tk, tv, p);
  else flash_attn_wgmma_kernel<false><<<grid, 128, kAttnWgSmem, st>>>(tq, tk, tv, p);
  CKL(h, "flash_attn_wgmma_kernel");
  return 0;
}

// Text attention of caption scoring (attention.cuh): q / k / v [N * T, H * 64] (row n * T + t = position t of caption n)
// back to back, image K / V [B * M, H * 64]; caption n attends to image image_index[n] (null: image n), img_lens (null, or
// [B]) limits its keys.  bf16: text_attn_wgmma_kernel, out rows o_rs apart.  fp32 (parity mode): text_attn_f32_kernel, out
// rows [hi | lo | hi] of 3 * H * 64 columns.
struct TextAttn {
  const void* q;
  const void* k;
  const void* v;
  const void* img_k;
  const void* img_v;
  bf16* out;
  int N, T, B, M, H;
  long long o_rs;
  const int* img_lens;
  const int* image_index;
};
static int launch_text_attention(gitb200_engine* h, const TextAttn& a, bool fp32, cudaStream_t st) {
  if (fp32) {
    TextAttnF32Params p{};
    p.q = static_cast<const float*>(a.q); p.k = static_cast<const float*>(a.k); p.v = static_cast<const float*>(a.v);
    p.img_k = static_cast<const float*>(a.img_k); p.img_v = static_cast<const float*>(a.img_v); p.out = a.out;
    p.N = a.N; p.T = a.T; p.H = a.H; p.d_model = a.H * 64; p.M = a.M; p.img_lens = a.img_lens; p.image_index = a.image_index;
    const size_t smem = static_cast<size_t>(4) * (64 + p.M + p.T) * sizeof(float);
    if (smem > 200 * 1024) return fail(h, "parity text attention: %d keys do not fit in shared memory", p.M + p.T);
    TRY(set_dyn_smem(h, reinterpret_cast<const void*>(text_attn_f32_kernel), smem));
    const long long items = static_cast<long long>(p.N) * p.H * p.T;
    text_attn_f32_kernel<<<static_cast<unsigned int>((items + 3) / 4), 128, smem, st>>>(p);
    CKL(h, "text_attn_f32_kernel");
    return 0;
  }
  TextAttnParams p{};
  p.out = a.out; p.N = a.N; p.T = a.T; p.H = a.H; p.M = a.M; p.img_lens = a.img_lens; p.image_index = a.image_index;
  p.o_rs = a.o_rs;
  p.scale_log2 = 0.125f * 1.44269504088896340736f;
  const long long rows = static_cast<long long>(a.N) * a.T, irows = static_cast<long long>(a.B) * a.M, cols = a.H * 64;
  CUtensorMap tq, tk, tv, tik, tiv;
  TRY(get_tmap(h, a.q, rows, cols, cols, kAttnWgRows, &tq));
  TRY(get_tmap(h, a.k, rows, cols, cols, kAttnWgRows, &tk));
  TRY(get_tmap(h, a.v, rows, cols, cols, kAttnWgRows, &tv));
  TRY(get_tmap(h, a.img_k, irows, cols, cols, kAttnWgRows, &tik));
  TRY(get_tmap(h, a.img_v, irows, cols, cols, kAttnWgRows, &tiv));
  const dim3 grid((a.T + kAttnWgRows - 1) / kAttnWgRows, a.H, a.N);
  text_attn_wgmma_kernel<<<grid, 128, kAttnWgSmem, st>>>(tq, tk, tv, tik, tiv, p);
  CKL(h, "text_attn_wgmma_kernel");
  return 0;
}

// Geometry of decode_attn_kernel for image slots of M keys (lens: null, or the n valid key counts of a ragged batch) and
// `items` (image, head) pairs.  The image K/V slice of one item is M rows of 128 B, staged in chunks of at most
// kDecAttnChunk rows: two (K + V) staging buffers of one chunk per CTA, and at least two CTAs per SM (M = 257 in one piece
// would be 131 KB per CTA = one 4-warp CTA per SM).  A uniform chunk is one TMA box.
static DecAttnGeom dec_attn_geometry(int M, const int* lens, int n, int num_sms, int items, int beam) {
  DecAttnGeom g;
  g.box_rows = g.chunk_rows = dec_attn_chunk_rows(M);
  if (lens != nullptr) {
    // every image is chunked by its own key count (dec_attn_chunk_rows) and fetched in 32-row boxes: the staging buffer
    // holds the longest chunk of the call rounded up to whole boxes
    int rows = 0;
    for (int b = 0; b < n; ++b) rows = std::max(rows, dec_attn_chunk_rows(lens[b]));
    g.box_rows = kDecAttnRaggedBox;
    g.chunk_rows = (rows + kDecAttnRaggedBox - 1) / kDecAttnRaggedBox * kDecAttnRaggedBox;
  }
  g.smem = static_cast<size_t>(4) * g.chunk_rows * 128 + 128;
  // + an upper bound of the kernel's static shared memory and the 1 KB per-CTA reserve, which come to 7 KB at NQ 4 and
  // 8 / 9 / 10 / 12 KB at NQ 5 .. 8 (ptxas)
  const size_t fixed = static_cast<size_t>(std::max(8, beam + 4)) * 1024;
  int per_sm = static_cast<int>((227 * 1024) / (g.smem + fixed));
  per_sm = std::max(1, std::min(per_sm, 4));
  g.grid = std::min(items, per_sm * num_sms);
  return g;
}

template <int NQ, bool kRagged>
static int launch_decode_attn_inst(gitb200_engine* h, const DecAttnParams& ap, int grid, size_t smem, bool pdl,
                                   cudaStream_t st, const CUtensorMap& tk, const CUtensorMap& tv) {
  TRY(set_dyn_smem(h, reinterpret_cast<const void*>(decode_attn_kernel<NQ, kRagged>), smem));
  CK(launch_k(pdl, decode_attn_kernel<NQ, kRagged>, dim3(grid), dim3(128), smem, st, tk, tv, ap));
  CKL(h, "decode_attn_kernel");
  return 0;
}

// Decode-step attention (attention.cuh) of B images x seqs sequences x beam rows at one text position (state->pos, or pos_fixed when state
// is null): adds the QKV GEMM's n_partials split-K buffers and the bias, appends k / v to the text cache [R, T_alloc, D]
// (rows through src_row when non-null) and attends to the image K/V [B, M, D] (img_lens: null, or [B] valid keys) and the
// text keys so far; the seqs sequences of an image (row groups of beam rows) read its one image K/V.  bf16:
// decode_attn_kernel<beam, ragged> over B * seqs groups, with geom from dec_attn_geometry.  fp32 (parity mode):
// decode_attn_f32_kernel, one warp per (row, head), ctx rows [hi | lo | hi].  *ctas receives the grid.
struct DecodeAttn {
  const float* qkv;
  int n_partials;
  const float* bqkv;
  const void* img_k;
  const void* img_v;
  void* txt_k;
  void* txt_v;
  const int* src_row;
  bf16* ctx;
  int B, seqs, beam, M, T_alloc, D;
  const StepState* state;
  int pos_fixed;
  const int* img_lens;
  DecAttnGeom geom;
  ChainSync chain;
  bool pdl;
};
static int launch_decode_attention(gitb200_engine* h, const DecodeAttn& a, bool fp32, cudaStream_t st, unsigned int* ctas) {
  const int R = a.B * a.seqs * a.beam;
  if (fp32) {
    DecAttnF32Params p{};
    p.qkv = a.qkv; p.n_partials = a.n_partials; p.partial_stride = static_cast<long long>(R) * 3 * a.D;
    p.bqkv = a.bqkv;
    p.img_k = static_cast<const float*>(a.img_k); p.img_v = static_cast<const float*>(a.img_v);
    p.txt_k = static_cast<float*>(a.txt_k); p.txt_v = static_cast<float*>(a.txt_v);
    p.src_row = a.src_row; p.ctx = a.ctx; p.R = R; p.rows_per_image = a.seqs * a.beam; p.M = a.M; p.T_alloc = a.T_alloc; p.D = a.D;
    p.state = a.state; p.pos_fixed = a.pos_fixed;
    p.chain = a.chain;
    p.img_lens = a.img_lens;
    const size_t smem = static_cast<size_t>(4) * dec_attn_f32_warp_floats(p.M, p.T_alloc) * sizeof(float);
    if (smem > 200 * 1024) return fail(h, "parity decode attention: %d keys do not fit in shared memory", p.M + p.T_alloc);
    TRY(set_dyn_smem(h, reinterpret_cast<const void*>(decode_attn_f32_kernel), smem));
    *ctas = static_cast<unsigned int>((R * (p.D / 64) + 3) / 4);
    CK(launch_k(a.pdl, decode_attn_f32_kernel, dim3(*ctas), dim3(128), smem, st, p));
    CKL(h, "decode_attn_f32_kernel");
    return 0;
  }
  DecAttnParams p{};
  p.qkv = a.qkv; p.n_partials = a.n_partials; p.partial_stride = static_cast<long long>(R) * 3 * a.D;
  p.bqkv = a.bqkv;
  p.img_k = static_cast<const bf16*>(a.img_k); p.img_v = static_cast<const bf16*>(a.img_v);
  p.txt_k = static_cast<bf16*>(a.txt_k); p.txt_v = static_cast<bf16*>(a.txt_v);
  p.src_row = a.src_row; p.ctx = a.ctx; p.B = a.B * a.seqs; p.seqs_per_image = a.seqs; p.M = a.M; p.T_alloc = a.T_alloc; p.D = a.D;
  p.state = a.state; p.pos_fixed = a.pos_fixed;
  p.chunk_rows = a.geom.chunk_rows; p.box_rows = a.geom.box_rows;
  p.chain = a.chain;
  p.img_lens = a.img_lens;
  CUtensorMap tk, tv;
  TRY(get_tmap(h, a.img_k, static_cast<long long>(a.B) * a.M, a.D, a.D, a.geom.box_rows, &tk, false));
  TRY(get_tmap(h, a.img_v, static_cast<long long>(a.B) * a.M, a.D, a.D, a.geom.box_rows, &tv, false));
  const bool rg = a.img_lens != nullptr;
  const int grid = a.geom.grid;
  const size_t smem = a.geom.smem;
  *ctas = static_cast<unsigned int>(grid);
  switch (a.beam) {
    case 1: return rg ? launch_decode_attn_inst<1, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<1, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 2: return rg ? launch_decode_attn_inst<2, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<2, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 3: return rg ? launch_decode_attn_inst<3, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<3, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 4: return rg ? launch_decode_attn_inst<4, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<4, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 5: return rg ? launch_decode_attn_inst<5, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<5, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 6: return rg ? launch_decode_attn_inst<6, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<6, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 7: return rg ? launch_decode_attn_inst<7, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<7, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    case 8: return rg ? launch_decode_attn_inst<8, true>(h, p, grid, smem, a.pdl, st, tk, tv)
                      : launch_decode_attn_inst<8, false>(h, p, grid, smem, a.pdl, st, tk, tv);
    default: return fail(h, "decode: beam size %d not supported (1 .. 8)", a.beam);
  }
}

__global__ void cvt_rows_kernel(const float* __restrict__ src, long long src_ld, bf16* __restrict__ dst, long long dst_ld,
                                long long rows, long long cols, long long dst_cols) {
  const long long total = rows * dst_cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dst_cols, c = i - r * dst_cols;
    dst[r * dst_ld + c] = __float2bfloat16_rn(c < cols ? src[r * src_ld + c] : 0.0f);
  }
}
// parity mode weights: [rows, 3 * dst_cols] = [hi | hi | lo]
__global__ void cvt_rows_split3_kernel(const float* __restrict__ src, long long src_ld, bf16* __restrict__ dst, long long rows,
                                       long long cols, long long dst_cols) {
  const long long total = rows * dst_cols;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / dst_cols, c = i - r * dst_cols;
    bf16 hi, lo;
    split_bf16(c < cols ? src[r * src_ld + c] : 0.0f, hi, lo);
    bf16* d = dst + r * 3 * dst_cols + c;
    d[0] = hi; d[dst_cols] = hi; d[2 * dst_cols] = lo;
  }
}
__global__ void sum_partials_kernel(const float* __restrict__ parts, float* __restrict__ out, long long n, int splits) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a = parts[i];
    for (int s = 1; s < splits; ++s) a += parts[s * n + i];
    out[i] = a;
  }
}
__global__ void set_state_kernel(StepState* st, int pos, int cur_len, unsigned int* chain) {
  st->pos = pos; st->cur_len = cur_len; st->finished = 0; st->final_len = cur_len; st->step = 0;
  st->empty_caption = 0; st->ticket = 0; st->live = 0; st->error = 0; st->bad_draw = 0;
  for (int k = 0; k < 64; ++k) chain[k] = 0;
}
__global__ void init_generate_kernel(long long* tokens_out, long long* next_token, float* logprob_sum,
                                     const long long* prefix, int P, int rows, int max_steps, int sos, long long prefix_row_stride) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const long long* pr = prefix ? prefix + r * prefix_row_stride : nullptr;   // stride 0: one prefix for all rows
  for (int i = 0; i < P; ++i) tokens_out[static_cast<long long>(r) * max_steps + i] = pr ? pr[i] : sos;
  next_token[r] = pr ? pr[0] : sos;
  logprob_sum[r] = 0.f;
}
__global__ void advance_prefix_kernel(StepState* st, long long* next_token, const long long* prefix, int idx, int rows,
                                      unsigned int* chain) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < rows) next_token[r] = prefix[idx];
  if (r == 0) st->pos = st->pos + 1;
  if (r < 64) chain[r] = 0;
}

// ------------------------------------------------------------------------------------------------
// create / destroy / weights
// ------------------------------------------------------------------------------------------------
extern "C" int gitb200_abi_version(void) { return GITB200_ABI_VERSION; }

extern "C" const char* gitb200_last_error(const gitb200_engine* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

extern "C" int64_t gitb200_launch_count(const gitb200_engine* h) { return h ? h->launches : 0; }

extern "C" int gitb200_set_option(gitb200_engine* h, const char* name, int64_t value) {
  if (!h || !name) return 1;
  // the captured decode-step graph bakes the launch configuration in: drop it whenever an option changes
  drop_step_graphs(h);
  if (strcmp(name, "use_graph") == 0) { h->use_graph = value != 0; return 0; }
  if (strcmp(name, "use_pdl") == 0) { h->use_pdl = value != 0; return 0; }
  if (strcmp(name, "use_mega") == 0) { h->use_mega = value != 0; return 0; }
  if (strcmp(name, "debug_layers") == 0) { h->debug_layers = static_cast<int>(value); return 0; }
  if (strcmp(name, "parity") == 0) {
    if (h->weights_from != nullptr) return fail(h, "parity: this engine borrows its weights; switch the owning engine");
    if (h->parity != (value != 0)) { h->parity = value != 0; h->finalized = false; h->seen.clear(); h->tmaps.clear(); }
    return 0;
  }
  return fail(h, "unknown option %s", name);
}

// The size checks of both size setters: 0, or fails with "<what>: <image><size> ..." (image: "" or "image b ").
static int check_image_size(gitb200_engine* h, const char* what, int b, int height, int width) {
  const int p = h->cfg.patch;
  const long long tokens = static_cast<long long>(height / p) * (width / p) + 1;
  if (b < 0) {
    if (height < p || width < p) return fail(h, "%s: %dx%d is smaller than one %dx%d patch", what, height, width, p, p);
    if (tokens > 16384) return fail(h, "%s: %dx%d gives %lld tokens per image (limit 16384)", what, height, width, tokens);
    return 0;
  }
  if (height < p || width < p) return fail(h, "%s: image %d is %dx%d, smaller than one %dx%d patch", what, b, height, width, p, p);
  if (tokens > 16384) return fail(h, "%s: image %d (%dx%d) gives %lld tokens (limit 16384)", what, b, height, width, tokens);
  return 0;
}

extern "C" int gitb200_set_input_size(gitb200_engine* h, int height, int width) {
  if (!h) return 1;
  if (h->pending) return fail(h, "set_input_size: a generate call is in flight");
  TRY(check_image_size(h, "set_input_size", -1, height, width));
  h->in_h = height;
  h->in_w = width;
  return 0;
}

extern "C" int gitb200_set_image_sizes(gitb200_engine* h, const int32_t* hw_host, int n) {
  if (!h) return 1;
  if (h->pending) return fail(h, "set_image_sizes: a generate call is in flight");
  if (!hw_host || n < 1) return fail(h, "set_image_sizes: bad argument");
  for (int b = 0; b < n; ++b) TRY(check_image_size(h, "set_image_sizes", b, hw_host[2 * b], hw_host[2 * b + 1]));
  h->next.image_hw.assign(hw_host, hw_host + 2 * n);
  return 0;
}

extern "C" int gitb200_create(const gitb200_config* cfg, int device, gitb200_engine** out) {
  gitb200_engine* h = nullptr;
  if (!cfg || !out) return fail(nullptr, "gitb200_create: null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
    return fail(nullptr, "gitb200_create: no CUDA device visible (this engine has no CPU path)");
  if (device < 0 || device >= ndev) return fail(nullptr, "gitb200_create: bad device %d", device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(nullptr, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, "gitb200_create: device %d is sm_%d%d; this library contains sm_90a code only", device, prop.major, prop.minor);
  if (cfg->image_size % cfg->patch != 0) return fail(nullptr, "image_size %% patch != 0");
  if (cfg->enc_width != 768 && cfg->enc_width != 1024) return fail(nullptr, "enc_width must be 768 or 1024");
  if (cfg->dec_hidden != 768 || cfg->dec_heads * 64 != cfg->dec_hidden || cfg->enc_heads * 64 != cfg->enc_width)
    return fail(nullptr, "head dim must be 64 and dec_hidden 768");
  if (cfg->dec_ffn % 64 != 0) return fail(nullptr, "dec_ffn must be a multiple of 64");
  h = new gitb200_engine();
  h->cfg = *cfg;
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  h->g = cfg->image_size / cfg->patch;
  h->L = h->g * h->g + 1;
  h->in_h = h->in_w = cfg->image_size;
  h->Kpatch = 3 * cfg->patch * cfg->patch;
  h->Kp = (h->Kpatch + 63) / 64 * 64;
  h->d = cfg->enc_width;
  h->D = cfg->dec_hidden;
  h->F = cfg->dec_ffn;
  h->V = cfg->vocab;
  h->enc.resize(cfg->enc_layers);
  h->dec.resize(cfg->dec_layers);
  cudaSetDevice(device);
  *out = h;
  return 0;
}

static void release_all(gitb200_engine* h) {
  DevBuf* bufs[] = {&h->w_patch, &h->cls, &h->pos_emb, &h->lnpre_g, &h->lnpre_b, &h->lnpost_g, &h->lnpost_b, &h->w_vp,
                    &h->b_vp, &h->lnvp_g, &h->lnvp_b, &h->words_f32, &h->words_bf16, &h->positions, &h->lnemb_g,
                    &h->lnemb_b, &h->out_bias, &h->temb, &h->m_lm, &h->y_t, &h->qb_t, &h->mega_bar, &h->x, &h->h, &h->qkv, &h->ctx, &h->u, &h->feats, &h->feats_f32, &h->pos_interp,
                    &h->pt, &h->pxd, &h->phd, &h->pq, &h->pctx, &h->pu, &h->img_kv, &h->txt_kv, &h->src_row[0],
                    &h->src_row[1], &h->xd_t, &h->hd_t, &h->qkv_t, &h->ctx_t, &h->t_t, &h->u_t, &h->logits, &h->state,
                    &h->next_token, &h->logprob_sum, &h->tokens_i64, &h->stage_img, &h->stage_tok, &h->stage_lp,
                    &h->prefix_dev, &h->beam_ws, &h->sel_ws, &h->chain, &h->rg_tab, &h->rg_lens, &h->sc_kv,
                    &h->sc_tgt, &h->sc_part, &h->sc_loss, &h->sc_valid, &h->sc_index};
  for (DevBuf* b : bufs) b->release();
  for (auto& l : h->enc) {
    DevBuf* lb[] = {&l.wqkv, &l.bqkv, &l.wo, &l.bo, &l.ln1g, &l.ln1b, &l.ln2g, &l.ln2b, &l.w1, &l.b1, &l.w2, &l.b2};
    for (DevBuf* b : lb) b->release();
  }
  for (auto& l : h->dec) {
    DevBuf* lb[] = {&l.wqkv, &l.bqkv, &l.wo, &l.bo, &l.lnag, &l.lnab, &l.w1, &l.b1, &l.w2, &l.b2, &l.lnog, &l.lnob,
                    &l.m_wqkv, &l.m_wo, &l.m_w1, &l.m_w2};
    for (DevBuf* b : lb) b->release();
  }
}

// Weight buffers of an engine, in a fixed order (the same for every engine of one geometry).
static std::vector<DevBuf*> weight_bufs(gitb200_engine* h) {
  std::vector<DevBuf*> v = {&h->w_patch, &h->cls, &h->pos_emb, &h->lnpre_g, &h->lnpre_b, &h->lnpost_g, &h->lnpost_b, &h->w_vp,
                            &h->b_vp, &h->lnvp_g, &h->lnvp_b, &h->words_f32, &h->words_bf16, &h->positions, &h->lnemb_g,
                            &h->lnemb_b, &h->out_bias, &h->temb, &h->m_lm};
  for (auto& l : h->enc)
    for (DevBuf* b : {&l.wqkv, &l.bqkv, &l.wo, &l.bo, &l.ln1g, &l.ln1b, &l.ln2g, &l.ln2b, &l.w1, &l.b1, &l.w2, &l.b2}) v.push_back(b);
  for (auto& l : h->dec)
    for (DevBuf* b : {&l.wqkv, &l.bqkv, &l.wo, &l.bo, &l.lnag, &l.lnab, &l.w1, &l.b1, &l.w2, &l.b2, &l.lnog, &l.lnob,
                      &l.m_wqkv, &l.m_wo, &l.m_w1, &l.m_w2}) v.push_back(b);
  return v;
}

extern "C" int gitb200_share_weights(gitb200_engine* h, gitb200_engine* src) {
  if (!h || !src) return 1;
  if (h == src) return fail(h, "share_weights: an engine cannot borrow from itself");
  if (!src->finalized) return fail(h, "share_weights: the source engine's weights are not finalized");
  if (src->weights_from != nullptr) return fail(h, "share_weights: the source engine borrows its weights itself");
  if (h->device != src->device) return fail(h, "share_weights: engines live on different devices");
  if (memcmp(&h->cfg, &src->cfg, sizeof(gitb200_config)) != 0) return fail(h, "share_weights: geometries differ");
  if (h->pending) return fail(h, "share_weights: a generate call is in flight");
  std::vector<DevBuf*> dst = weight_bufs(h), from = weight_bufs(src);
  for (size_t i = 0; i < dst.size(); ++i) dst[i]->borrow(*from[i]);
  h->tmaps.clear();
  drop_step_graphs(h);
  h->seen = src->seen;
  h->parity = src->parity;
  h->mega_ready = src->mega_ready;
  h->finalized = true;
  h->weights_from = src;
  return 0;
}

extern "C" void gitb200_destroy(gitb200_engine* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  drop_step_graphs(h);
  if (h->host_state) cudaFreeHost(h->host_state);
  if (h->own_event) cudaEventDestroy(h->own_event);
  for (int i = 0; i < 2; ++i) if (h->chunk_ev[i]) cudaEventDestroy(h->chunk_ev[i]);
  for (int i = 0; i < 2; ++i) if (h->dec_ev[i]) cudaEventDestroy(h->dec_ev[i]);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  release_all(h);
  delete h;
}

// Copy an fp32 source tensor into an engine buffer: fp32 (as is) or bf16 [rows, dst_cols] with zero padding,
// at a row offset inside the destination (used to fuse q/k/v into one matrix).
static int store_f32(gitb200_engine* h, DevBuf& dst, size_t total_elems, size_t elem_off, const float* src, size_t n,
                     cudaStream_t st) {
  CK(dst.ensure(total_elems * sizeof(float)));
  CK(cudaMemcpyAsync(dst.as<float>() + elem_off, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return 0;
}
static int store_bf16(gitb200_engine* h, DevBuf& dst, long long total_rows, long long dst_cols, long long row_off,
                      const float* src, long long rows, long long cols, cudaStream_t st) {
  CK(dst.ensure(static_cast<size_t>(total_rows) * dst_cols * h->ks() * sizeof(bf16)));
  const long long total = rows * dst_cols;
  const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(h->num_sms) * 16));
  if (h->parity) cvt_rows_split3_kernel<<<grid, 256, 0, st>>>(src, cols, dst.as<bf16>() + row_off * 3 * dst_cols, rows, cols, dst_cols);
  else cvt_rows_kernel<<<grid, 256, 0, st>>>(src, cols, dst.as<bf16>() + row_off * dst_cols, dst_cols, rows, cols, dst_cols);
  CKL(h, "cvt_rows_kernel");
  return 0;
}

static bool shape_is(const int64_t* s, int nd, std::initializer_list<int64_t> want) {
  if (nd != static_cast<int>(want.size())) return false;
  int i = 0;
  for (int64_t w : want) if (s[i++] != w) return false;
  return true;
}

extern "C" int gitb200_set_weight(gitb200_engine* h, const char* ref_key, const void* dev_ptr, const int64_t* shape,
                                  int ndim, int dtype, void* stream) {
  if (!h) return 1;
  if (!ref_key || !dev_ptr || !shape) return fail(h, "set_weight: null argument");
  if (dtype != GITB200_F32) return fail(h, "set_weight(%s): only fp32 sources are accepted", ref_key);
  cudaSetDevice(h->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float* src = static_cast<const float*>(dev_ptr);
  const std::string key(ref_key);
  const int d = h->d, D = h->D, F = h->F, V = h->V, L = h->L;
  auto bad_shape = [&]() { return fail(h, "set_weight(%s): unexpected shape", ref_key); };
  if (h->weights_from != nullptr) return fail(h, "set_weight(%s): this engine borrows its weights (gitb200_share_weights)", ref_key);
  h->finalized = false;
  int layer = -1;
  char sub[128];
  if (key == "image_encoder.proj" || key == "textual.output.weight") { h->seen.insert(key); return 0; }
  if (key == "image_encoder.class_embedding") {
    if (!shape_is(shape, ndim, {d})) return bad_shape();
    TRY(store_f32(h, h->cls, d, 0, src, d, st));
  } else if (key == "image_encoder.positional_embedding") {
    if (!shape_is(shape, ndim, {L, d})) return bad_shape();
    TRY(store_f32(h, h->pos_emb, static_cast<size_t>(L) * d, 0, src, static_cast<size_t>(L) * d, st));
  } else if (key == "image_encoder.conv1.weight") {
    if (!shape_is(shape, ndim, {d, 3, h->cfg.patch, h->cfg.patch})) return bad_shape();
    TRY(store_bf16(h, h->w_patch, d, h->Kp, 0, src, d, h->Kpatch, st));
  } else if (key == "image_encoder.ln_pre.weight") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, h->lnpre_g, d, 0, src, d, st));
  } else if (key == "image_encoder.ln_pre.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, h->lnpre_b, d, 0, src, d, st));
  } else if (key == "image_encoder.ln_post.weight") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, h->lnpost_g, d, 0, src, d, st));
  } else if (key == "image_encoder.ln_post.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, h->lnpost_b, d, 0, src, d, st));
  } else if (sscanf(ref_key, "image_encoder.transformer.resblocks.%d.%127s", &layer, sub) == 2) {
    if (layer < 0 || layer >= static_cast<int>(h->enc.size())) return fail(h, "set_weight(%s): layer out of range", ref_key);
    EncLayer& l = h->enc[layer];
    const std::string s(sub);
    if (s == "attn.in_proj_weight") { if (!shape_is(shape, ndim, {3 * d, d})) return bad_shape(); TRY(store_bf16(h, l.wqkv, 3 * d, d, 0, src, 3 * d, d, st)); }
    else if (s == "attn.in_proj_bias") { if (!shape_is(shape, ndim, {3 * d})) return bad_shape(); TRY(store_f32(h, l.bqkv, 3 * d, 0, src, 3 * d, st)); }
    else if (s == "attn.out_proj.weight") { if (!shape_is(shape, ndim, {d, d})) return bad_shape(); TRY(store_bf16(h, l.wo, d, d, 0, src, d, d, st)); }
    else if (s == "attn.out_proj.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.bo, d, 0, src, d, st)); }
    else if (s == "ln_1.weight") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.ln1g, d, 0, src, d, st)); }
    else if (s == "ln_1.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.ln1b, d, 0, src, d, st)); }
    else if (s == "ln_2.weight") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.ln2g, d, 0, src, d, st)); }
    else if (s == "ln_2.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.ln2b, d, 0, src, d, st)); }
    else if (s == "mlp.c_fc.weight") { if (!shape_is(shape, ndim, {4 * d, d})) return bad_shape(); TRY(store_bf16(h, l.w1, 4 * d, d, 0, src, 4 * d, d, st)); }
    else if (s == "mlp.c_fc.bias") { if (!shape_is(shape, ndim, {4 * d})) return bad_shape(); TRY(store_f32(h, l.b1, 4 * d, 0, src, 4 * d, st)); }
    else if (s == "mlp.c_proj.weight") { if (!shape_is(shape, ndim, {d, 4 * d})) return bad_shape(); TRY(store_bf16(h, l.w2, d, 4 * d, 0, src, d, 4 * d, st)); }
    else if (s == "mlp.c_proj.bias") { if (!shape_is(shape, ndim, {d})) return bad_shape(); TRY(store_f32(h, l.b2, d, 0, src, d, st)); }
    else return fail(h, "set_weight: unknown key %s", ref_key);
  } else if (key == "textual.visual_projection.0.weight") {
    if (!shape_is(shape, ndim, {D, d})) return bad_shape();
    TRY(store_bf16(h, h->w_vp, D, d, 0, src, D, d, st));
  } else if (key == "textual.visual_projection.0.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, h->b_vp, D, 0, src, D, st));
  } else if (key == "textual.visual_projection.1.weight") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, h->lnvp_g, D, 0, src, D, st));
  } else if (key == "textual.visual_projection.1.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, h->lnvp_b, D, 0, src, D, st));
  } else if (key == "textual.embedding.words.weight") {
    if (!shape_is(shape, ndim, {V, D})) return bad_shape();
    TRY(store_f32(h, h->words_f32, static_cast<size_t>(V) * D, 0, src, static_cast<size_t>(V) * D, st));
    TRY(store_bf16(h, h->words_bf16, V, D, 0, src, V, D, st));
  } else if (key == "textual.embedding.positions.weight") {
    if (!shape_is(shape, ndim, {h->cfg.max_positions, D})) return bad_shape();
    TRY(store_f32(h, h->positions, static_cast<size_t>(h->cfg.max_positions) * D, 0, src, static_cast<size_t>(h->cfg.max_positions) * D, st));
  } else if (key == "textual.embedding.layer_norm.weight") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, h->lnemb_g, D, 0, src, D, st));
  } else if (key == "textual.embedding.layer_norm.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, h->lnemb_b, D, 0, src, D, st));
  } else if (key == "textual.output.bias") { if (!shape_is(shape, ndim, {V})) return bad_shape(); TRY(store_f32(h, h->out_bias, V, 0, src, V, st));
  } else if (sscanf(ref_key, "textual.transformer.encoder.layer.%d.%127s", &layer, sub) == 2) {
    if (layer < 0 || layer >= static_cast<int>(h->dec.size())) return fail(h, "set_weight(%s): layer out of range", ref_key);
    DecLayer& l = h->dec[layer];
    const std::string s(sub);
    const char* qkvn[3] = {"query", "key", "value"};
    bool done = false;
    for (int i = 0; i < 3 && !done; ++i) {
      if (s == std::string("attention.self.") + qkvn[i] + ".weight") {
        if (!shape_is(shape, ndim, {D, D})) return bad_shape();
        TRY(store_bf16(h, l.wqkv, 3 * D, D, static_cast<long long>(i) * D, src, D, D, st));
        done = true;
      } else if (s == std::string("attention.self.") + qkvn[i] + ".bias") {
        if (!shape_is(shape, ndim, {D})) return bad_shape();
        TRY(store_f32(h, l.bqkv, 3 * D, static_cast<size_t>(i) * D, src, D, st));
        done = true;
      }
    }
    if (done) { /* stored */ }
    else if (s == "attention.output.dense.weight") { if (!shape_is(shape, ndim, {D, D})) return bad_shape(); TRY(store_bf16(h, l.wo, D, D, 0, src, D, D, st)); }
    else if (s == "attention.output.dense.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.bo, D, 0, src, D, st)); }
    else if (s == "attention.output.LayerNorm.weight") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.lnag, D, 0, src, D, st)); }
    else if (s == "attention.output.LayerNorm.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.lnab, D, 0, src, D, st)); }
    else if (s == "intermediate.dense.weight") { if (!shape_is(shape, ndim, {F, D})) return bad_shape(); TRY(store_bf16(h, l.w1, F, D, 0, src, F, D, st)); }
    else if (s == "intermediate.dense.bias") { if (!shape_is(shape, ndim, {F})) return bad_shape(); TRY(store_f32(h, l.b1, F, 0, src, F, st)); }
    else if (s == "output.dense.weight") { if (!shape_is(shape, ndim, {D, F})) return bad_shape(); TRY(store_bf16(h, l.w2, D, F, 0, src, D, F, st)); }
    else if (s == "output.dense.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.b2, D, 0, src, D, st)); }
    else if (s == "output.LayerNorm.weight") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.lnog, D, 0, src, D, st)); }
    else if (s == "output.LayerNorm.bias") { if (!shape_is(shape, ndim, {D})) return bad_shape(); TRY(store_f32(h, l.lnob, D, 0, src, D, st)); }
    else return fail(h, "set_weight: unknown key %s", ref_key);
  } else if (sscanf(ref_key, "img_temperal_embedding.%d", &layer) == 1) {
    if (layer < 0 || layer >= h->cfg.num_frames_emb) return fail(h, "set_weight(%s): frame out of range", ref_key);
    if (!shape_is(shape, ndim, {1, 1, d})) return bad_shape();
    TRY(store_f32(h, h->temb, static_cast<size_t>(h->cfg.num_frames_emb) * d, static_cast<size_t>(layer) * d, src, d, st));
  } else {
    return fail(h, "set_weight: unknown key %s", ref_key);
  }
  h->seen.insert(key);
  return 0;
}

extern "C" int gitb200_finalize_weights(gitb200_engine* h, void* stream) {
  if (!h) return 1;
  cudaSetDevice(h->device);
  std::vector<std::string> need = {"image_encoder.class_embedding", "image_encoder.positional_embedding",
                                   "image_encoder.conv1.weight", "image_encoder.ln_pre.weight", "image_encoder.ln_pre.bias",
                                   "image_encoder.ln_post.weight", "image_encoder.ln_post.bias",
                                   "textual.visual_projection.0.weight", "textual.visual_projection.0.bias",
                                   "textual.visual_projection.1.weight", "textual.visual_projection.1.bias",
                                   "textual.embedding.words.weight", "textual.embedding.positions.weight",
                                   "textual.embedding.layer_norm.weight", "textual.embedding.layer_norm.bias",
                                   "textual.output.bias"};
  const char* encs[] = {"attn.in_proj_weight", "attn.in_proj_bias", "attn.out_proj.weight", "attn.out_proj.bias",
                        "ln_1.weight", "ln_1.bias", "ln_2.weight", "ln_2.bias", "mlp.c_fc.weight", "mlp.c_fc.bias",
                        "mlp.c_proj.weight", "mlp.c_proj.bias"};
  for (int i = 0; i < h->cfg.enc_layers; ++i)
    for (const char* s : encs) need.push_back("image_encoder.transformer.resblocks." + std::to_string(i) + "." + s);
  const char* decs[] = {"attention.self.query.weight", "attention.self.query.bias", "attention.self.key.weight",
                        "attention.self.key.bias", "attention.self.value.weight", "attention.self.value.bias",
                        "attention.output.dense.weight", "attention.output.dense.bias", "attention.output.LayerNorm.weight",
                        "attention.output.LayerNorm.bias", "intermediate.dense.weight", "intermediate.dense.bias",
                        "output.dense.weight", "output.dense.bias", "output.LayerNorm.weight", "output.LayerNorm.bias"};
  for (int j = 0; j < h->cfg.dec_layers; ++j)
    for (const char* s : decs) need.push_back("textual.transformer.encoder.layer." + std::to_string(j) + "." + s);
  for (int f = 0; f < h->cfg.num_frames_emb; ++f) need.push_back("img_temperal_embedding." + std::to_string(f));
  for (const std::string& k : need)
    if (!h->seen.count(k)) return fail(h, "finalize_weights: missing tensor %s", k.c_str());
  // fragment-packed weight tiles of the persistent decode-step kernel (decode_mega.cuh)
  h->mega_ready = false;
  if (!h->parity && h->D == kMegaD && h->F == kMegaF && h->cfg.dec_heads == kMegaH && h->cfg.dec_layers <= 6) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto pack = [&](DevBuf& dst, const DevBuf& src, long long ldw, int n_feat, int k0, long long n_tiles, int stride, int offset) -> int {
      CK(dst.ensure(static_cast<size_t>(n_tiles) * stride * kMegaTileBytes));
      const long long total = n_tiles * 48 * 32;
      pack_tiles_kernel<<<static_cast<int>(std::min<long long>((total + 255) / 256, static_cast<long long>(h->num_sms) * 16)), 256, 0, st>>>(
          src.as<bf16>(), ldw, n_feat, k0, dst.as<uint8_t>(), n_tiles, stride, offset);
      CKL(h, "pack_tiles_kernel");
      return 0;
    };
    for (auto& l : h->dec) {
      TRY(pack(l.m_wqkv, l.wqkv, h->D, 3 * h->D, 0, 3 * h->D / 8, 1, 0));
      TRY(pack(l.m_wo, l.wo, h->D, h->D, 0, h->D / 8, 1, 0));
      TRY(pack(l.m_w1, l.w1, h->D, h->F, 0, h->F / 8, 1, 0));
      for (int sl = 0; sl < kMegaFc2Slices; ++sl)   // k slice sl of feature tile f goes to tile mega_w2_tile(f, sl)
        TRY(pack(l.m_w2, l.w2, h->F, h->D, sl * kMegaD, h->D / 8, kMegaFc2Slices, sl));
    }
    TRY(pack(h->m_lm, h->words_bf16, h->D, h->V, 0, (h->V + 7) / 8, 1, 0));
    h->mega_ready = true;
  }
  CK(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  CK(cudaGetLastError());
  h->finalized = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// hot path A: encoder
// ------------------------------------------------------------------------------------------------
// The images of a call (include/gitb200.h gitb200_encode; frames < 1: a bare tensor, no temporal embeddings; hw: empty, or
// the (height, width) of each of the B images, set for this call by gitb200_set_image_sizes).  Each image gets the row
// of its grid in the call's positional table (pos_table): every image of the model's own grid reads the stored table,
// else the table holds one block per distinct grid in order of first appearance.
static int image_batch(gitb200_engine* h, const char* what, int B, int frames, const std::vector<int>& hw, ImageBatch* out) {
  ImageBatch& ib = *out;
  ib.B = B;
  ib.frames = frames < 1 ? 1 : frames;
  ib.list_input = frames >= 1;
  ib.ragged = !hw.empty();
  if (B < 1) return fail(h, "%s: bad batch/frames", what);
  if (ib.ragged && (static_cast<int>(hw.size()) != 2 * B || ib.frames != 1))
    return fail(h, "%s: %d image sizes were set for a batch of %d x %d frames (images of their own sizes take frames 0 or 1)",
                what, static_cast<int>(hw.size() / 2), B, ib.frames);
  ib.bytes = 3ULL * h->in_h * h->in_w * B * ib.frames * sizeof(float);
  if (ib.list_input && h->cfg.num_frames_emb > 0 && ib.frames > h->cfg.num_frames_emb) {
    // reference zip() truncates to the number of temporal embeddings (layers/decoder.py:848-849)
    ib.frames = h->cfg.num_frames_emb;
  }
  const int p = h->cfg.patch, NI = B * ib.frames;
  std::vector<std::pair<int, int>> grids;     // distinct (gh, gw) in order of first appearance
  std::vector<int> grid_row;                  // their first row in the positional table
  long long off = 0;
  ib.imgs.resize(NI);
  for (int i = 0; i < NI; ++i) {
    RaggedImg& e = ib.imgs[i];
    e.h = ib.ragged ? hw[2 * i] : h->in_h;
    e.w = ib.ragged ? hw[2 * i + 1] : h->in_w;
    e.gh = e.h / p;      // nn.Conv2d(kernel = stride = patch, no padding) drops a trailing partial patch
    e.gw = e.w / p;
    e.L = e.gh * e.gw + 1;
    e.src_off = off;
    off += 3LL * e.h * e.w;
    size_t k = 0;
    while (k < grids.size() && grids[k] != std::make_pair(e.gh, e.gw)) ++k;
    if (k == grids.size()) { grids.emplace_back(e.gh, e.gw); grid_row.push_back(ib.pos_rows); ib.pos_rows += e.L; }
    e.pos_row = grid_row[k];
    ib.L_max = std::max(ib.L_max, e.L);
    if (ib.ragged) ib.lens.push_back(e.L);
  }
  if (ib.ragged) ib.bytes = static_cast<size_t>(off) * sizeof(float);
  if (grids.size() == 1 && grids[0] == std::make_pair(h->g, h->g)) ib.pos_rows = 0;
  return 0;
}

// The positional table of a call's images (image_batch; reference layers/CLIP/model.py:245-251) -> *pos: the stored one,
// or pos_interp with the stored one copied for the model's own grid and the bicubic re-sampling for any other.  Made on
// every call: the parameters may have changed.
static int pos_table(gitb200_engine* h, const ImageBatch& ib, const float** pos, cudaStream_t st) {
  *pos = h->pos_emb.as<float>();
  if (ib.pos_rows == 0) return 0;
  const int d = h->d;
  CK(h->pos_interp.ensure(static_cast<size_t>(ib.pos_rows) * d * 4));
  int next = 0;   // the blocks are numbered in order of first appearance: the first image of a grid starts the next one
  for (const RaggedImg& e : ib.imgs) {
    if (e.pos_row != next) continue;
    float* dst = h->pos_interp.as<float>() + static_cast<size_t>(next) * d;
    next += e.L;
    if (e.gh == h->g && e.gw == h->g) {
      CK(cudaMemcpyAsync(dst, h->pos_emb.p, static_cast<size_t>(h->L) * d * 4, cudaMemcpyDeviceToDevice, st));
      continue;
    }
    const long long total = static_cast<long long>(e.L) * (d / 4);
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, h->num_sms * 8));
    pos_embed_bicubic_kernel<<<grid, 256, 0, st>>>(h->pos_emb.as<float>(), dst, h->g, e.gh, e.gw, d);
    CKL(h, "pos_embed_bicubic_kernel");
  }
  *pos = h->pos_interp.as<float>();
  return 0;
}

// Copies `bytes` from host memory to buf on `st` unless the last copy through here left exactly these bytes there (last;
// forgotten when buf is re-allocated or released, which changes its capacity).
static int upload_changed(gitb200_engine* h, DevBuf& buf, std::string& last, const void* src, size_t bytes, cudaStream_t st) {
  const size_t cap = buf.cap;
  CK(buf.ensure(bytes));
  if (buf.cap != cap) last.clear();
  if (last.size() == bytes && memcmp(last.data(), src, bytes) == 0) return 0;
  CK(cudaMemcpyAsync(buf.p, src, bytes, cudaMemcpyHostToDevice, st));
  last.assign(static_cast<const char*>(src), bytes);
  return 0;
}

// Valid image keys of each image on the device when the images of `ib` had their own sizes, else null.
static const int* img_lens(const gitb200_engine* h, const ImageBatch& ib) { return ib.ragged ? h->rg_lens.as<int>() : nullptr; }

static int encode_impl(gitb200_engine* h, const float* images, const ImageBatch& ib, float* feats_out, cudaStream_t st) {
  if (!h->finalized) return fail(h, "weights not finalized");
  h->cur_img.ragged = false;
  const int B = ib.B, frames = ib.frames, L = ib.L_max;
  TRY(upload_changed(h, h->rg_tab, h->rg_tab_up, ib.imgs.data(), ib.imgs.size() * sizeof(RaggedImg), st));
  if (ib.ragged) TRY(upload_changed(h, h->rg_lens, h->rg_lens_up, ib.lens.data(), ib.lens.size() * sizeof(int), st));
  const int d = h->d, Kp = h->Kp, H = h->cfg.enc_heads;
  const int NI = B * frames;
  const long long Me = static_cast<long long>(NI) * L;
  const int ks = h->ks();                 // parity mode: GEMM operands are [hi | lo | hi] -> 3x the K extent
  const bool par = h->parity;
  const size_t qkv_eb = h->kvb();         // q | k | v: bf16, fp32 in parity mode
  CK(h->x.ensure(Me * d * 4));
  CK(h->h.ensure(Me * d * 2 * ks));
  CK(h->qkv.ensure(Me * 3 * d * qkv_eb));
  CK(h->ctx.ensure(Me * d * 2 * ks));
  CK(h->u.ensure(std::max<long long>(Me * 4 * d * 2, static_cast<long long>(NI) * (L - 1) * Kp * 2) * ks));
  CK(h->feats.ensure(Me * d * 2 * ks));
  float* x = h->x.as<float>();
  bf16* hb = h->h.as<bf16>();
  bf16* ctx = h->ctx.as<bf16>();
  bf16* u = h->u.as<bf16>();
  const RaggedImg* tab = h->rg_tab.as<RaggedImg>();
  const float* pos = nullptr;
  TRY(pos_table(h, ib, &pos, st));
  // patch embedding: im2col + GEMM, rows land at token index 1 + patch (CLS row is filled by the next kernel); every image
  // owns L_max - 1 patch rows, the ones past its own grid are zero
  {
    const long long total = static_cast<long long>(NI) * (L - 1) * (Kp / 8);
    const int grid = static_cast<int>(std::min<long long>((total + 255) / 256, h->num_sms * 16));
    im2col_patch_kernel<<<grid, 256, 0, st>>>(images, u, tab, NI, L - 1, h->cfg.patch, Kp, par ? 1 : 0);
    CKL(h, "im2col_patch_kernel");
    GemmCall c = gemm_rows(h, RowOut::F32, u, h->w_patch.as<bf16>(), NI * (L - 1), d, Kp, nullptr, ACT_NONE, nullptr, x);
    c.p.rows_per_batch = L - 1;
    c.p.batch_stride = L;
    c.p.row_offset = 1;
    TRY(launch_gemm(h, c, st));
    const int gridr = static_cast<int>((Me + 7) / 8);
    auto kern = d == 768 ? cls_pos_lnpre_kernel<768> : cls_pos_lnpre_kernel<1024>;
    kern<<<gridr, 256, 0, st>>>(x, h->cls.as<float>(), pos, h->lnpre_g.as<float>(), h->lnpre_b.as<float>(), static_cast<int>(Me), L, tab);
    CKL(h, "cls_pos_lnpre_kernel");
  }
  const int rows = static_cast<int>(Me);
  const char* qkv = h->qkv.as<char>();
  SelfAttn attn{};
  attn.q = qkv; attn.k = qkv + d * qkv_eb; attn.v = qkv + 2 * d * qkv_eb; attn.out = ctx;
  attn.B = NI; attn.S = L; attn.H = H;
  attn.q_rs = attn.kv_rs = 3 * d; attn.q_bs = attn.kv_bs = static_cast<long long>(L) * 3 * d;
  attn.o_rs = d * ks; attn.o_bs = static_cast<long long>(L) * attn.o_rs;
  attn.seq_lens = img_lens(h, ib);
  for (int i = 0; i < h->cfg.enc_layers; ++i) {
    EncLayer& l = h->enc[i];
    TRY(launch_ln(h, ln_operand(h, x, l.ln1g.as<float>(), l.ln1b.as<float>(), 1e-5f, nullptr, hb, rows), d, st));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::QKV, hb, l.wqkv.as<bf16>(), rows, 3 * d, d, l.bqkv.as<float>(), ACT_NONE, nullptr, h->qkv.p), st));
    TRY(launch_self_attention(h, attn, par, st));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::F32, ctx, l.wo.as<bf16>(), rows, d, d, l.bo.as<float>(), ACT_NONE, x, x), st));
    TRY(launch_ln(h, ln_operand(h, x, l.ln2g.as<float>(), l.ln2b.as<float>(), 1e-5f, nullptr, hb, rows), d, st));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::OPERAND, hb, l.w1.as<bf16>(), rows, 4 * d, d, l.b1.as<float>(), ACT_QUICKGELU, nullptr, u), st));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::F32, u, l.w2.as<bf16>(), rows, d, 4 * d, l.b2.as<float>(), ACT_NONE, x, x), st));
  }
  // ln_post on all tokens (+ temporal embedding), re-ordered to [B, frames*L, d]
  {
    LnParams p = ln_operand(h, x, h->lnpost_g.as<float>(), h->lnpost_b.as<float>(), 1e-5f, feats_out, h->feats.as<bf16>(), rows);
    p.remap_B = B; p.remap_F = frames; p.remap_L = L;
    // temporal embeddings only for list inputs (reference layers/decoder.py:846-849; a bare tensor skips them)
    p.temb = (ib.list_input && h->cfg.num_frames_emb > 0) ? h->temb.as<float>() : nullptr;
    TRY(launch_ln(h, p, d, st));
  }
  h->cur_B = B;
  h->cur_frames = frames;
  h->cur_M = frames * L;
  h->cur_img = ib;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// hot path B: prefill (image rows of the decoder, computed once) + decode step
// ------------------------------------------------------------------------------------------------
// Split-K factors of the decode-step GEMMs: a handful of activation rows against [features, K] weights is latency
// bound, so K is spread over enough CTAs that each one has all of its weight tiles in flight at once.  Every split
// stores its own partial-sum buffer; the consumer (decode attention / LayerNorm) adds them in split order.
constexpr int kQkvSplits = 3, kOutProjSplits = 6, kFc2Splits = 8, kMaxProjSplits = 8;

// K/V caches: bf16, or fp32 in parity mode (void*: the element size is the engine's kvb())
static char* img_kv_ptr(gitb200_engine* h, int layer, int kv, long long elem_off = 0) {
  const long long per = static_cast<long long>(h->cur_B) * h->cur_M * h->D;
  return h->img_kv.as<char>() + ((static_cast<long long>(layer) * 2 + kv) * per + elem_off) * h->kvb();
}
static char* txt_kv_ptr(gitb200_engine* h, int layer, int kv, long long elem_off = 0) {
  const long long per = static_cast<long long>(h->cur_rows) * h->T_alloc * h->D;
  return h->txt_kv.as<char>() + ((static_cast<long long>(layer) * 2 + kv) * per + elem_off) * h->kvb();
}

// Workspaces of the decoder-layer pass for the image rows of the last encode and `text_rows` further rows (the larger of
// the two), and the image K/V cache.  Sized before a call's first launch: DevBuf::ensure frees the buffer it replaces.
static int decoder_buffers(gitb200_engine* h, long long text_rows) {
  const int D = h->D, F = h->F, nl = h->cfg.dec_layers;
  const long long img_rows = static_cast<long long>(h->cur_B) * h->cur_M;
  const long long rows = std::max(img_rows, text_rows);
  const int ks = h->ks();
  const long long kvb = static_cast<long long>(h->kvb());
  CK(h->pt.ensure(rows * D * 4));
  CK(h->pxd.ensure(rows * D * 4));
  CK(h->phd.ensure(rows * D * 2 * ks));
  CK(h->pq.ensure(rows * D * kvb));
  CK(h->pctx.ensure(rows * D * 2 * ks));
  CK(h->pu.ensure(rows * F * 2 * ks));
  CK(h->img_kv.ensure(static_cast<long long>(nl) * 2 * img_rows * D * kvb));
  return 0;
}

// The decoder layers (post-LN, erf-GELU) over `rows` rows whose input is in pxd (fp32) and phd (GEMM operand).  Layer j's
// k / v rows go to kv: [layer][k|v][rows][D] when kv_per_layer (the image K/V cache), else every layer overwrites the one
// [k|v][rows][D] pair there.  attend(j, q, k, v, ctx) launches layer j's attention.  last_qkv_only: the last layer stops
// after its QKV GEMM (only its k / v are read).  Buffers from decoder_buffers.
template <typename Attend>
static int decoder_layers(gitb200_engine* h, int rows, char* kv, bool kv_per_layer, bool last_qkv_only, Attend&& attend,
                          cudaStream_t st) {
  const int D = h->D, F = h->F, nl = h->cfg.dec_layers;
  const long long kv_bytes = static_cast<long long>(rows) * D * h->kvb();   // one k or v block
  float* t = h->pt.as<float>();
  float* xd = h->pxd.as<float>();
  bf16* hd = h->phd.as<bf16>();
  bf16* ctx = h->pctx.as<bf16>();
  bf16* u = h->pu.as<bf16>();
  auto ln = [&](const DevBuf& g, const DevBuf& b) {
    return launch_ln(h, ln_operand(h, t, g.as<float>(), b.as<float>(), 1e-12f, xd, hd, rows), D, st);
  };
  for (int j = 0; j < nl; ++j) {
    DecLayer& l = h->dec[j];
    char* k = kv + (kv_per_layer ? 2 * j * kv_bytes : 0);
    char* v = k + kv_bytes;
    GemmCall c = gemm_rows(h, RowOut::QKV, hd, l.wqkv.as<bf16>(), rows, 3 * D, D, l.bqkv.as<float>(), ACT_NONE, nullptr, h->pq.p);
    c.p.seg_n = D;
    c.p.out[1] = k; c.p.out[2] = v;
    c.p.ldo = D;
    TRY(launch_gemm(h, c, st));
    if (last_qkv_only && j + 1 == nl) break;
    TRY(attend(j, h->pq.p, k, v, ctx));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::F32, ctx, l.wo.as<bf16>(), rows, D, D, l.bo.as<float>(), ACT_NONE, xd, t), st));
    TRY(ln(l.lnag, l.lnab));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::OPERAND, hd, l.w1.as<bf16>(), rows, F, D, l.b1.as<float>(), ACT_GELU_ERF, nullptr, u), st));
    TRY(launch_gemm(h, gemm_rows(h, RowOut::F32, u, l.w2.as<bf16>(), rows, D, F, l.b2.as<float>(), ACT_NONE, xd, t), st));
    TRY(ln(l.lnog, l.lnob));
  }
  return 0;
}

// The image rows of the decoder, computed once per encode: visual projection, then the layers over the image rows only
// (they never attend to text, reference layers/decoder.py:119-120), whose k / v rows fill the image K/V cache.  Buffers
// from decoder_buffers.
static int image_rows(gitb200_engine* h, float* vproj_out, cudaStream_t st) {
  const int D = h->D, d = h->d, M = h->cur_M, B = h->cur_B;
  const int rows = B * M;
  float* t = h->pt.as<float>();
  float* xd = h->pxd.as<float>();
  // visual projection: Linear(dv -> 768) + LayerNorm(1e-5)
  TRY(launch_gemm(h, gemm_rows(h, RowOut::F32, h->feats.as<bf16>(), h->w_vp.as<bf16>(), rows, D, d, h->b_vp.as<float>(), ACT_NONE, nullptr, t), st));
  TRY(launch_ln(h, ln_operand(h, t, h->lnvp_g.as<float>(), h->lnvp_b.as<float>(), 1e-5f, xd, h->phd.as<bf16>(), rows), D, st));
  if (vproj_out) CK(cudaMemcpyAsync(vproj_out, xd, static_cast<size_t>(rows) * D * 4, cudaMemcpyDeviceToDevice, st));
  SelfAttn a{};
  a.B = B; a.S = M; a.H = h->cfg.dec_heads;
  a.q_rs = a.kv_rs = D; a.q_bs = a.kv_bs = static_cast<long long>(M) * D;
  a.o_rs = D * h->ks(); a.o_bs = static_cast<long long>(M) * a.o_rs;
  a.seq_lens = img_lens(h, h->cur_img);
  auto self_attention = [&](int, const void* q, const void* k, const void* v, bf16* ctx) {
    a.q = q; a.k = k; a.v = v; a.out = ctx;
    return launch_self_attention(h, a, h->parity, st);
  };
  return decoder_layers(h, rows, h->img_kv.as<char>(), true, true, self_attention, st);
}

// Sizes the decode step for B images x seqs sequences x beam rows; the image K/V cache holds the B images once.
static int prefill_impl(gitb200_engine* h, int B, int seqs, int beam, int T_alloc, float* vproj_out, cudaStream_t st) {
  if (B != h->cur_B || h->cur_M <= 0) return fail(h, "prefill: call encode with the same batch first");
  const int D = h->D, F = h->F, nl = h->cfg.dec_layers;
  const int R = B * seqs * beam;
  const int ks = h->ks();
  const long long kvb = static_cast<long long>(h->kvb());
  TRY(decoder_buffers(h, 0));
  {
    // decode_mega_kernel fetches the text cache in 16-position steps up to the caption's end and masks the positions past
    // it in the last step by giving them probability 0 -- which only works if what lies there is finite: a fresh allocation is zeroed once
    // (afterwards the buffer only ever holds K/V values or zeros of one element size).  A parity switch keeps the buffer
    // but changes the element size: fp32 K/V read as bf16 pairs hold Inf / NaN patterns, so the cache is zeroed again.
    const void* before = h->txt_kv.p;
    CK(h->txt_kv.ensure(static_cast<long long>(nl) * 2 * R * T_alloc * D * kvb));
    if (h->txt_kv.p != before || h->txt_kv_eb != h->kvb()) CK(cudaMemsetAsync(h->txt_kv.p, 0, h->txt_kv.cap, st));
    h->txt_kv_eb = h->kvb();
  }
  CK(h->src_row[0].ensure(static_cast<size_t>(R) * T_alloc * 4));
  CK(h->src_row[1].ensure(static_cast<size_t>(R) * T_alloc * 4));
  CK(h->xd_t.ensure(static_cast<size_t>(R) * D * 4));
  CK(h->hd_t.ensure(static_cast<size_t>(R) * D * 2 * ks));
  CK(h->qkv_t.ensure(static_cast<size_t>(kQkvSplits) * R * 3 * D * 4));   // split-K partial-sum buffers
  CK(h->ctx_t.ensure(static_cast<size_t>(R) * D * 2 * ks));
  CK(h->t_t.ensure(static_cast<size_t>(kMaxProjSplits) * R * D * 4));
  CK(h->u_t.ensure(static_cast<size_t>(R) * F * 2 * ks));
  CK(h->logits.ensure(static_cast<size_t>(R) * h->V * 4));
  CK(h->state.ensure(sizeof(StepState) + 64));            // + the megakernel's error word
  CK(h->y_t.ensure(static_cast<size_t>(R) * D * 4));
  CK(h->qb_t.ensure(static_cast<size_t>(R) * D * 2));
  CK(h->mega_bar.ensure(64));
  CK(h->next_token.ensure(static_cast<size_t>(R) * 8));
  CK(h->logprob_sum.ensure(static_cast<size_t>(R) * 4));
  h->cur_beam = beam;
  h->cur_seqs = seqs;
  h->cur_rows = R;
  h->T_alloc = T_alloc;
  return image_rows(h, vproj_out, st);
}

// One decode step for the cur_rows sequences: embed next_token at state->pos, 6 layers against the KV caches,
// optional LM head -> h->logits.  Every kernel reads the position / finished flag from device state so the
// same launch sequence (and CUDA graph) serves every step.  *tail (optional) receives the chain position of the last
// kernel launched, for the selection kernel that follows.
static int step_layers(gitb200_engine* h, cudaStream_t st, const long long* tokens, const int* src_row, bool lm_head,
                       ChainSync* tail = nullptr) {
  const int D = h->D, F = h->F, R = h->cur_rows, beam = h->cur_beam;
  const int nl = (h->debug_layers >= 0) ? std::min(h->debug_layers, h->cfg.dec_layers) : h->cfg.dec_layers;
  StepState* state = h->state.as<StepState>();
  const int* skip = &state->finished;
  const int ks = h->ks();
  const bool par = h->parity;
  float* xd = h->xd_t.as<float>();
  bf16* hd = h->hd_t.as<bf16>();
  float* qkv = h->qkv_t.as<float>();
  bf16* ctx = h->ctx_t.as<bf16>();
  float* t = h->t_t.as<float>();
  bf16* u = h->u_t.as<bf16>();
  float* logits = h->logits.as<float>();
  const bool pdl = h->use_pdl;
  // Ordering inside the step: flag chain (greedy; the beam bookkeeping kernels still use grid dependencies).
  const bool chain_on = pdl && beam == 1;
  ChainSync cs{};
  cs.counters = chain_on ? h->chain.as<unsigned int>() : nullptr;
  cs.idx = 0;
  cs.pred_ctas = 0;
  auto next_link = [&](unsigned int ctas_of_this_kernel) {  // call after each launch
    cs.idx += 1;
    cs.pred_ctas = ctas_of_this_kernel;
  };
  // chain head: launched WITHOUT the PDL attribute -> fully ordered after the previous step
  CK(launch_k(false, embed_ln_kernel<768>, dim3((R + 7) / 8), dim3(256), 0, st, tokens, 1LL, h->words_f32.as<float>(),
              h->positions.as<float>(), h->lnemb_g.as<float>(), h->lnemb_b.as<float>(), xd, hd, R, 0,
              static_cast<const StepState*>(state), h->V, par ? 1 : 0, cs));
  CKL(h, "embed_ln_kernel");
  next_link((R + 7) / 8);
  // split-K GEMMs write partial-sum buffers; bias / residual / LayerNorm live in the consumer kernel
  auto skinny = [&](GemmCall c) -> int {
    c.p.chain = cs;
    TRY(launch_gemm(h, c, st));
    next_link(static_cast<unsigned int>(h->last_gemm_grid));
    return 0;
  };
  auto ln_partials = [&](const float* parts, int n, int rows, const float* bias, const float* resid, const float* g,
                         const float* b, float* of32, bf16* obf16) {
    LnParams p = ln_params(parts, bias, resid, g, b, 1e-12f, of32, obf16, rows);
    p.n_partials = n;
    p.partial_stride = static_cast<long long>(rows) * D;
    p.split3 = par ? 1 : 0;
    return p;
  };
  DecodeAttn da{};
  da.n_partials = kQkvSplits;
  da.src_row = src_row; da.ctx = ctx;
  da.B = h->cur_B; da.seqs = h->cur_seqs; da.beam = beam; da.M = h->cur_M; da.T_alloc = h->T_alloc; da.D = D;
  da.state = state;
  da.img_lens = img_lens(h, h->cur_img);
  da.geom = h->attn_geom;
  da.pdl = pdl;
  auto ln = [&](LnParams p) -> int {
    p.skip_flag = skip; p.chain = cs;
    TRY(launch_ln(h, p, D, st, pdl));
    next_link((p.rows + 7) / 8);
    return 0;
  };
  for (int j = 0; j < nl; ++j) {
    DecLayer& l = h->dec[j];
    TRY(skinny(gemm_skinny(hd, D * ks, l.wqkv.as<bf16>(), D * ks, R, 3 * D, D * ks, nullptr, ACT_NONE, qkv, 3 * D, false, kQkvSplits, skip, pdl)));
    da.qkv = qkv; da.bqkv = l.bqkv.as<float>();
    da.img_k = img_kv_ptr(h, j, 0); da.img_v = img_kv_ptr(h, j, 1);
    da.txt_k = txt_kv_ptr(h, j, 0); da.txt_v = txt_kv_ptr(h, j, 1);
    da.chain = cs;
    unsigned int ctas = 0;
    TRY(launch_decode_attention(h, da, par, st, &ctas));
    next_link(ctas);
    TRY(skinny(gemm_skinny(ctx, D * ks, l.wo.as<bf16>(), D * ks, R, D, D * ks, nullptr, ACT_NONE, t, D, false, kOutProjSplits, skip, pdl)));
    TRY(ln(ln_partials(t, kOutProjSplits, R, l.bo.as<float>(), xd, l.lnag.as<float>(), l.lnab.as<float>(), xd, hd)));
    {
      GemmCall c1 = gemm_skinny(hd, D * ks, l.w1.as<bf16>(), D * ks, R, F, D * ks, l.b1.as<float>(), ACT_GELU_ERF, u, static_cast<long long>(F) * ks, true, 1, skip, pdl);
      c1.p.split3 = par ? 1 : 0;
      TRY(skinny(c1));
    }
    TRY(skinny(gemm_skinny(u, F * ks, l.w2.as<bf16>(), F * ks, R, D, F * ks, nullptr, ACT_NONE, t, D, false, kFc2Splits, skip, pdl)));
    TRY(ln(ln_partials(t, kFc2Splits, R, l.b2.as<float>(), xd, l.lnog.as<float>(), l.lnob.as<float>(), xd, hd)));
  }
  if (lm_head)
    TRY(skinny(gemm_skinny(hd, D * ks, h->words_bf16.as<bf16>(), D * ks, R, h->V, D * ks, h->out_bias.as<float>(), ACT_NONE, logits, h->V, false, 1, skip, pdl)));
  if (tail) *tail = cs;
  return 0;
}

// Decode-attention geometry of the last prefill (dec_attn_geometry) and the step chain's counters.
static int set_decode_geometry(gitb200_engine* h) {
  h->attn_geom = dec_attn_geometry(h->cur_M, h->cur_img.ragged ? h->cur_img.lens.data() : nullptr, h->cur_B, h->num_sms,
                                   h->cur_B * h->cur_seqs * h->cfg.dec_heads, h->cur_beam);
  CK(h->chain.ensure(256));
  CK(cudaMemset(h->chain.p, 0, 256));
  return 0;
}

#include "engine_api.inc"
#include "preproc_api.inc"
