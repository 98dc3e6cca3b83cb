/* gitb200 -- C ABI of the H100-native (sm_90a) GIT captioning engine (libgitb200.so).
 *
 * This is the drop-in boundary for the reference's hot path.  The reference is 100 % Python/PyTorch
 * (there is no FFI of its own), so the "binding a maintainer would add" is a ctypes stub
 * (INTEGRATION.md); each entry point names the reference function it replaces.  Paths are relative to
 * the reference's generativeimage2text/.
 *
 * Conventions
 *   - plain C types only; every `dev` pointer is a CUDA device pointer owned by the caller
 *     (e.g. `tensor.data_ptr()`), every `host` pointer is ordinary host memory;
 *   - all work is enqueued on the `stream` argument (a cudaStream_t passed as void*); entry points do
 *     not synchronise unless documented;
 *   - return 0 on success, non-zero on error; `gitb200_last_error` returns a message for the handle
 *     (or for the last failed `gitb200_create` when h == NULL); nothing throws across the ABI;
 *   - one engine per device and per thread of use (the reference model object is not re-entrant
 *     either: layers/decoder.py:991 stores per-call state on the module).
 */
#ifndef GITB200_H_
#define GITB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gitb200_engine gitb200_engine;

/* Model geometry.  Mirrors what `get_git_model(tokenizer, param)` hard-codes / reads from `param`
 * (model.py:9-61, 63-91): encoder = CLIP ViT-B/16 or ViT-L/14, decoder = 6 x 768 BERT-style layers. */
typedef struct gitb200_config {
  int32_t image_size;      /* param['test_crop_size'] (224)                          model.py:13  */
  int32_t patch;           /* 16 (CLIPViT_B_16) / 14 (CLIPViT_L_14)                   model.py:64-67 */
  int32_t enc_width;       /* 768 / 1024                                                           */
  int32_t enc_layers;      /* 12 / 24                                                              */
  int32_t enc_heads;       /* 12 / 16                                                              */
  int32_t dec_hidden;      /* 768                                                     model.py:17  */
  int32_t dec_layers;      /* 6                                                       model.py:18  */
  int32_t dec_heads;       /* 12                                                      model.py:19  */
  int32_t dec_ffn;         /* 3072                                                    model.py:20  */
  int32_t vocab;           /* 30522                                                   model.py:16  */
  int32_t max_positions;   /* 1024                                                    model.py:21  */
  int32_t num_frames_emb;  /* param['num_image_with_embedding'] or 0                  model.py:59  */
  int32_t sos_id;          /* tokenizer.cls_token_id                                  model.py:54  */
  int32_t eos_id;          /* tokenizer.sep_token_id                                  model.py:35,55 */
} gitb200_config;

/* Search configuration: the two decoders of model.py:27-40. */
enum { GITB200_SEARCH_GREEDY = 0, GITB200_SEARCH_BEAM = 1 };
typedef struct gitb200_search {
  int32_t mode;            /* GREEDY = AutoRegressiveBeamSearch(beam 1, per-node 1)  layers/decoder.py:208-440
                              BEAM   = GeneratorWithBeamSearch                        layers/decoder.py:1056-1341 */
  int32_t max_steps;       /* output length cap incl. start tokens (40 in BASELINE.json; 1024 stock) */
  int32_t beam_size;       /* 4 (BEAM: 2 .. 8)                                        model.py:38  */
  int32_t per_node_beam;   /* 2                                                       layers/decoder.py:1062 */
  float length_penalty;    /* 0.6                                                     model.py:39  */
} gitb200_search;

enum { GITB200_F32 = 0, GITB200_BF16 = 1, GITB200_I64 = 2 };

/* Replaces: get_git_model (construction)                                            model.py:9-61 */
int gitb200_create(const gitb200_config* cfg, int device, gitb200_engine** out);
void gitb200_destroy(gitb200_engine* h);
const char* gitb200_last_error(const gitb200_engine* h);
/* ABI version of the library (bumped on any signature change): 12 (gitb200_set_sequences_per_image); 11 added
 * gitb200_set_beam_sampling and gitb200_op_beam_sample; 10 added gitb200_op_gemm_ex, gitb200_op_layernorm_ex and gitb200_op_lse_combine; 9 added gitb200_score and gitb200_op_text_attention. */
int gitb200_abi_version(void);

/* Replaces: torch_common.load_state_dict -> module parameters           torch_common.py:93-145.
 * `ref_key` is the reference state-dict key (e.g. "image_encoder.conv1.weight"); `dev_ptr` an fp32
 * device tensor of `shape[ndim]`.  The engine repacks into its own layouts (bf16 GEMM operands,
 * fused QKV, padded patch kernel); the caller keeps ownership of the source and may free it after
 * gitb200_finalize_weights returns.  Unknown keys return an error; "image_encoder.proj" and
 * "textual.output.weight" (tied) are accepted and ignored. */
int gitb200_set_weight(gitb200_engine* h, const char* ref_key, const void* dev_ptr, const int64_t* shape,
                       int ndim, int dtype, void* stream);
/* Checks that every tensor of the geometry has been provided. Synchronises the stream. */
int gitb200_finalize_weights(gitb200_engine* h, void* stream);
/* Several engines of one geometry on one device (one per batch in flight, see gitb200_generate_async) need only one
 * copy of the parameters: `h` borrows the finalized weight buffers of `src` (which must outlive it) instead of taking
 * its own gitb200_set_weight calls -- the module-level equivalent is calling one nn.Module from several threads.
 * Keeps the decoder weights of all in-flight batches on the same L2 lines. */
int gitb200_share_weights(gitb200_engine* h, gitb200_engine* src);

/* Replaces: CaptioningModel.forward_one image branch = VisualTransformer.forward per frame
 * (+ img_temperal_embedding, token-axis concat)      layers/decoder.py:846-857, layers/CLIP/model.py:240-268.
 * images_dev: fp32 [frames][B,3,H,W] contiguous (frames >= 1; frame f at offset f*B*3*H*W; H = W = image_size unless
 * gitb200_set_input_size says otherwise), or B images of their own sizes back to back (gitb200_set_image_sizes).
 * feats_out_dev: fp32 [B, frames*L, enc_width] or NULL (kept internally for gitb200_prefill); [B, L_max, enc_width] for
 * images of their own sizes (image b's first L_b rows are its features, the rest finite padding). */
int gitb200_encode(gitb200_engine* h, const float* images_dev, int batch, int frames, float* feats_out_dev,
                   void* stream);

/* Input size of the following gitb200_encode / gitb200_generate* calls when it differs from image_size x image_size
 * (MinMaxResizeForTest inputs, inference.py:29-64): the patch grid becomes (height / patch) x (width / patch) and the
 * positional embedding is re-sampled to it on the device, bicubic, as VisualTransformer.forward does at run time
 *                                                                                  layers/CLIP/model.py:245-251.
 * All images of one call share the size (gitb200_set_image_sizes gives every image its own).  Sticky until changed;
 * gitb200_create starts at image_size x image_size. */
int gitb200_set_input_size(gitb200_engine* h, int height, int width);

/* Ragged batches: every image of the NEXT gitb200_encode / gitb200_generate* call has its own size (MinMaxResizeForTest
 * inputs of different aspect ratios in one call).  hw_host: int32 [n][2] = (height, width) of each image; that call's
 * images (images_dev or the host buffer) hold the n images back to back, fp32 [3, H_b, W_b] each; its batch must equal n
 * and frames must be 0 or 1.  Image b has L_b = (H_b / patch) * (W_b / patch) + 1 tokens in a slot of L_max = max L_b
 * rows: row b of the results is what a batch-1 call with that image alone returns.  The greedy decode steps of such a
 * call run on the kernel chain (use_mega does not apply).  gitb200_set_input_size is left as it was.
 * Inputs of the next call only (this one, gitb200_set_row_prefixes, gitb200_set_sampling, gitb200_set_beam_sampling,
 * gitb200_set_sequences_per_image): the next call that can use them takes them at entry, right after its in-flight check --
 * gitb200_encode and gitb200_score take the image sizes, a gitb200_generate* call takes all five -- and they are gone from the engine whether that call succeeds or fails. */
int gitb200_set_image_sizes(gitb200_engine* h, const int32_t* hw_host, int n);

/* Replaces: visual_projection + the image rows of BertEncoderAsDecoder, computed once (KV cache)
 *                                      layers/decoder.py:535, 92-174; layers/bert/modeling_bert.py:92-334.
 * Uses the features of the last gitb200_encode; beam 1 .. 8. vproj_out_dev: fp32 [B, M, 768] or NULL. */
int gitb200_prefill(gitb200_engine* h, int batch, int beam, float* vproj_out_dev, void* stream);

/* Replaces: CaptioningModel.decoding_step (one new token per row)       layers/decoder.py:1013-1054.
 * tokens_dev: int64 [rows] newest token of each row (rows = batch*beam), appended at text position
 * `pos` (rows and beam as the last gitb200_prefill: beam 1 .. 8); beam_idx_dev (int32 [rows], may be NULL) re-orders the text KV cache first
 * (layers/decoder.py:1231).  logits_out_dev: fp32 [rows, vocab] raw last-position logits. */
int gitb200_decode_step(gitb200_engine* h, const int64_t* tokens_dev, const int32_t* beam_idx_dev, int rows,
                        int pos, float* logits_out_dev, void* stream);

/* Replaces: CaptioningModel.forward / infer + decoder.search            layers/decoder.py:838-1011,
 * AutoRegressiveBeamSearch.search :224-440, GeneratorWithBeamSearch.search :1083-1290.
 * images_dev as gitb200_encode.  prefix_dev: int64 [P] start tokens (NULL/0 -> [sos]); reference asserts
 * batch == 1 with a prefix (layers/decoder.py:988).
 * forced_dev (int64 [B, max_steps] or NULL): teacher forcing for parity tests -- at every step the
 * engine records its own choice but feeds forced[:, t] as the next input (greedy only).
 * tokens_out_dev: int64 [B, max_steps] (incl. start tokens; EOS padded);  logprobs_out_dev: fp32 [B];
 * out_len_host: number of valid columns (greedy may stop early, layers/decoder.py:319), written after
 * an internal stream synchronise (the only sync of the call).
 * step_logits_dev: optional fp32 [steps, rows, vocab] dump of raw step logits (parity hook). */
int gitb200_generate(gitb200_engine* h, const float* images_dev, int batch, int frames, const int64_t* prefix_dev,
                     int prefix_len, const gitb200_search* search, const int64_t* forced_dev,
                     int64_t* tokens_out_dev, float* logprobs_out_dev, int32_t* out_len_host,
                     float* step_logits_dev, void* stream);

/* Same as gitb200_generate but with HOST buffers (pinned or pageable): copies the pixels host->device,
 * runs, copies tokens / logprobs back and synchronises.  This is the call a C host makes. */
int gitb200_generate_host(gitb200_engine* h, const float* images_host, int batch, int frames,
                          const int64_t* prefix_host, int prefix_len, const gitb200_search* search,
                          int64_t* tokens_out_host, float* logprobs_out_host, int32_t* out_len_host, void* stream);

/* Asynchronous form of the two calls above (same arguments minus out_len_host): everything is enqueued on `stream`
 * and the call returns; gitb200_generate_finish synchronises that stream and reports the loop length.  One call may
 * be in flight per engine; a host that keeps two engines (two streams) busy overlaps the encoder of batch i+1 with
 * the latency-bound decode loop of batch i (bench.py "pipeline": 2). Output buffers must stay valid until finish. */
int gitb200_generate_async(gitb200_engine* h, const float* images_dev, int batch, int frames, const int64_t* prefix_dev,
                           int prefix_len, const gitb200_search* search, const int64_t* forced_dev,
                           int64_t* tokens_out_dev, float* logprobs_out_dev, float* step_logits_dev, void* stream);
int gitb200_generate_host_async(gitb200_engine* h, const float* images_host, int batch, int frames,
                                const int64_t* prefix_host, int prefix_len, const gitb200_search* search,
                                int64_t* tokens_out_host, float* logprobs_out_host, void* stream);
int gitb200_generate_finish(gitb200_engine* h, int32_t* out_len_host);

/* Replaces: the training branch of CaptioningModel.forward_one_ce with dropout off  layers/decoder.py:916-972, i.e.
 * TransformerDecoderTextualHead.forward over given captions :521-600 and SmoothLabelCrossEntropyLoss :620-671 (eps 0.1,
 * padding id 0 ignored).  Scores N captions of T positions against the images in ONE teacher-forced pass.
 * images_dev, batch, frames as gitb200_generate (gitb200_set_input_size, and gitb200_set_image_sizes for the next call,
 * apply).  tokens_dev int64 [N, T]: CLS .. SEP rows padded with 0, ids in [0, vocab) (not checked here; out-of-range ids
 * are clamped).  need_predict_dev int64 [N, T] of 0 / 1 (the data layout of train.py:38-61).  image_index_dev int32 [N] in
 * [0, batch): the image of each caption, or NULL when N == batch (caption n, image n); captions of one image share its
 * encoder pass and image K/V.  2 <= T <= max_positions.
 * token_logprob_out_dev fp32 [N, T - 1]: log_softmax(logits[n, t])[tokens[n, t + 1]] for every t.
 * loss_out_dev fp32 [1] or NULL: the mean smoothed loss over the positions with need_predict[n, t + 1] == 1 and
 * tokens[n, t + 1] != 0 (NaN when there are none; the reference asserts).  Enqueued on `stream` without a host sync. */
int gitb200_score(gitb200_engine* h, const float* images_dev, int batch, int frames, const int64_t* tokens_dev,
                  const int64_t* need_predict_dev, const int32_t* image_index_dev, int n_captions, int positions,
                  float* token_logprob_out_dev, float* loss_out_dev, void* stream);

/* Measurement hook (bench.py's roofline): device time, by CUDA events on the engine's stream, of the decode loop of the
 * last generate on this engine -- first step launch to last -- with the number of step launches in it and whether each
 * was the single decode_mega_kernel launch.  Waits for that loop to finish.  No reference counterpart. */
int gitb200_last_decode_ms(gitb200_engine* h, float* ms_out, int32_t* steps_out, int32_t* one_kernel_out);

/* Per-row prefixes for the NEXT generate call, which takes them as gitb200_set_image_sizes describes (question batches;
 * the reference allows one prefix and batch 1 only, layers/decoder.py:985-1006): prefix_dev int64 [rows, stride],
 * lens_dev int32 [rows] (1 <= len <= stride, len < max_steps; tokens past a row's length are ignored).  rows must equal
 * that call's batch; pass prefix_len = 0 to it.  Every row is generated exactly as a batch-1 call with its own prefix
 * would be; tokens_out rows hold prefix + generated tokens.  The buffers must stay valid until the call has finished. */
int gitb200_set_row_prefixes(gitb200_engine* h, const int64_t* prefix_dev, int rows, int stride, const int32_t* lens_dev);

/* Replaces: TrieAutoRegressiveBeamSearch.search + TokenTrie                            trie_decoder.py:27-258
 * (the vocabulary-constrained greedy decoder model.py:42-48 keeps commented out next to the default one).  The trie is
 * passed in CSR form from HOST memory: node n's outgoing edges are [child_begin[n], child_begin[n + 1]), edge e accepts
 * token child_token[e] and leads to node child_node[e]; node 0 is the root.  While a trie is set, GREEDY generate calls
 * raise the log-probs of the allowed next tokens by (max logit - min logit + 1) before the top-1 (:61-62, :141-142),
 * move the cursor (:70, :153) and accumulate the raised value (:163).  Every row of the batch owns a cursor (the
 * reference has one and constrains row 0 only: it is a batch-1 decoder).  Sticky; n_nodes = 0 removes the trie. */
int gitb200_set_trie(gitb200_engine* h, const int32_t* child_begin_host, const int32_t* child_token_host,
                     const int32_t* child_node_host, int n_nodes, int n_edges);

/* Replaces: the do_sample branches of AutoRegressiveBeamSearch.search            layers/decoder.py:260-272, 364-375
 * for the NEXT generate call, which must be greedy and takes them as gitb200_set_image_sizes describes: row r draws its
 * token at caption length t from softmax(logits / temperature) by an inverse-CDF lookup in index order with
 * uniforms_dev[t * rows + r] (fp32 [steps >= max_steps, rows == batch], device; torch.multinomial's random stream cannot
 * be reproduced, the distribution is the same).  Log-probs as the reference computes them: tempered log-softmax at a
 * row's first decision, un-tempered afterwards.  The buffer must stay valid until the call has finished. */
int gitb200_set_sampling(gitb200_engine* h, const float* uniforms_dev, int steps, int rows, float temperature);

/* Replaces: the do_sample branch of GeneratorWithBeamSearch.search                layers/decoder.py:1138-1166, 1343-1375
 * for the NEXT generate call, which must be a beam search (per_node_beam 2) and takes them as gitb200_set_image_sizes
 * describes.  Every step, row r (of rows == batch * beam_size) filters scores = logits / temperature by top_k (<= 0: off;
 * k = min(max(top_k, 2), V), ties at the k-th value kept) and top_p (0 or >= 1: off; sorted by value desc, index asc, the
 * positions up to the first whose cumulative softmax exceeds top_p are kept, and never fewer than three), then draws two
 * tokens without replacement from softmax(filtered), each by an inverse-CDF lookup in index order with
 * uniforms_dev[(t * rows + r) * 2 + d] at caption length t (fp32 [steps >= max_steps, rows, 2], device).  A candidate's
 * score is log_softmax(filtered)[token] + the row's beam score; the candidates of an image stay in (beam, draw) order.
 * A row with fewer than two tokens of non-zero probability stops the search, and gitb200_generate_finish (or the
 * synchronous generate call) fails naming its step and row.  The buffer must stay valid until the call has finished. */
int gitb200_set_beam_sampling(gitb200_engine* h, const float* uniforms_dev, int steps, int rows, float temperature,
                              int top_k, float top_p);

/* Replaces: the num_return_sequences argument of the three searches   layers/decoder.py:232-237, 1093-1096,
 * trie_decoder.py:51-55, for the NEXT generate call, which takes it as gitb200_set_image_sizes describes: that call runs
 * n >= 1 sequences for each of its `batch` images, in image-major order (sequence b * n + i belongs to image b), each
 * searching independently.  Every image is encoded and its K/V cached once; its n sequences read that one copy.  The
 * call's other per-row arguments count sequences, not images: the rows of gitb200_set_row_prefixes and of the sampling
 * uniforms (batch * n, or batch * n * beam_size for beam sampling), forced_dev [batch * n, max_steps], tokens_out
 * [batch * n, max_steps], logprobs_out [batch * n] and step_logits [steps, batch * n (* beam_size), vocab].  Each
 * sequence's result is bit for bit what the call with every image repeated n times returns (greedy steps without the
 * one-kernel step: a call with n > 1 runs on the kernel chain).  n = 1 is the call without it. */
int gitb200_set_sequences_per_image(gitb200_engine* h, int n);

/* Number of kernels the engine launched since creation (bench.py's gpu_launches). */
int64_t gitb200_launch_count(const gitb200_engine* h);
/* Engine switches (defaults in parentheses): use_graph (1) CUDA-graph replay of the decode step, use_pdl (1) programmatic
 * dependent launch inside the step (greedy steps on the kernel chain are then ordered by a flag chain),
 * use_mega (1) greedy decode steps of <= 64 sequences as one persistent, cooperatively launched kernel,
 * parity (0) fp32-grade verification mode: every GEMM operand is a (hi, lo) bf16 pair and each product is computed as
 * a_hi w_hi + a_lo w_hi + a_hi w_lo by the same wgmma kernel (three K-segments side by side), attention / K/V caches /
 * q, k, v in fp32 -- set it BEFORE gitb200_set_weight (switching it forgets the uploaded weights). */
int gitb200_set_option(gitb200_engine* h, const char* name, int64_t value);

/* ---- single-kernel entry points (unit tests, micro-benchmarks, ncu) -------------------------------- */
/* C = A[M,K] * W[N,K]^T (+bias) (+act: 0 none, 1 QuickGELU, 2 erf-GELU) (+resid fp32 [M,N]).
 * a_dev, w_dev bf16; out fp32 or bf16.  transposed != 0 runs the swap-AB skinny path used by the decode
 * step (a_dev = activations [M<=256,K], w_dev = weight [N,K], out[M,N]); k_splits > 1 (transposed only, raw
 * fp32 out, no bias / act): every split stores its own partial sums, which are added in split order -- bit-reproducible. bn: tile width override (0 = heuristic). */
int gitb200_op_gemm(const void* a_dev, const void* w_dev, const float* bias_dev, const float* resid_dev,
                    void* out_dev, int M, int N, int K, int act, int out_bf16, int transposed, int k_splits,
                    int bn, void* stream);
/* y = LayerNorm(x (+bias) (+resid)) * gamma + beta over the last dim D (768 or 1024), fp32 in,
 * fp32 and/or bf16 out (either may be NULL). */
int gitb200_op_layernorm(const float* x_dev, const float* bias_dev, const float* resid_dev, const float* gamma_dev,
                         const float* beta_dev, float eps, float* out_f32_dev, void* out_bf16_dev, int rows, int D,
                         void* stream);
/* One launch of gemm_bf16_wgmma with everything its launcher takes, in the kernel's own operand terms:
 *   C[m][n] = sum_k a[m][k] * b[n][k], a [M, K] (128-row tiles) and b [N, K] (bn-row tiles) bf16, row pitches lda / ldb.
 * transposed == 0: out[seg][row_map(m)][n % seg_n] = C (+bias[n]) (+act) (+resid[m][n]), seg = n / seg_n (up to three column
 *   segments with their own base pointers and the one row pitch ldo), row_map(m) = (m / rows_per_batch) * batch_stride +
 *   m % rows_per_batch + row_offset (rows_per_batch <= 0: identity); resid fp32, pitch ld_resid, may be out[0] (in place).
 *   split3: bf16 rows [hi | lo | hi] of 3 * N columns.  lse_target != NULL: the LM-head statistics epilogue, out[0] =
 *   float4 (max, sum exp(x - max), sum x, x[target]) per (row, half tile) at [m * ldo + 2 * (n / 256) + half], bias required.
 * transposed != 0 (swap-AB: a = weight [features, K], b = activations [rows, K]): out[0][n][m] = C (+bias[m]) (+act).
 *   k_splits > 1: split s leaves its raw fp32 partial sums at out[0] + s * split_stride (nothing adds them up);
 *   *k_splits_out (may be NULL) receives the number of splits that ran (empty ones are dropped: 8 over 12 k-blocks -> 6).
 * act: 0 none, 1 QuickGELU (tanh.approx), 2 erf-GELU, 3 QuickGELU (expf).  bn: tile width, 0 = heuristic.
 * skip: NULL or a device int; non-zero -> the launch stores nothing. */
typedef struct gitb200_gemm_desc {
  const void* a;
  const void* b;
  const float* bias;
  const float* resid;
  void* out[3];
  const int32_t* lse_target;
  const int32_t* skip;
  int64_t lda, ldb, ld_resid, ldo, batch_stride, split_stride;
  int32_t M, N, K;
  int32_t act, out_bf16, split3, transposed, k_splits, bn;
  int32_t seg_n, rows_per_batch, row_offset;
} gitb200_gemm_desc;
int gitb200_op_gemm_ex(const gitb200_gemm_desc* desc, int* k_splits_out, void* stream);
/* gitb200_op_layernorm with the rest of layernorm_kernel's inputs: x_dev is the first of n_partials (>= 1) split-K
 * partial buffers, partial_stride elements apart, added in split order; split3: out_bf16 rows [hi | lo | hi] (3 * D);
 * temb_dev [F, D] or NULL with remap_B / F / L (remap_F == 0: none): input row (f * B + b) * L + l -> output row
 * (b * F + f) * L + l, temb[f] added after the normalisation; skip_flag_dev: NULL or a device int, non-zero -> no-op;
 * pre != 0: the <768, PRE = true> instantiation of the decode chain (D = 768 only). */
int gitb200_op_layernorm_ex(const float* x_dev, int n_partials, long long partial_stride, const float* bias_dev,
                            const float* resid_dev, const float* gamma_dev, const float* beta_dev, float eps,
                            float* out_f32_dev, void* out_bf16_dev, int rows, int D, int split3, const float* temb_dev,
                            int remap_B, int remap_F, int remap_L, const int32_t* skip_flag_dev, int pre, void* stream);
/* lse_combine_kernel, then loss_mean_kernel when loss_dev != NULL, on caller-supplied LM-head partials: parts_dev float4
 * [rows, n_parts] (max, sum exp, sum x, x[target]), rows = captions * T, targets_dev int32 [rows], need_predict_dev int64
 * [rows] -> logprob_dev [captions, T - 1], row_loss_dev fp32 [rows], row_valid_dev int32 [rows], loss_dev fp32 [1]
 * (NaN when no row is valid). */
int gitb200_op_lse_combine(const void* parts_dev, int n_parts, int rows, int T, int V, const int32_t* targets_dev,
                           const int64_t* need_predict_dev, float eps, float* logprob_dev, float* row_loss_dev,
                           int32_t* row_valid_dev, float* loss_dev, void* stream);
/* Non-causal multi-head attention over packed bf16 rows: q/k/v [B, S, H*64] with the given row strides (elements);
 * batches are stored back to back (q_batch_stride = S * q_row_stride, kv_batch_stride = S * kv_row_stride; other batch
 * strides are refused); out bf16 [B, S, H*64] with its own row and batch strides. softmax(q k^T / 8) v. */
int gitb200_op_attention(const void* q_dev, const void* k_dev, const void* v_dev, void* out_dev, int B, int S, int H,
                         long long q_row_stride, long long kv_row_stride, long long q_batch_stride,
                         long long kv_batch_stride, long long out_row_stride, long long out_batch_stride,
                         void* stream);
/* gitb200_op_attention plus per-batch lengths and parity mode.  seq_lens_host: NULL or B lengths in 1..S (ragged: batch b
 * is computed as a call with S = seq_lens[b] and its rows past that length are
 * zeros).  fp32 != 0: attn_f32_kernel on fp32 q/k/v; output rows are 3*H*64 bf16 [hi | lo | hi], out_row_stride is
 * ignored. */
int gitb200_op_attention_ex(const void* q_dev, const void* k_dev, const void* v_dev, void* out_dev, int B, int S, int H,
                            long long q_row_stride, long long kv_row_stride, long long q_batch_stride,
                            long long kv_batch_stride, long long out_row_stride, long long out_batch_stride,
                            const int32_t* seq_lens_host, int fp32, void* stream);
/* One layer's decode-step attention as the kernel chain runs it: decode_attn_kernel<beam, img_lens != NULL>,
 * or decode_attn_f32_kernel when fp32 != 0.
 * qkv_dev: n_partials (1..4) fp32 split-K partial buffers [B*beam, 3*D], B*beam*3*D elements apart; bqkv_dev fp32 [3*D].
 * img_k/v_dev [B, M, D] and txt_k/v_dev [B*beam, T_alloc, D]: bf16, or fp32 when fp32 != 0.  Position pos of every text
 * row is written (k / v of this step + bias).  src_row_dev int32 [B*beam, T_alloc] or NULL (identity).
 * img_lens_host: NULL (uniform) or B key counts in 1..M (ragged).  ctx_dev: bf16 [B*beam, D], or split rows [B*beam, 3*D]
 * when fp32 != 0.  grid: CTAs of decode_attn_kernel in 0..B*D/64, 0 = what the engine would launch (ignored when
 * fp32 != 0).  beam 1..4, D % 64 == 0. */
int gitb200_op_decode_attention(const float* qkv_dev, int n_partials, const float* bqkv_dev, const void* img_k_dev,
                                const void* img_v_dev, void* txt_k_dev, void* txt_v_dev, const int32_t* src_row_dev,
                                void* ctx_dev, int B, int beam, int M, const int32_t* img_lens_host, int T_alloc, int pos,
                                int D, int fp32, int grid, void* stream);

/* One step of sampled beam search's per-row selection (beam_sample_kernel, see gitb200_set_beam_sampling) on given logits:
 * logits_dev fp32 [rows, V] (V <= 49152), beam_scores_dev fp32 [rows], uniforms_dev fp32 [rows, 2].  Writes the two
 * candidates of each row, cand_val_out_dev fp32 [rows, 2] (log_softmax(filtered)[token] + beam score) and
 * cand_idx_out_dev int32 [rows, 2], and kept_out_dev int32 [rows] = the size of the row's kept set.  Synchronises the
 * stream; fails when a row has fewer than two tokens of non-zero probability. */
int gitb200_op_beam_sample(const float* logits_dev, int rows, int V, const float* beam_scores_dev, const float* uniforms_dev,
                           float temperature, int top_k, float top_p, float* cand_val_out_dev, int32_t* cand_idx_out_dev,
                           int32_t* kept_out_dev, void* stream);

/* Caption scoring's attention (text_attn_wgmma_kernel, or text_attn_f32_kernel when fp32 != 0): text row t of caption n
 * attends to the image keys of image image_index[n] and to text keys 0 .. t of caption n; softmax(q k^T / 8) v per head.
 * q / txt_k / txt_v [N * T, H * 64] rows (caption n at rows n * T ..), img_k / img_v [B * M, H * 64] (image b at rows b * M ..):
 * bf16, or fp32 when fp32 != 0.  img_lens_host: NULL (every image has M keys) or B key counts in 1..M.  image_index_host:
 * NULL (N == B, caption n uses image n) or N indices in 0..B-1.  out_dev bf16 [N * T, H * 64], or split rows
 * [N * T, 3 * H * 64] ([hi | lo | hi]) when fp32 != 0. */
int gitb200_op_text_attention(const void* q_dev, const void* txt_k_dev, const void* txt_v_dev, const void* img_k_dev,
                              const void* img_v_dev, void* out_dev, int N, int T, int B, int M, const int32_t* img_lens_host,
                              const int32_t* image_index_host, int H, int fp32, void* stream);

/* ---- test-time image transform on the GPU ----------------------------------------------------------------
 * Replaces: get_image_transform(param)(pil_image)                                       inference.py:111-132
 *   = torchvision Resize(crop, BICUBIC) -> CenterCrop(crop) -> ToTensor -> Normalize(CLIP mean/std), or, with
 *   param['test_respect_ratio_max'], MinMaxResizeForTest                                inference.py:29-64
 * applied to DECODED images (uint8 RGB, HWC -- what PIL's Image.convert('RGB') holds).  Results are bit-identical to
 * the PIL / torchvision pipeline (Pillow's two-pass fixed-point bicubic with antialiasing, libImaging/Resample.c).
 * The caller computes the size rule (it is host arithmetic on two integers, see generativeimage2text_b200/inference.py)
 * and passes one descriptor per image; images of one call may all differ in size. */
typedef struct gitb200_preproc gitb200_preproc;
typedef struct gitb200_image_desc {
  int64_t src_offset;      /* bytes: first pixel of this image inside the packed source buffer                    */
  int32_t src_h, src_w;    /* decoded size                                                                        */
  int32_t resize_h, resize_w; /* size after the bicubic resize (== src: that axis is not resampled)               */
  int32_t crop_top, crop_left; /* window of the resized image that is produced (CenterCrop; 0,0 + full size = none) */
  int32_t out_h, out_w;
  int64_t dst_offset;      /* fp32 elements: the image lands as [3, out_h, out_w] at out_dev + dst_offset          */
} gitb200_image_desc;

int gitb200_preproc_create(int device, gitb200_preproc** out);
void gitb200_preproc_destroy(gitb200_preproc* p);
const char* gitb200_preproc_last_error(const gitb200_preproc* p);
int64_t gitb200_preproc_launch_count(const gitb200_preproc* p);
/* Reserved for future switches (none at present: every call returns non-zero). */
int gitb200_preproc_set_option(gitb200_preproc* p, const char* name, int64_t value);
/* src: packed uint8 RGB images, on the device (src_on_host == 0) or in host memory (pinned or pageable; copied to the
 * device on `stream` first).  mean3 / std3: host float[3].  Work is enqueued on `stream`; a second call on the same
 * handle first waits (on the host) for the previous call's kernels, so use one handle per stream to overlap calls. */
int gitb200_preproc_run(gitb200_preproc* p, const uint8_t* src, int64_t src_bytes, int src_on_host,
                        const gitb200_image_desc* descs_host, int n, const float* mean3, const float* std3,
                        float* out_dev, int64_t out_elems, void* stream);
/* Host-only helper (no GPU needed): the fixed-point weight table of one axis, i.e. Resample.c precompute_coeffs +
 * normalize_coeffs_8bpc for BICUBIC: bounds_out int32 [out_size][2] (first tap, taps), kk_out int32 [out_size][kk_cap]. */
int gitb200_preproc_coeffs(int in_size, int out_size, int32_t* ksize_out, int32_t* bounds_out, int32_t* kk_out, int kk_cap);

/* Debug: copies one decode-step work buffer of the engine ("x", "y" fp32 [rows,768]; "hb", "ctx", "qb" bf16 [rows,768];
 * "ub" bf16 [rows,3072]) or cache ("img_kv": the image K/V [layer][k|v][image][token][768] of the last prefill, batch x
 * tokens rows; "txt_kv": the text K/V [layer][k|v][row][T_alloc][768], T_alloc = bytes / (layers * 2 * rows * 768 * element
 * size); both bf16, fp32 in parity mode) to host memory after a device synchronise.  The last encode (test hooks):
 *   "enc_x"       fp32 [batch*frames*L][width]: the encoder's residual stream after its last block, before ln_post, images
 *                 in the encoder's order f*batch + b (L: tokens per image; a ragged batch's slot length L_max);
 *   "enc_feats"   the features as the prefill's GEMM operand: bf16 [batch*frames*L][width], or [hi | lo | hi] rows of
 *                 3*width in parity mode (hi = bf16(f), lo = bf16(f - hi)); rows in the output order b*frames*L + f*L + l;
 *   "pos_interp"  fp32 [rows][width]: the positional table the encode made, one block of 1 + gh*gw rows per distinct patch
 *                 grid of its images in order of first appearance (the model's own grid copied, any other re-sampled);
 *                 0 bytes when every image had the model's grid and the encode used the stored table.
 * Beam search bookkeeping, current side of each ping-pong:
 *   "src_row"     int32 [rows][T_alloc]: the text-K/V indirection table the next beam step reads (position j of logical
 *                 row r is held by physical row src_row[r][j]); after a beam generate or the raw decode_step API;
 *   "beam_ids"    int64 [rows][max_steps]: the token history (input_ids) of each beam, after a beam generate;
 *   "beam_scores" fp32 [rows]: the running beam scores, after a beam generate;
 *   "beam_hyp"    [4][batch] 4-byte words, after a beam generate: done (int32), hyp_len (int32, 0 = no hypothesis),
 *                 hyp_score (fp32, length-normalised), worst_score (fp32).
 *   "beam_cand"   [2][rows][C] 4-byte words, after a beam generate: the last step's per-row candidate list, scores
 *                 (fp32: log-softmax + beam score) then token ids (int32); C = 8 for beam sizes 2 .. 4 and 16 for 5 .. 8;
 *                 the first 2 * beam entries of a row are valid.
 * Returns bytes copied or -1. */
long long gitb200_debug_read(gitb200_engine* h, const char* name, void* out_host, long long max_bytes);
/* Debug aid: in-situ timeline of the decode-step kernels. enable != 0 arms it; enable == 0 copies up to
 * max_entries (globaltimer ns, kernel id) pairs to out_host, disarms, and returns the number of entries. */
int gitb200_debug_timeline(int enable, unsigned long long* out_host, int max_entries);

#ifdef __cplusplus
}
#endif
#endif /* GITB200_H_ */
