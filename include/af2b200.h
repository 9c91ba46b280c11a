/* libaf2b200.so — C ABI of the H100-native Evoformer trunk hot path.
 *
 * The reference (lucidrains/alphafold2 @ 931466e) is 100 % Python and has no FFI: its boundary for this
 * path is the nn.Module API (alphafold2_pytorch/alphafold2.py).  Each entry point below therefore replaces
 * the forward() of one reference module and is bound from Python with ctypes (alphafold2_b200/_lib.py);
 * INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer on the current CUDA device (sm_90a only); nothing is allocated
 *     or retained by the library: outputs and workspace are caller-owned;
 *   - activations x / m are fp32, channel-last, contiguous; weights are packed bf16 (see packing.py) with
 *     fp32 biases / LayerNorm affine parameters; masks are 1-byte bools (torch.bool);
 *   - residual adds are performed in place on the fp32 stream (x <- x + f(x));
 *   - launches are asynchronous on `stream` (a cudaStream_t); CUDA-graph capturable (no sync, no malloc);
 *   - return 0 on success, negative on error (af2_last_error() holds the message). There is NO CPU fallback.
 */
#ifndef AF2B200_H
#define AF2B200_H
#ifdef __cplusplus
extern "C" {
#endif

typedef void* af2_stream_t; /* cudaStream_t */

#define AF2_OK 0
#define AF2_ERR_BAD_ARG (-1)
#define AF2_ERR_CUDA (-2)
#define AF2_ERR_UNSUPPORTED_DEVICE (-3)
#define AF2_ERR_WORKSPACE (-4)

const char* af2_last_error(void);
int af2_abi_version(void);
/* 0 if the current device is compute capability 9.0 (H100, sm_90a), AF2_ERR_UNSUPPORTED_DEVICE otherwise */
int af2_check_device(void);

/* Kernel launches issued by this library since load (bench.py's gpu_launches). */
unsigned long long af2_launch_count(void);
/* Optional CUDA-event profiling per kernel class (0 linear GEMM, 1 per-channel GEMM, 2 attention, 3 LayerNorm,
 * 4 channel->token, 5 misc): enable(1) clears the records; read() synchronises and sums elapsed ms, algorithmic
 * FLOPs and bytes of the recorded launches of one class and returns their count. */
void af2_profile_enable(int on);
long long af2_profile_read(int cls, double* ms, double* flops, double* bytes);

/* ---------------- FeedForward: alphafold2.py:74-94 (+ residual of :439 / :444) -----------------------
 * x <- x + W2 (a * gelu_erf(g)) + b2,  [a|g] = W1 LN(x) + b1.
 * w1 is packed per column tile of `bn` accumulator columns as [bn/2 value rows | bn/2 gate rows]
 * (zero rows pad the last tile); b1 is permuted the same way. */
typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* FeedForward.norm          [d]            */
  const void* w1; const float* b1;                    /* FeedForward.net.0         packed [n1p, d]  */
  const void* w2; const float* b2;                    /* FeedForward.net.3         [d, hid] , [d]   */
  int bn;                                             /* column tile used for the w1 packing        */
} af2_ff_weights;
int af2_feed_forward(const af2_ff_weights* w, float* x, long long tokens, int d, int hidden,
                     void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_feed_forward_workspace(long long tokens, int d, int hidden);

/* ---------------- AxialAttention: alphafold2.py:192-255 driving Attention :98-190 (+ residual) --------
 * x [B, h, w, d] <- x + to_out( softmax(q k^T + bias, mask) v * sigmoid(gating) ).
 * row_attn = 1: attend along w for every (b, h) row; 0: along h for every (b, w) column.
 * edges: RAW fp32 pair tensor [B, n, n, d] (n = attended length) or NULL; bias = edges . w_edge^T,
 * identical for every folded row/column, orientation [head, query, key] (quirks Q4/Q5). */
typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* AxialAttention.norm                        */
  const void* w_qkv;                                  /* [3I, d]: to_q * dim_head^-0.5 | to_kv      */
  const void* w_gate; const float* b_gate;            /* Attention.gating          [I, d], [I]      */
  const void* w_out; const float* b_out;              /* Attention.to_out          [d, I], [d]      */
  const float* w_edge;                                /* edges_to_attn_bias.0      [H, d] fp32/NULL */
} af2_attn_weights;
int af2_axial_attention(const af2_attn_weights* w, float* x, const float* edges, const unsigned char* mask,
                        int B, int h, int wdim, int d, int heads, int dim_head, int row_attn,
                        void* workspace, long long workspace_bytes, af2_stream_t stream);
/* af2_axial_attention with flags: bit 0 = tied ("global") queries -- the queries are averaged over the folded batch before
 * the dot products (alphafold2.py:142-151; AxialAttention(global_query_attn=True), :250; used by the extra-MSA stack :518-527) */
int af2_axial_attention_ex(const af2_attn_weights* w, float* x, const float* edges, const unsigned char* mask, int B,
                           int h, int wdim, int d, int heads, int dim_head, int row_attn, int flags, void* workspace,
                           long long workspace_bytes, af2_stream_t stream);
long long af2_axial_attention_workspace(int B, int h, int wdim, int d, int heads, int dim_head, int row_attn);

/* ---------------- TriangleMultiplicativeModule: alphafold2.py:257-317 (+ residual :381-382) ----------
 * x [B, N, N, d] <- x + to_out( LN_c( mix(L, R) ) * sigmoid(out_gate) ),  hidden_dim == d.
 * outgoing (mix=0): O[i,j,c] = sum_k L[i,k,c] R[j,k,c];  ingoing (mix=1): O[i,j,c] = sum_k L[k,j,c] R[k,i,c].
 * w_left / w_right are packed per tile as [value rows | gate rows] like w1 above. */
typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* .norm                                      */
  const void* w_left; const float* b_left;            /* left_proj + left_gate, packed              */
  const void* w_right; const float* b_right;          /* right_proj + right_gate, packed            */
  const void* w_ogate; const float* b_ogate;          /* out_gate                  [d, d], [d]      */
  const float* on_gamma; const float* on_beta;        /* to_out_norm                                */
  const void* w_out; const float* b_out;              /* to_out                    [d, d], [d]      */
  int bn;
} af2_trimul_weights;
int af2_triangle_multiply(const af2_trimul_weights* w, float* x, const unsigned char* mask, int B, int N, int d,
                          int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_triangle_multiply_workspace(int B, int N, int d);

/* ---------------- OuterMean: alphafold2.py:321-351 (+ residual :379) ---------------------------------
 * x [B, N, N, d] <- x + proj_out( sum_s L[s,i,:] * R[s,j,:] / S  [/ (count_ij + eps) when masked] ).
 * Never materialises the (S, N, N, d) tensor of alphafold2.py:341. */
typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* .norm                                      */
  const void* w_lr; const float* b_lr;                /* [2d, d]: left_proj | right_proj, [2d]      */
  const void* w_out; const float* b_out;              /* proj_out                  [d, d], [d]      */
} af2_outer_weights;
int af2_outer_mean(const af2_outer_weights* w, float* x, const float* m, const unsigned char* msa_mask,
                   int B, int S, int N, int d, float eps, void* workspace, long long workspace_bytes,
                   af2_stream_t stream);
long long af2_outer_mean_workspace(int B, int S, int N, int d);

/* ---------------- stage-level entry points used by the axis-sharded (multi-GPU) schedule ---------------------
 * The reference has no multi-device path; these split the modules above at the points where the sharded
 * schedule (alphafold2_b200/parallel.py) must exchange operands over NCCL.  Batch size 1 per call.
 *   channel-major operand layout: bf16 [channels][chan_stride], token t of a [rows, inner] token grid at
 *   (t / inner) * align8(inner) + t % inner (pad columns zero). */
/* pair bias of a band of pair rows: out bf16 [H][rows][align8(n)] = <x[r, j, :], w_edge[h, :]> (w_edge as packed) */
int af2_pair_bias(const float* x_rows, const float* w_edge, void* bias_out, int rows, int n, int d, int heads,
                  af2_stream_t stream);
/* af2_axial_attention with a precomputed bias [B][H][n][align8(n)] (or NULL) instead of raw edges */
int af2_axial_attention_prebias(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask,
                                int B, int h, int wdim, int d, int heads, int dim_head, int row_attn, void* workspace,
                                long long workspace_bytes, af2_stream_t stream);
/* Tied-query ("global") column attention of a column shard x [h][wdim][d] (batch 1, bf16 mode) whose tied queries average
 * over ncols_total columns held by several ranks, in two calls on one workspace (af2_axial_attention_workspace(1, h, wdim, d,
 * heads, dim_head, 0)) that the caller leaves untouched between them:
 *   _begin: LayerNorm and the q|k|v and gate projections into the workspace, then qsum_out fp32 [h][heads * dim_head] = the sum
 *     of the bf16 queries over this call's wdim columns, added from 0 in column order;
 *   (the caller gathers every shard's qsum_out in column-shard order: parts [nparts][h][heads * dim_head])
 *   _end: q <- bf16((sum of the parts from 0 in part order) / ncols_total) in every local column, then the attention and
 *     to_out + residual into x.
 * Both take the same operands (bias_bf16 [H][h][align8(h)] or NULL, mask [h][wdim] or NULL); only _end reads them.  With
 * nparts = 1 and ncols_total = wdim the pair is bitwise af2_axial_attention_ex(flags = 1) with this bias.  AF2_ERR_BAD_ARG on
 * a null w, x, qsum_out / parts or workspace, h or wdim < 1, nparts < 1 or ncols_total < wdim. */
int af2_axial_attention_tied_begin(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask, int h,
                                   int wdim, int d, int heads, int dim_head, float* qsum_out, void* workspace,
                                   long long workspace_bytes, af2_stream_t stream);
int af2_axial_attention_tied_end(const af2_attn_weights* w, float* x, const void* bias_bf16, const unsigned char* mask, int h,
                                 int wdim, int d, int heads, int dim_head, const float* parts, int nparts, int ncols_total,
                                 void* workspace, long long workspace_bytes, af2_stream_t stream);
/* LN + left/right (masked, gated) -> channel-major Lc, Rc [d][chan_stride]; sigmoid(out_gate) -> gate [tokens, d] */
int af2_triangle_project(const af2_trimul_weights* w, const float* x, const unsigned char* mask, long long tokens,
                         int inner, int d, void* Lc, void* Rc, long long chan_stride, void* gate, void* workspace,
                         long long workspace_bytes, af2_stream_t stream);
long long af2_triangle_project_workspace(long long tokens, int d);
/* x [rows, cols, d] += to_out(LN_c(O) * gate);  Rg holds `pieces` gathered shards, piece_stride elements apart.
 *   outgoing: O[i][j] = sum_k L[i][k] R[j][k], L [c][rows][align8(K)], piece p = R rows j of shard p [c][cols/pieces][align8(K)]
 *   ingoing : O[i][j] = sum_k R[k][i] L[k][j], L [c][K][align8(cols)], piece p = R columns i of shard p [c][K][align8(rows/pieces)] */
int af2_triangle_contract(const af2_trimul_weights* w, float* x, const void* Lc, long long cs_l, const void* Rg,
                          long long cs_r, long long piece_stride, int pieces, const void* gate, int rows, int cols,
                          int K, int d, int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_triangle_contract_workspace(int rows, int cols, int d);
/* af2_triangle_contract of one L / R pair with explicit pitches ld_l / ld_r (elements, multiples of 8) and channel strides
 * cs_l / cs_r: the operands may be windows into larger channel-major tensors.  Workspace: af2_triangle_contract_workspace.
 *   outgoing: L [c][rows][ld_l] (k < K), R [c][cols][ld_r] (k < K)
 *   ingoing : L [c][K][ld_l] (j < cols), R [c][K][ld_r] (i < rows; e.g. the column window R[c][k][i0 .. i0 + rows)) */
int af2_triangle_contract_pitched(const af2_trimul_weights* w, float* x, const void* Lc, long long cs_l, long long ld_l,
                                  const void* Rc, long long cs_r, long long ld_r, const void* gate, int rows, int cols, int K,
                                  int d, int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream);
/* LN + left|right projections of m [S, inner, d] (masked) -> channel-major LRc [2d][chan_stride] */
int af2_outer_project(const af2_outer_weights* w, const float* m, const unsigned char* msa_mask, long long tokens,
                      int inner, int d, void* LRc, long long chan_stride, void* workspace, long long workspace_bytes,
                      af2_stream_t stream);
long long af2_outer_project_workspace(long long tokens, int d);
/* pair rows [row0, row0+rows): x [rows, N, d] += proj_out(sum_s L[s][i] R[s][j] * scale_ij); msa_mask_full [S][N] or NULL */
int af2_outer_contract(const af2_outer_weights* w, float* x, const void* Lc, long long cs_l, const void* Rg,
                       long long cs_r, long long piece_stride, int pieces, const unsigned char* msa_mask_full,
                       int row0, int rows, int N, int S, int d, float eps, void* workspace, long long workspace_bytes,
                       af2_stream_t stream);
long long af2_outer_contract_workspace(int rows, int N, int d);

/* ---------------- rotary.py:9-20 apply_rotary_pos_emb (dead code at HEAD; standalone op) -------------
 * x, y [b, h, n, dh] fp32; sin, cos [sincos_batch, n, rot] with sincos_batch in {1, b}. */
int af2_rotary(const float* x, const float* sin_, const float* cos_, float* y, int b, int h, int n, int dh,
               int rot, int sincos_batch, af2_stream_t stream);

/* ---------------- building blocks, exported for the parity tests -------------------------------------- */
/* y_bf16[T, d] = LayerNorm(x) (nn.LayerNorm semantics) */
int af2_layernorm_bf16(const float* x, const float* gamma, const float* beta, void* y_bf16, long long T, int d,
                       float eps, af2_stream_t stream);
/* C[b] = A[b] B[b]^T (mn_major = 0: A [M,K], B [N,K]) or A[b]^T B[b] (mn_major = 1: A [K,M], B [K,N]);
 * bf16 operands, fp32 accumulation, fp32 output C [batch, M, ldc]. */
int af2_gemm_bf16_f32(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb,
                      long long b_batch, float* C, long long ldc, long long c_batch, int M, int N, int K,
                      int batch, int mn_major, af2_stream_t stream);
/* The same GEMM with the epilogue the module launches use, applied per accumulator column tile of `bn` (64 / 128 / 256,
 * used as given) columns.  mode: 0 bf16 store, 1 gated bf16 (B rows packed per tile as [bn/2 value rows | bn/2 gate rows],
 * out = (u + b_u) * act(g + b_g)), 2 fp32 acc + bias + resid (batch 1 only), 3 fp32 store.  act: 0 none, 1 sigmoid,
 * 2 erf-GELU (applied to the value, or to the gate when gated).  layout: 0 token-major out[b][row][col] (row pitch ld_out),
 * 1 channel-major bf16 out[b][col * ld_out + (row / cm_inner) * cm_pitch + row % cm_inner].  rowscale: fp32 [batch * M]
 * multiplier of every output row when use_rowscale (bf16 modes; mode 2 scales acc + bias before the residual add).  bias: fp32 per accumulator column (N rounded up
 * to even) or NULL.
 * out_cols: valid output columns (0: N, or N / 2 when gated).  out_batch: element stride between batches of out. */
typedef struct {
  int bn, mode, act, layout, use_rowscale;
  const float* bias; const float* rowscale;
  const float* resid; long long ld_resid;
  void* out; long long ld_out; long long out_batch;
  int cm_inner, cm_pitch, out_cols;
} af2_gemm_epilogue;
int af2_gemm_bf16_epilogue(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb, long long b_batch,
                           int M, int N, int K, int batch, int mn_major, const af2_gemm_epilogue* epi, af2_stream_t stream);
/* out[tok, h*dh + e] = gate[tok, h*dh + e] * sum_j softmax_j(q_i . k_j + bias[h][i][j]) v_j[e]  (all in the log2 domain:
 * the softmax is exp2 based, fold dim_head^-0.5 * log2(e) into q and log2(e) into the bias) over the n tokens
 * tok = b * tok_sb + i * tok_si of each of the nbatch folded rows / columns.  qkv bf16 [tokens, 3 * heads * dim_head]
 * (q | k | v), gate bf16 [tokens, heads * dim_head] (sigmoid already applied), bias bf16 [heads][n][align8(n)] or NULL,
 * mask bool indexed like the tokens or NULL: logits where !(mask[i] & mask[j]) are replaced by -FLT_MAX (a fully masked
 * query averages all n values).  dim_head 16, 32, 64 or 128 (the bf16 axial-attention entries take the same set; their
 * strict-mode forms take any multiple of 4). */
int af2_attention_bf16(const void* qkv, const void* gate, const void* bias, const unsigned char* mask, void* out, int n,
                       int nbatch, int heads, int dim_head, long long tok_sb, long long tok_si, af2_stream_t stream);
/* af2_gemm_bf16_f32 with the tile width `bn` (64 / 128 / 256) as given and gathered operands, as the sharded contractions
 * issue it: a_pr > 0 makes A `a_pr`-row (K-major) or -column (MN-major) pieces `a_piece` elements apart, row / column
 * r = p * a_pr + rr of piece p; b_pr / b_piece likewise for B.  0 = a plain operand.  K-major A pieces must be a multiple
 * of 128 rows and B pieces a multiple of 8 rows that divides or is divided by bn; MN-major pieces a multiple of 64 columns. */
int af2_gemm_bf16_f32_gathered(const void* A, long long lda, long long a_batch, const void* Bm, long long ldb, long long b_batch,
                               float* C, long long ldc, long long c_batch, int M, int N, int K, int batch, int mn_major, int bn,
                               int a_pr, long long a_piece, int b_pr, long long b_piece, af2_stream_t stream);
/* The tail of the triangle / outer-product contractions: channel-major fp32 src[c * chan_stride + row * pitch + j] (c < d,
 * row < rows, j < n) -> token-major bf16 y[t][c], t = row * n + j:
 *   mode 0: y = (LayerNorm_c(src) * gamma + beta) * gate[t][c]      (gate bf16 [tokens][d])
 *   mode 1: y = src * scale[t]                                       (scale fp32 [tokens], or scale_const when NULL)
 * variant: 0 the kernel the modules get, 1 SIMT, 2 tile, 3 TMA; a forced kernel whose preconditions the call does not meet
 * returns AF2_ERR_BAD_ARG and launches nothing.  *ran (may be NULL) receives the kernel launched (0: none, T = 0).
 * af2_chan_to_token_select returns the kernel variant 0 would launch for these arguments, without launching. */
int af2_chan_to_token(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode, const float* gamma,
                      const float* beta, const void* gate, const float* scale, float scale_const, float eps, void* y, int variant,
                      int* ran, af2_stream_t stream);
int af2_chan_to_token_select(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode,
                             const float* gamma, const float* beta, const void* gate, const float* scale, float scale_const,
                             float eps, void* y);
/* OuterMean normaliser of pair rows [row0, row0 + rows): scale[(i - row0) * N + j] = 1 / (S * (count_ij + eps)), count_ij =
 * sum_s (mask[s][i] & mask[s][j]), mask bool [S][N].  words: workspace of ceil(S / 32) * N uint32 for the bit-packed
 * kernel, or NULL.  variant: 0 the modules' choice (bit-packed when words is given and ceil(S / 32) * N * 4 <= 160 KB),
 * 1 byte loop, 2 bit-packed (AF2_ERR_BAD_ARG when it does not apply).  *ran (may be NULL) receives the variant launched. */
int af2_outer_scale(const unsigned char* mask, float* scale, void* words, int row0, int rows, int S, int N, float eps, int variant,
                    int* ran, af2_stream_t stream);

/* ======================================================================================================================
 * STRICT precision mode (alphafold2_b200.set_precision(model, "strict")): the same modules with fp32 activations between
 * kernels and split-bf16 operands on the tensor cores (v = p0 + p1 + p2, three bf16 planes = 24 mantissa bits; the six
 * products down to 2^-24 accumulated in fp32), so that results match the reference's fp32 path inside the north star's
 * rtol 1e-3 / atol 1e-4 also after 12 blocks.  Split weights: bf16 [rows][3][align8(cols)] (plane-major per row), built by
 * ops.split_weight().
 * ====================================================================================================================== */
typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* FeedForward.norm                                   */
  const void* w1; const float* b1;                    /* net.0  split [2*hid][3][align8(d)], fp32 [2*hid]    */
  const void* w2; const float* b2;                    /* net.3  split [d][3][align8(hid)],   fp32 [d]        */
} af2_ff_weights_strict;
long long af2_feed_forward_strict_workspace(long long tokens, int d, int hidden);
int af2_feed_forward_strict(const af2_ff_weights_strict* w, float* x, long long tokens, int d, int hidden, void* workspace,
                            long long workspace_bytes, af2_stream_t stream);                 /* alphafold2.py:74-94 */

typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* AxialAttention.norm                                              */
  const void* w_qkvg; const float* b_qkvg;            /* [to_q * dim_head^-0.5 ; to_kv ; gating] split [4I][3][align8(d)], bias [4I] (zeros | gating.bias) */
  const void* w_out; const float* b_out;              /* attn.to_out split [d][3][align8(I)], fp32 [d]                    */
  const float* w_edge;                                /* edges_to_attn_bias.0.weight fp32 [H][d] or NULL                  */
} af2_attn_weights_strict;
long long af2_axial_attention_strict_workspace(int B, int h, int w, int d, int heads, int dim_head, int row_attn);
int af2_axial_attention_strict(const af2_attn_weights_strict* w, float* x, const float* edges, const unsigned char* mask, int B,
                               int h, int wdim, int d, int heads, int dim_head, int row_attn, int flags, void* workspace,
                               long long workspace_bytes, af2_stream_t stream);              /* alphafold2.py:98-255; flags as af2_axial_attention_ex */

typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* norm                                                                          */
  const void* w5; const float* b5;                    /* [left_proj; right_proj; left_gate; right_gate; out_gate] split [5d][3][align8(d)], fp32 [5d] */
  const float* on_gamma; const float* on_beta;        /* to_out_norm                                                                   */
  const void* w_out; const float* b_out;              /* to_out split [d][3][align8(d)], fp32 [d]                                      */
} af2_trimul_weights_strict;
long long af2_triangle_multiply_strict_workspace(int B, int N, int d);
int af2_triangle_multiply_strict(const af2_trimul_weights_strict* w, float* x, const unsigned char* mask, int B, int N, int d,
                                 int ingoing, void* workspace, long long workspace_bytes, af2_stream_t stream);   /* alphafold2.py:257-317 */

typedef struct {
  const float* ln_gamma; const float* ln_beta;        /* norm                                                       */
  const void* w_lr; const float* b_lr;                /* [left_proj; right_proj] split [2d][3][align8(d)], fp32 [2d] */
  const void* w_out; const float* b_out;              /* proj_out split [d][3][align8(d)], fp32 [d]                 */
} af2_outer_weights_strict;
long long af2_outer_mean_strict_workspace(int B, int S, int N, int d);
int af2_outer_mean_strict(const af2_outer_weights_strict* w, float* x, const float* m, const unsigned char* msa_mask, int B, int S,
                          int N, int d, float eps, void* workspace, long long workspace_bytes, af2_stream_t stream);   /* alphafold2.py:321-351 */

/* building blocks exported for the parity tests: the launches the strict modules make, one entry point per kernel.  A split
 * operand row holds its 3 bf16 planes `half` elements apart; every SIMT kernel below writes p0 = bf16(v), p1 = bf16(v - p0),
 * p2 = bf16(v - p0 - p1).  Token-major split rows are [rows][3][align8(cols)] with the pad columns [cols, align8(cols))
 * zeroed, except where noted.
 * af2_split_bf16: y split of x fp32 [rows][K] (af2_strict_ln_split without the LayerNorm).
 * af2_gemm_split_f32: C[b] fp32 [M][ldc] = A[b] B[b]^T on split A [batch][M][3][align8(K)], B [batch][N][3][align8(K)].
 * af2_gemm_split_epilogue: the split GEMM as the modules issue it.  mn_major = 0: A row m at A + b * a_batch + m * lda,
 *   plane p at + p * a_half, k contiguous; mn_major = 1: A element (k, m) of plane p at A + b * a_batch + p * a_half + k * lda
 *   + m; B likewise.  Six tensor-core passes (A plane, B plane) = (0,2) (2,0) (1,1) (0,1) (1,0) (0,0) into one fp32
 *   accumulator.  epi: bn (64 / 128 / 256) used as given; mode 3 (fp32 store, bias or NULL) or 2 (fp32 acc + bias + resid,
 *   batch 1) only, act 0, layout 0, no row scale; anything else returns AF2_ERR_BAD_ARG and launches nothing.
 * af2_strict_ln_split: y split [T][3][align8(d)] = LayerNorm(x) * gamma + beta (eps 1e-5), or x when gamma = beta = NULL.
 * af2_strict_geglu_split: y split [T][3][align8(hidden)] = a * gelu_erf(g), h fp32 [T][2 * hidden] = (a | g).
 * af2_strict_gelu_split: y split [rows][3][align8(d)] = gelu_erf(h), h fp32 [rows][d].
 * af2_strict_qkv_split: from p1 fp32 [tokens][4I] = (q | k | v | gate logits), I = heads * dim_head, token(b', i) =
 *   (b0 + b') * tok_sb + i * tok_si for the folded batch elements b' < nb: Q, K split [nb * heads][n][3][align8(dim_head)],
 *   Vt split [nb * heads][dim_head][3][align8(n)].
 * af2_strict_pair_bias: bias fp32 [heads][T] = x fp32 [T][d] . w_edge fp32 [heads][d].
 * af2_strict_softmax_split: P split [nb * heads][n][3][align8(n)] = softmax_j(S[r][j] + bias[h][i][j]) of the logits S fp32
 *   [nb * heads][n][lds]; bias fp32 [heads][n][n] or NULL; mask bool or NULL, key j of folded batch element b' at
 *   mask[(b0 + b') * mask_sb + j * mask_si]: where !(mask[i] & mask[j]) the logit is replaced by -FLT_MAX.
 * af2_strict_gate_split: og split rows of the tokens of b' < nb, [tokens][3][align8(I)] = O[(b' heads + h) n + i][e] (row
 *   pitch ldo) * sigmoid(p1[token][3I + h dim_head + e]).
 * af2_strict_tok2chan_split: out[c * cs + plane * hs + r * rs + k] = src[t][val_off + c] * sigmoid(src[t][gate_off + c])
 *   (no gate when gate_off < 0) * mask[t] (mask bool or NULL), t = r * inner + k, src row pitch ld; writes no pad.
 * af2_strict_chan_to_token: y split [rows * n][3][align8(d)] of src fp32 [c * chan_stride + row * pitch + j]: mode 0
 *   (LayerNorm_c(src) * gamma + beta) * sigmoid(gate_src[t][gate_off + c]) (row pitch gate_ld), mode 1 src * (scale[t] or
 *   scale_const when scale is NULL).
 * af2_tie_queries_f32 / _bf16: buf[(b tok_sb + i tok_si) * ld + c] <- mean over b < nbatch, for i < n and c < cols. */
int af2_split_bf16(const float* x, void* y_split, long long rows, int K, af2_stream_t stream);
int af2_gemm_split_f32(const void* A_split, const void* B_split, float* C, long long ldc, int M, int N, int K, int batch,
                       af2_stream_t stream);
int af2_gemm_split_epilogue(const void* A, long long lda, long long a_half, long long a_batch, const void* Bm, long long ldb,
                            long long b_half, long long b_batch, int M, int N, int K, int batch, int mn_major,
                            const af2_gemm_epilogue* epi, af2_stream_t stream);
int af2_strict_ln_split(const float* x, const float* gamma, const float* beta, void* y, long long T, int d, af2_stream_t stream);
int af2_strict_geglu_split(const float* h, void* y, long long T, int hidden, af2_stream_t stream);
int af2_strict_gelu_split(const float* h, void* y, long long rows, int d, af2_stream_t stream);
int af2_strict_qkv_split(const float* p1, void* Q, void* K, void* Vt, int b0, int nb, int heads, int n, int dim_head,
                         long long tok_sb, long long tok_si, af2_stream_t stream);
int af2_strict_pair_bias(const float* x, const float* w_edge, float* bias, long long T, int d, int heads, af2_stream_t stream);
int af2_strict_softmax_split(const float* S, long long lds, const float* bias, const unsigned char* mask, void* P, int b0, int nb,
                             int heads, int n, long long mask_sb, long long mask_si, af2_stream_t stream);
int af2_strict_gate_split(const float* O, long long ldo, const float* p1, void* og, int b0, int nb, int heads, int n, int dim_head,
                          long long tok_sb, long long tok_si, af2_stream_t stream);
int af2_strict_tok2chan_split(const float* src, long long ld, int val_off, int gate_off, const unsigned char* mask, void* out, int C,
                              int rows, int inner, long long cs, long long hs, long long rs, af2_stream_t stream);
int af2_strict_chan_to_token(const float* src, long long chan_stride, int pitch, int rows, int n, int d, int mode, const float* gamma,
                             const float* beta, const float* gate_src, long long gate_ld, int gate_off, const float* scale,
                             float scale_const, float eps, void* y, af2_stream_t stream);
int af2_tie_queries_f32(float* buf, long long ld, int cols, int n, int nbatch, long long tok_sb, long long tok_si, af2_stream_t stream);
int af2_tie_queries_bf16(void* buf, long long ld, int cols, int n, int nbatch, long long tok_sb, long long tok_si, af2_stream_t stream);

/* ---------------- pre- / post-trunk glue as fused kernels (SURVEY.md 8f n1) -------------------------------------------
 * af2_embed_pair_init: alphafold2.py:676-726 -- token embedding gather, m = (emb[msa] + msa_embed) + emb[seq],
 *   x[i][j] = (left[i] + right[j]) + pos_emb[clamp(idx_i - idx_j, -R, R) + R] with [left|right] = to_pairwise_repr(emb[seq] + seq_embed).
 *   seq [B][n], msa [B][S][n] int64 token ids (msa / m may be NULL); seq_embed, msa_embed, seq_index optional (NULL).
 * af2_distogram_head: alphafold2.py:821-823 -- out = Linear_{d -> buckets}(LayerNorm((x + x^T) / 2)), all fp32. */
long long af2_embed_pair_init_workspace(int B, int n, int d);
int af2_embed_pair_init(const long long* seq, const long long* msa, const float* token_emb, int vocab, const float* seq_embed,
                        const float* msa_embed, const float* w_pair, const float* b_pair, const float* pos_emb, int max_rel_dist,
                        const long long* seq_index, float* x, float* m, int B, int S, int n, int d, void* workspace,
                        long long workspace_bytes, af2_stream_t stream);
int af2_distogram_head(const float* x, const float* gamma, const float* beta, const float* w, const float* bias, float* out, int B,
                       int n, int d, int buckets, af2_stream_t stream);
/* Row shards of the glue and the heads (parallel.shard_alphafold2(pair_rows=True)): each gives, bitwise, the pair rows
 * [row0, row0 + rows) of its whole-tensor sibling, with the sibling's argument rules plus 0 <= row0, 0 <= rows, row0 + rows <= n;
 * otherwise AF2_ERR_BAD_ARG and nothing is written.
 * af2_embed_pair_init_rows: x_rows [B][rows][n][d]; m [B][S][n][d] whole, as af2_embed_pair_init.
 * af2_distogram_head_rows / af2_angle_heads_rows (one batch element): x_rows [rows][n][d] and the same rows as columns,
 *   x_cols [n][rows][d] with x_cols[j][i - row0] = x[j][i] (the rows -> columns exchange of the shard) -> [rows][n][buckets].
 *   af2_angle_heads_rows reads x_cols only when symmetrize (it may be NULL otherwise). */
int af2_embed_pair_init_rows(const long long* seq, const long long* msa, const float* token_emb, int vocab, const float* seq_embed,
                             const float* msa_embed, const float* w_pair, const float* b_pair, const float* pos_emb, int max_rel_dist,
                             const long long* seq_index, float* x_rows, float* m, int B, int S, int n, int d, int row0, int rows,
                             void* workspace, long long workspace_bytes, af2_stream_t stream);
int af2_distogram_head_rows(const float* x_rows, const float* x_cols, const float* gamma, const float* beta, const float* w,
                            const float* bias, float* out, int rows, int n, int d, int buckets, af2_stream_t stream);
int af2_angle_heads_rows(const float* x_rows, const float* x_cols, const void* w_planes, const float* bias, float* theta, float* phi,
                         float* omega, int rows, int n, int d, int n_theta, int n_phi, int n_omega, int symmetrize,
                         af2_stream_t stream);
/* af2_angle_heads: alphafold2.py:813-836 (predict_angles) -- one pass over x [B][n][n][d] fp32:
 *   theta[b][i][j] = W_t x[b][i][j] + b_t    [B][n][n][n_theta]      phi = W_p x + b_p    [B][n][n][n_phi]
 *   omega[b][i][j] = W_o s + b_o             [B][n][n][n_omega],     s = (x[b][i][j] + x[b][j][i]) * 0.5 if symmetrize, else x[b][i][j]
 *   (symmetrized, omega is bitwise symmetric in i, j).  fp32 results from split-bf16 tensor-core passes: the same kernel serves
 *   both precision modes.
 *   w_planes: bf16 [d / 32][3][64][32], the three split planes (p0 = bf16(w), p1 = bf16(w - p0), p2 = bf16(w - p0 - p1)) of the
 *     64-row weight [W_t; W_p; W_o; zero rows], 32 channels per block; bias [64] fp32 [b_t; b_p; b_o; zeros].
 *   d % 32 == 0 and d <= 320 (dim 320 symmetrized, 384 otherwise: shared memory); n_theta + n_phi + n_omega <= 64; symmetrized,
 *   omega's columns fit the 32-column window from min(8 floor((n_theta + n_phi) / 8), 32).  x and w_planes 16-byte aligned.  No workspace.  Otherwise AF2_ERR_BAD_ARG. */
int af2_angle_heads(const float* x, const void* w_planes, const float* bias, float* theta, float* phi, float* omega, int B, int n,
                    int d, int n_theta, int n_phi, int n_omega, int symmetrize, af2_stream_t stream);
/* af2_recycle_embed: alphafold2.py:730-739 -- the recycling embedder, in place, one launch:
 *   x[b][i][j] = (x[b][i][j] + LN_pair(prev_pair[b][i][j])) + table[k(b, i, j)]        x, prev_pair [B][n][n][d]
 *   m[b][0][j] = m[b][0][j] + LN_msa(single_row[b][j])                                 single_row [B][n][d]; no other row of m changes
 *   k = lower bound of dist in boundaries[0 .. nb-2] under !(boundary >= dist), i.e. torch.bucketize(right=False): NaN -> nb - 1,
 *   and nb == 1 -> 0.  dist = sqrtf(sum_e (coords[b][i][e] - coords[b][j][e])^2) over coords [B][n][c] fp32, summed in order
 *   (the direct distance; torch.cdist switches to a less exact formula for n > 25).  boundaries [nb] as built by the caller
 *   (torch.linspace(2, 20, nb)); table [nb][d]; LayerNorm fp32, two-pass, biased variance, eps.
 *   m is addressed as m + b * m_bstride + j * d (elements): m may hold more rows than the S MSA rows (template angles).
 *   Rows (x, m, prev_pair, single_row, table, gammas, betas) 16-byte aligned, d % 4 == 0, d <= 1024, c >= 1, nb >= 1; otherwise
 *   AF2_ERR_BAD_ARG and nothing is launched.  All fp32: strict mode uses the same kernel. */
int af2_recycle_embed(const float* coords, int c, const float* single_row, const float* prev_pair, const float* msa_gamma,
                      const float* msa_beta, const float* pair_gamma, const float* pair_beta, const float* table,
                      const float* boundaries, int nb, float* x, float* m, long long m_bstride, int B, int n, int d, float eps,
                      af2_stream_t stream);
/* af2_recycle_embed_rows: the same on pair rows [row0, row0 + rows): x_rows, prev_pair_rows [B][rows][n][d] (coords whole);
 *   row 0 of m is updated whole, as af2_recycle_embed does. */
int af2_recycle_embed_rows(const float* coords, int c, const float* single_row, const float* prev_pair_rows, const float* msa_gamma,
                           const float* msa_beta, const float* pair_gamma, const float* pair_beta, const float* table,
                           const float* boundaries, int nb, float* x_rows, float* m, long long m_bstride, int B, int n, int d,
                           float eps, int row0, int rows, af2_stream_t stream);

/* ---------------- template embedder: alphafold2.py:743-785 (SURVEY.md 8f n3) ---------------------------------------------
 * The template pair stack is af2_triangle_multiply / af2_axial_attention with batch B * T.  The rest:
 *
 * af2_template_pointwise_attention: Attention(x, context = t, mask = x_mask, context_mask = t_mask) at every pair position, in
 *   place on x [B][n][n][d], multiplied by the pooled mask and added (alphafold2.py:764-785):
 *     q = to_q(x) * dim_head^-0.5, [k | v] = to_kv(t), no LayerNorm on either side; template t of pair p = (b, i, j) is row
 *     (b T + t) n^2 + i n + j of t [B T][n][n][d] and of the crossed template mask t_mask [B T][n][n] (NULL: all valid);
 *     logits where !(x_mask[p] & t_mask[...]) are -FLT_MAX, so a pair masked by x_mask, or with every template masked, gets
 *     the uniform mean over all T templates;  x[p] += pooled[p] * (to_out(softmax_t(q k_t) v_t * sigmoid(gating(x[p]))) + b_out)
 *     with pooled[p] = any_t t_mask (NOT x_mask).  x_mask [B][n][n] or NULL.  dim_head / 8 a power of two <= 32 (8..256),
 *     any heads, any T >= 1, d % 8 == 0.  The strict twin: dim_head / 4 a power of two <= 32, fp32 attention with expf. */
typedef struct {
  const void* w_q;                                    /* to_q * dim_head^-0.5 * log2(e)  bf16 [I][d]      */
  const void* w_gate; const float* b_gate;            /* gating                          bf16 [I][d], [I] */
  const void* w_kv;                                   /* to_kv                           bf16 [2I][d]     */
  const void* w_out; const float* b_out;              /* to_out                          bf16 [d][I], [d] */
} af2_template_attn_weights;
long long af2_template_pointwise_attention_workspace(int B, int T, int n, int d, int heads, int dim_head);
int af2_template_pointwise_attention(const af2_template_attn_weights* w, float* x, const float* t, const unsigned char* x_mask,
                                     const unsigned char* t_mask, int B, int T, int n, int d, int heads, int dim_head,
                                     void* workspace, long long workspace_bytes, af2_stream_t stream);
typedef struct {
  const void* w_qg; const float* b_qg;                /* [to_q * dim_head^-0.5 ; gating] split [2I][3][align8(d)], fp32 [2I] (zeros | gating.bias) */
  const void* w_kv;                                   /* to_kv split [2I][3][align8(d)]                                        */
  const void* w_out; const float* b_out;              /* to_out split [d][3][align8(I)], fp32 [d]                              */
} af2_template_attn_weights_strict;
long long af2_template_pointwise_attention_strict_workspace(int B, int T, int n, int d, int heads, int dim_head);
int af2_template_pointwise_attention_strict(const af2_template_attn_weights_strict* w, float* x, const float* t,
                                            const unsigned char* x_mask, const unsigned char* t_mask, int B, int T, int n, int d,
                                            int heads, int dim_head, void* workspace, long long workspace_bytes, af2_stream_t stream);
/* The pointwise kernel alone, on P = B * pairs pair positions:  out[p] = gate[p] * sum_t softmax_t(q[p] . k) v,  k | v = kv row
 * (b T + t) * pairs + (p % pairs), kv [B T pairs][2I] (k | v); pooled fp32 [P] = any_t t_mask; masks as above (t_mask indexed
 * like the kv rows).  _bf16: q [P][I] pre-scaled by dim_head^-0.5 * log2(e) (exp2-domain softmax), gate [P][I] with the sigmoid
 * applied, out bf16 [P][I].  _f32 (the strict instantiation): q pre-scaled by dim_head^-0.5, gate_logits BEFORE the sigmoid,
 * out fp32.  q, gate, kv and out 16-byte aligned.  A shape the kernel does not support returns AF2_ERR_BAD_ARG and launches
 * nothing. */
int af2_template_pointwise_bf16(const void* q, const void* gate, const void* kv, const unsigned char* x_mask,
                                const unsigned char* t_mask, void* out, float* pooled, int B, int T, long long pairs, int heads,
                                int dim_head, af2_stream_t stream);
int af2_template_pointwise_f32(const float* q, const float* gate_logits, const float* kv, const unsigned char* x_mask,
                               const unsigned char* t_mask, float* out, float* pooled, int B, int T, long long pairs, int heads,
                               int dim_head, af2_stream_t stream);
/* The same kernel over one group of templates, carrying the online-softmax state from launch to launch: kv / t_mask hold the
 * group's T templates only.  State, all fp32: run_max and run_sum [P][heads], acc [P][I] (16-byte aligned), and pooled [P],
 * which holds "any template valid" (0 / 1) between groups.  first = 1: start from no state (nothing is read);  last = 1: write out
 * and pooled as above (nothing else);  last = 0: write the state instead (out is not touched and may be NULL).  first = last = 1
 * is af2_template_pointwise_bf16 / _f32 and the state pointers may be NULL.  Running every group in order gives out and pooled
 * bitwise equal to one launch over all templates.  out may be q (_bf16) or acc (_f32): each element is read before it is
 * written, by the same thread. */
int af2_template_pointwise_bf16_state(const void* q, const void* gate, const void* kv, const unsigned char* x_mask,
                                      const unsigned char* t_mask, void* out, float* pooled, float* run_max, float* run_sum, float* acc,
                                      int first, int last, int B, int T, long long pairs, int heads, int dim_head, af2_stream_t stream);
int af2_template_pointwise_f32_state(const float* q, const float* gate_logits, const float* kv, const unsigned char* x_mask,
                                     const unsigned char* t_mask, float* out, float* pooled, float* run_max, float* run_sum, float* acc,
                                     int first, int last, int B, int T, long long pairs, int heads, int dim_head, af2_stream_t stream);
/* af2_template_pointwise_attention in groups of templates, so that only one group's t and k|v are in memory at a time
 * (af2_template_pointwise_attention{,_strict} is exactly begin, one group of all T with first = last = 1, end):
 *   begin: q, gate from x into caller-owned buffers: bf16 q [P][I] and gate [P][I] (sigmoid-ed);  strict: qg fp32 [P][2I]
 *     = [q * dim_head^-0.5 | gating logits].  P = B n^2.
 *   group: for G templates, t fp32 [B G][n][n][d] and their crossed mask t_mask [B G][n][n] (template g of pair (b, i, j) is
 *     row (b G + g) n^2 + i n + j), in order over the groups with first = 1 on the first and last = 1 on the last: the k|v
 *     projection and the state-carrying kernel above.  run_max, run_sum, acc, pooled: the caller-owned state (fp32; acc
 *     16-byte aligned; run_max / run_sum / acc may be NULL when first = last = 1).  On the last group the gated attention output
 *     goes to out: bf16 [P][I], which may be q;  strict fp32 [P][I], which may be acc.
 *   end: x += pooled * (to_out(out) + b_out).
 * The state lives in caller memory because each call draws its workspace afresh. */
long long af2_template_pointwise_begin_workspace(int B, int n, int d);
int af2_template_pointwise_begin(const af2_template_attn_weights* w, const float* x, int B, int n, int d, int heads, int dim_head,
                                 void* q, void* gate, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_group_workspace(int B, int G, int n, int d, int heads, int dim_head);
int af2_template_pointwise_group(const af2_template_attn_weights* w, const float* t, const unsigned char* x_mask,
                                 const unsigned char* t_mask, int B, int G, int n, int d, int heads, int dim_head, const void* q,
                                 const void* gate, float* run_max, float* run_sum, float* acc, float* pooled, void* out, int first,
                                 int last, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_end_workspace(int B, int n, int heads, int dim_head);
int af2_template_pointwise_end(const af2_template_attn_weights* w, float* x, const void* out, const float* pooled, int B, int n, int d,
                               int heads, int dim_head, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_begin_strict_workspace(int B, int n, int d);
int af2_template_pointwise_begin_strict(const af2_template_attn_weights_strict* w, const float* x, int B, int n, int d, int heads,
                                        int dim_head, float* qg, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_group_strict_workspace(int B, int G, int n, int d, int heads, int dim_head);
int af2_template_pointwise_group_strict(const af2_template_attn_weights_strict* w, const float* t, const unsigned char* x_mask,
                                        const unsigned char* t_mask, int B, int G, int n, int d, int heads, int dim_head, const float* qg,
                                        float* run_max, float* run_sum, float* acc, float* pooled, float* out, int first, int last,
                                        void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_end_strict_workspace(int B, int n, int heads, int dim_head);
int af2_template_pointwise_end_strict(const af2_template_attn_weights_strict* w, float* x, const float* out, const float* pooled, int B,
                                      int n, int d, int heads, int dim_head, void* workspace, long long workspace_bytes,
                                      af2_stream_t stream);
/* begin / group / end (bf16) on a window of P consecutive pairs of one batch element, e.g. a band of pair rows [i0, i1) of
 * batch element b: P = (i1 - i0) n, window offset o = b n^2 + i0 n.  Every pointer points at the window: x + o d, q, gate and
 * out [P][I] (window-sized, caller-owned), x_mask + o, and the window's slice of the whole-tensor state: run_max + o heads,
 * run_sum + o heads, acc + o I, pooled + o.  group: t points at template 0's first window row, t_mask at its crossed-mask
 * entry; template g's rows start g t_stride pairs later (t_stride >= P; for t [B G][n][n][d] from the grouped entry points,
 * t + (b G n^2 + i0 n) d and t_stride = n^2).  Workspaces are sized for the window only.  Running, for every group in order,
 * every window's begin and group (first / last as above), and end after the last group, gives x bitwise equal to the
 * whole-tensor calls.  x, t, q, gate, out and acc 16-byte aligned; d a multiple of 8. */
long long af2_template_pointwise_rows_begin_workspace(long long P, int d);
int af2_template_pointwise_rows_begin(const af2_template_attn_weights* w, const float* x, long long P, int d, int heads, int dim_head,
                                      void* q, void* gate, void* workspace, long long workspace_bytes, af2_stream_t stream);
long long af2_template_pointwise_rows_group_workspace(int G, long long P, int d, int heads, int dim_head);
int af2_template_pointwise_rows_group(const af2_template_attn_weights* w, const float* t, const unsigned char* x_mask,
                                      const unsigned char* t_mask, int G, long long P, long long t_stride, int d, int heads,
                                      int dim_head, const void* q, const void* gate, float* run_max, float* run_sum, float* acc,
                                      float* pooled, void* out, int first, int last, void* workspace, long long workspace_bytes,
                                      af2_stream_t stream);
long long af2_template_pointwise_rows_end_workspace(long long P, int heads, int dim_head);
int af2_template_pointwise_rows_end(const af2_template_attn_weights* w, float* x, const void* out, const float* pooled, long long P,
                                    int d, int heads, int dim_head, void* workspace, long long workspace_bytes, af2_stream_t stream);
/* to_template_embed (alphafold2.py:751): t fp32 [rows][d] = feats fp32 [rows][K] W^T + bias.  w bf16 [d][align8(K)] (zero pad
 * columns); _strict: w split [d][3][align8(K)]. */
long long af2_template_embed_workspace(long long rows, int K);
int af2_template_embed(const void* w, const float* bias, const float* feats, float* t, long long rows, int K, int d, void* workspace,
                       long long workspace_bytes, af2_stream_t stream);
long long af2_template_embed_strict_workspace(long long rows, int K);
int af2_template_embed_strict(const void* w_split, const float* bias, const float* feats, float* t, long long rows, int K, int d,
                              void* workspace, long long workspace_bytes, af2_stream_t stream);
/* template_angle_mlp (alphafold2.py:789-792): Linear(K -> d), exact-erf GELU, Linear(d -> d) of angles fp32 [B][T][n][K], written
 * as fp32 rows row0 .. row0 + T - 1 of m [B][m_rows][n][d] (the reference appends them after the S MSA rows: row0 = S). */
typedef struct {
  const void* w1; const float* b1;                    /* template_angle_mlp.0  bf16 [d][align8(K)] (zero pad columns), [d] */
  const void* w2; const float* b2;                    /* template_angle_mlp.2  bf16 [d][d], [d]                            */
} af2_template_angle_weights;
long long af2_template_angles_workspace(int B, int T, int n, int K, int d);
int af2_template_angles(const af2_template_angle_weights* w, const float* angles, float* m, int B, int T, int n, int K, int d,
                        int m_rows, int row0, void* workspace, long long workspace_bytes, af2_stream_t stream);
typedef struct {
  const void* w1; const float* b1;                    /* split [d][3][align8(K)], fp32 [d] */
  const void* w2; const float* b2;                    /* split [d][3][align8(d)], fp32 [d] */
} af2_template_angle_weights_strict;
long long af2_template_angles_strict_workspace(int B, int T, int n, int K, int d);
int af2_template_angles_strict(const af2_template_angle_weights_strict* w, const float* angles, float* m, int B, int T, int n, int K,
                               int d, int m_rows, int row0, void* workspace, long long workspace_bytes, af2_stream_t stream);

/* ---- peer-memory exchange for the sharded trunk (alphafold2_b200/parallel.py; no reference counterpart: the reference
 * has no multi-GPU path, SURVEY.md 8(e)) ----
 * Every rank owns one arena (af2_peer_alloc: cudaMalloc, zeroed; the first af2_peer_ctrl_bytes() bytes are the barrier
 * control block) which the other ranks of the node map with CUDA IPC (export -> 64-byte handle -> open).  One
 * af2_peer_exchange launch re-lays a row shard out as column shards (or back): chunk p = `rows` rows of `row_bytes`
 * contiguous bytes, read at src + p*src_peer_stride + row*src_row_stride, stored into rank p's arena at
 * dst_off + row*dst_row_stride, followed inside the same kernel by a flag barrier over all P ranks (channel 0 or 1: two
 * exchanges may be in flight on two streams).  peer_base is a DEVICE array of the P arena bases as mapped in this
 * process (own arena at index `rank`).  Every rank must issue the same sequence of exchanges per channel.
 * af2_peer_error returns 1 if a barrier ever gave up waiting (20 s) for a rank. */
int af2_peer_ctrl_bytes(void);
int af2_peer_can_access(int device, int peer_device);
int af2_peer_alloc(long long bytes, void** ptr);
int af2_peer_free(void* ptr);
int af2_peer_export(const void* ptr, unsigned char* handle64);
int af2_peer_open(const unsigned char* handle64, void** ptr);
int af2_peer_close(void* ptr);
int af2_peer_error(const void* my_base);
int af2_peer_exchange(const void* src, long long src_peer_stride, long long src_row_stride, void* const* peer_base,
                      long long dst_off, long long dst_row_stride, int rows, long long row_bytes, int channel, int rank, int P,
                      af2_stream_t stream);
/* The same exchange for uneven shards: chunks is a HOST array of P entries, chunks[p] the chunk bound for rank p
 * (`rows` rows of `row_bytes`, read at src + src_off + row*src_row_stride, stored into rank p's arena at
 * dst_off + row*dst_row_stride).  rows may be 0 (0 .. 65535); a rank with nothing to send still joins the barrier.
 * Offsets, strides and row bytes are multiples of 16, row_bytes >= 16 where rows > 0.  At most 32 ranks. */
typedef struct {
  long long src_off, dst_off, dst_row_stride, row_bytes;
  int rows, reserved;
} af2_peer_chunk;
int af2_peer_exchange_chunks(const void* src, long long src_row_stride, const af2_peer_chunk* chunks, void* const* peer_base,
                             int channel, int rank, int P, af2_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* AF2B200_H */
