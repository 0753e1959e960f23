/* bevbert_b200 C ABI — the sm_90a kernels behind the BEVBert hybrid-map encoder hot path.
 *
 * Conventions (SURVEY.md 8b):
 *   - every pointer is a DEVICE pointer on the current CUDA device unless the name ends in _host;
 *   - the caller owns every buffer (inputs, outputs, workspaces); nothing here allocates device memory;
 *   - every launch goes on the caller's `stream` (a cudaStream_t passed as void*); no internal sync;
 *   - return value: 0 = ok, <0 = error; bb_last_error() returns a thread-local message;
 *   - re-entrant; one process per GPU.
 *
 * The reference (MarSaKi/VLN-BEVBert) has no FFI layer of its own: each entry point cites the PyTorch
 * call sites in the reference that it replaces (paths relative to the reference root).
 */
#ifndef BEVBERT_B200_H
#define BEVBERT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* bb_last_error(void);
int bb_abi_version(void);
/* number of kernels launched through this library by the calling process since load / last reset */
int64_t bb_launch_count(void);
void bb_reset_launch_count(void);

/* Registers a 64-bit word in DEVICE memory that every kernel XORs into its dropout seed (NULL = none, the default).
 * Needed for CUDA-graph replay of a training step: seeds are kernel parameters and therefore frozen in a captured graph;
 * the caller rewrites this word before each replay to draw fresh masks (forward and backward of one step see the same
 * value, so masks are still replayed exactly).  Synchronous (cudaMemcpyToSymbol); call it once, outside capture. */
int bb_set_drop_salt_ptr(const uint64_t* device_word);

/* Deterministic mode.  on = 1: every kernel gives bit-identical results for bit-identical inputs on the same build and
 * GPU model, whatever the scheduling (side stream, CUDA-graph replay, concurrent work).  Reductions across CTAs (split-K
 * weight gradients, LayerNorm dgamma / dbeta, bias column sums, graph-bias gradients, the gradient sum of squares)
 * store partials to the workspace and add them in a fixed order; no CTA waits on another.  The atomic scatter-adds
 * (bb_embed_scatter_grad's word table, bb_scatter_add_rows, bb_segment_wsum_bwd) fail in this mode: their callers sort
 * by destination and use bb_scatter_rows_sorted.  A launch without a deterministic implementation (the fused-scores
 * graph-bias gradient of bb_attn_scores) fails.  on = 2: the same, except that such a launch runs (the caller warns).
 * on = 0 (default): fp32 atomics, as before.  Host state, takes effect at the next launch. */
int bb_set_deterministic(int on);
/* Workspaces of the deterministic mode, owned by the caller, 256-byte aligned, `bytes` each, zero-filled before
 * registration: the first 64 KB hold split-K arrival counters that every launch leaves at zero.  Launches on the
 * registered side stream (bb_set_side_stream) use side_ws, every other launch main_ws.  A deterministic launch whose
 * workspace is missing or too small fails and bb_last_error() gives the size it needs: 64 KB plus, for a split-K GEMM,
 * split x output tiles x 128 x tile width x 4 bytes (tiles 64 or 128 wide), for the other reductions a few MB at most.
 * NULL, NULL, 0 unregisters. */
int bb_set_det_workspace(void* main_ws, void* side_ws, int64_t bytes);

/* ---------------------------------------------------------------------------------------------
 * Batched bf16 GEMM on wgmma tensor cores, TMA-fed, fp32 accumulation in registers.
 *   D[b] = epi( alpha * A[b] (M x K) * B[b]^T (N x K) )
 * Operand element (m,k) of A lives at  A + b1*a_s1 + b2*a_s2 + (a_mn ? k*lda + m : m*lda + k),
 * operand element (n,k) of B lives at  B + b1*b_s1 + b2*b_s2 + (b_mn ? k*ldb + n : n*ldb + k).
 * All strides are in elements; lda, ldb and the batch strides must be multiples of 8 (16-byte TMA strides).
 * Replaces: every nn.Linear / torch.matmul on the path (pretrain_src/model/vilmodel.py:92-94,108-110,
 * 117,133,146,171,185,314-316,335,348; transformer.py:138-141; pretrain_cmt.py:38-41) and their autograd
 * backward GEMMs.
 * ------------------------------------------------------------------------------------------- */
typedef struct bb_gemm_args {
  const void* A; /* bf16 */
  const void* B; /* bf16 */
  void* D;       /* bf16 or f32 */
  int32_t M, N, K;
  int32_t nb1, nb2; /* batch grid; batch index b = (b1, b2) */
  int32_t a_mn;     /* 0: A is K-major (row-major M x K); 1: A is MN-major (stored K x M) */
  int32_t b_mn;     /* 0: B is K-major (row-major N x K); 1: B is MN-major (stored K x N) */
  int64_t lda, a_s1, a_s2;
  int64_t ldb, b_s1, b_s2;
  int64_t ldd, d_s1, d_s2; /* output row stride and batch strides (elements of the output dtype) */
  int32_t out_f32;         /* 0: bf16 output, 1: fp32 output */
  int32_t accumulate;      /* 1: D += result with fp32 atomics (needs out_f32); implied by split_k>1 */
  int32_t split_k;         /* >=1; >1 splits K across CTAs (D must be zeroed / hold the addend) */
  float alpha;
  const float* bias; /* [N] or NULL; added before the activation */
  int32_t act;       /* 0 none, 1 exact-erf GELU, 2 ReLU */
  void* aux_out;     /* bf16, same strides as D: pre-activation (alpha*acc+bias) or NULL */
  const void* aux_in; /* bf16, same strides as D, or NULL */
  int32_t epi_mul;   /* 0 none; 1: result *= gelu'(aux_in); 2: result *= (aux_in > 0) */
  uint64_t drop_seed;  /* inverted dropout on the result (after act / epi_mul, before add_in); */
  uint32_t drop_thresh; /*   keep iff rng(seed, output element offset) >= thresh; 0 = no dropout   */
  float drop_scale;     /*   1/(1-p)                                                              */
  const void* add_in; /* bf16, same strides as D, or NULL: result += add_in (last) */
  int32_t block_n;   /* 0 = pick automatically; else a tile-width hint (16..256, multiple of 16, of 64 when b_mn): <= 64 selects 64-wide N tiles, larger 128-wide */
} bb_gemm_args;

int bb_gemm_bf16(const bb_gemm_args* args, void* stream);
/* High-precision VERIFICATION arm (csrc/gemm_f32.cu + the float instantiations of every row kernel): after
 * bb_set_act_f32(1) every "bf16" activation pointer of this header (GEMM operands / outputs, row-kernel inputs and
 * outputs, P / dS of the unfused attention sequence) is interpreted as fp32 and bb_gemm_bf16 runs an fp32 CUDA-core
 * GEMM with the same epilogue semantics.  The fused attention cores (bb_flash_*, bb_attn_scores) and the native
 * sub-layer executors (bb_attn_*, bb_ffn_*, bb_pano_*) are bf16-only: the caller composes the unfused kernels instead.
 * Used by the parity tests to hold the model to 1e-3 against the fp32 oracle (north_star); process-wide, default 0.
 * Returns the previous mode. */
int bb_set_act_f32(int on);
int bb_get_act_f32(void);
/* Optional measurement hook (bench.py roofline): the caller registers a device buffer of 2 x capacity 64-bit words
 * (starts initialised to ~0, ends to 0); while profiling is enabled every bb_gemm_bf16 launch gets the next slot and its
 * CTAs stamp %globaltimer into it (min of the starts, max of the ends): the kernel's own execution span, with no events
 * between launches (programmatic dependent launch and CUDA-graph capture stay intact; a graph replay re-stamps the slots
 * of the launches it contains).  bb_gemm_profile(1) resets the slot counter and starts, (0) stops; _count() = launches
 * recorded; _read(i, &ms, dims) copies slot i back (synchronous) and returns its span and (M, N, K, batches, a_mn, b_mn). */
int bb_gemm_profile_buffer(unsigned long long* device_buf, int64_t capacity_launches);
/* Debug: when device_buf is not NULL every bb_gemm_bf16 launch writes, per CTA c and local tile i < 16, four
 * %globaltimer stamps at device_buf[(c*16+i)*4 + {0: MMA issue start, 1: MMA issue end, 2: epilogue start, 3: end}]. */
int bb_gemm_trace(long long* device_buf);
int bb_gemm_profile(int enable);
int64_t bb_gemm_profile_count(void);
int bb_gemm_profile_read(int64_t idx, float* ms, int64_t* dims6);

/* ---------------------------------------------------------------------------------------------
 * BEV lifting (pretrain_src/model/pretrain_cmt.py:114-137 + bev_utils.py:349-378, 381-406).
 * depths: f32 (B, V, Hf, Wf) stored units (x depth_scale inside, reference uses x10);
 * T_c2w f32 (B, V, 4, 4); S_w2c f32 (B, 3); T_w2c f32 (B, 4, 4).
 * cell_idx: int32 (B, V*Hf*Wf): D*z+x of the BEV cell, or -1 when the point is dropped
 *           (no depth / outside the map / above the z clip).  Integer path is bit-exact with the oracle.
 * pc_out: optional f32 (B, V*Hf*Wf, 3) ego-frame point cloud (for tests), may be NULL.
 * ------------------------------------------------------------------------------------------- */
int bb_bev_lift_index(const float* depths, const float* T_c2w, const float* S_w2c, const float* T_w2c, int B, int V,
                      int Hf, int Wf, float depth_scale, float fx, float fy, float cx, float cy, int map_dim,
                      float map_res, float y_clip, int32_t* cell_idx, float* pc_out, void* stream);

/* Cell index of a ready-made ego-frame point cloud (PointCloud.project_bev, pretrain_src/model/bev_utils.py:381-406,
 * map_nav_src/models/bev_utils.py:382-401): pc f32 (npoints, 3), no_depth u8 (npoints) or NULL -> cell_idx int32
 * (npoints): D*round(z/res + (D-1)/2) + round(x/res + (D-1)/2) (round half to even), -1 when the point has no depth,
 * falls outside the map or lies above y_clip. */
int bb_bev_cell_index(const float* pc, const uint8_t* no_depth, int64_t npoints, int map_dim, float map_res, float y_clip,
                      int32_t* cell_idx, void* stream);

/* Scatter-mean pool of point features into BEV cells (torch_scatter.scatter_mean call sites
 * bev_utils.py:407-410): feats f32 (B, P, C) -> bev f32 (B, D*D, C) and/or bev_bf16; deterministic
 * (points of a cell are summed in ascending point order). ob_mask u8 (B, D*D) = !(max==0 && min==0)
 * (bev_utils.py:412). counts int32 (B, D*D). Any of bev_f32 / bev_bf16 / ob_mask / counts may be NULL. */
int bb_bev_scatter_mean_f32(const float* feats, const int32_t* cell_idx, int B, int P, int C, int ncell,
                            float* bev_f32, void* bev_bf16, uint8_t* ob_mask, int32_t* counts, void* stream);
/* Same with bf16 point features (16-bit wire format of the grid features; sums and the mean stay fp32). */
int bb_bev_scatter_mean_bf16(const void* feats_bf16, const int32_t* cell_idx, int B, int P, int C, int ncell,
                             float* bev_f32, void* bev_bf16, uint8_t* ob_mask, int32_t* counts, void* stream);
/* Same for the float64 semantic one-hots (bev_utils.py:417-423): mean, then sem>0 -> 1,
 * sem_mask u8 (B, D*D) = (sum over classes > 0). */
int bb_bev_scatter_sem_f64(const double* sems, const int32_t* cell_idx, int B, int P, int S, int ncell,
                           double* bev_sem, uint8_t* sem_mask, void* stream);
/* Same result from the labels as stored on disk: sem_ids u8 (B, P) class ids in [0, S) (the one-hot expansion of
 * pretrain_src/data/dataset.py:402 never leaves the host).  bev_sem f64 (B, D*D, S) in {0, 1}, sem_mask u8 (B, D*D). */
int bb_bev_scatter_sem_u8(const uint8_t* sem_ids, const int32_t* cell_idx, int B, int P, int S, int ncell, double* bev_sem,
                          uint8_t* sem_mask, void* stream);

/* Agent-side BEV straight from the per-node point clouds of the navigation graph (map_nav_src/r2r/agent.py:293-337:
 * GraphMap.gather_node_pc -> pad_sequence -> splat -> project_bev, without the concatenation and padding copies).
 * One row per node (32 bytes): world-frame points f32 (n, 3), no-depth mask u8/bool (n) or NULL, features (n, C) f32 or
 * bf16 (feat_bf16 = 1; rows 16- resp. 8-byte aligned), n >= 0.  Sample b takes the nodes sample_nodes[b] ..
 * sample_nodes[b+1]-1 (B+1 non-decreasing offsets) in that order, the order the reference concatenates them; a node
 * may appear in several samples.  Per point: p = pc - S_w2c[b], e_j = ((p0 E_j0 + p1 E_j1) + p2 E_j2) + E_j3 with
 * E = T_w2c[b] (4x4 row major), one rounding per operation; the cell index of bb_bev_cell_index; then the
 * scatter-mean of bb_bev_scatter_mean_f32 over the concatenated cloud (points of a cell added in ascending
 * concatenated order, no atomics, no limit on the points per sample).  bev f32 (B, D*D, C), ob_mask u8 (B, D*D);
 * a sample without nodes gives zeros and a false mask.
 * nodes and sample_nodes are HOST arrays: they are validated, then copied on `stream` into table_dev (device,
 * 8-byte aligned, n_nodes*32 + (B+1)*4 bytes: the rows, then the offsets), which the kernel reads.  From pinned memory
 * the copy is asynchronous and the host arrays must stay unchanged until the stream has executed it. */
typedef struct bb_bev_node {
  const float* pc;
  const uint8_t* no_depth;
  const void* feat;
  int64_t n;
} bb_bev_node;
int bb_bev_splat_nodes(const bb_bev_node* nodes, int n_nodes, const int32_t* sample_nodes, int B, void* table_dev,
                       const float* S_w2c, const float* T_w2c, int C, int feat_bf16, int map_dim, float map_res,
                       float y_clip, float* bev, uint8_t* ob_mask, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Row kernels (coalesced, vectorised, warp reductions; fp32 math, bf16 storage).
 * Every row-matrix and vector pointer of the entry points below that read or write 16-byte vectors (LayerNorm forward /
 * backward, bb_add_rows, bb_gather_rows_bf16, bb_segment_wsum / _bwd, bb_embed_sum, bb_colsum_bf16 when ld % 8 == 0,
 * the casts, bb_scatter_rows_sorted) must be 16-byte aligned; a misaligned one is rejected with an error, nothing runs.
 * ------------------------------------------------------------------------------------------- */
/* f32 -> bf16 cast with optional inverted dropout (nn.Dropout on inputs, pretrain_cmt.py:102-106).
 * drop_thresh = p * 2^32 (0 = no dropout); scale = 1/(1-p). Element index is the RNG counter. */
int bb_cast_f32_bf16(const float* src, void* dst, int64_t n, uint64_t seed, uint32_t drop_thresh, float scale,
                     void* stream);
int bb_cast_bf16_f32(const void* src, float* dst, int64_t n, void* stream);

/* y = LayerNorm( dropout(x) + residual ) * gamma + beta, optional output dropout
 * (BertSelfOutput / BertOutput vilmodel.py:150-154,189-193; BertEmbeddings :75-76; nn.LayerNorm sites).
 * x bf16 or f32 (rows, H); residual bf16 or NULL; y bf16; y_f32 optional f32 copy; mean/rstd f32 (rows)
 * saved for backward. H % 8 == 0, H <= 1024. */
int bb_layernorm_fwd(const void* x, int x_f32, const void* residual, const float* gamma, const float* beta,
                     float eps, int64_t rows, int H, uint64_t seed_in, uint32_t thresh_in, float scale_in,
                     uint64_t seed_out, uint32_t thresh_out, float scale_out, void* y, float* y_f32, float* mean,
                     float* rstd, void* stream);
/* Backward of the above. dy bf16 (or f32 when dy_f32); recomputes z = dropout(x)+residual.
 * Outputs: dx (bf16, grad wrt x, dropout mask applied) or NULL; dres (bf16, grad wrt residual) or NULL;
 * dgamma/dbeta f32 [H] are ACCUMULATED into (atomics) — caller zeroes them.  dxsum f32 [H] (optional) += column
 * sums of dx: the bias gradient of the dense layer that produced x, without a separate pass. */
int bb_layernorm_bwd(const void* dy, int dy_f32, const void* x, int x_f32, const void* residual, const float* gamma,
                     const float* mean, const float* rstd, int64_t rows, int H, uint64_t seed_in, uint32_t thresh_in,
                     float scale_in, uint64_t seed_out, uint32_t thresh_out, float scale_out, void* dx, int dx_f32,
                     void* dres, float* dgamma, float* dbeta, float* dxsum, void* stream);

/* Column sums of a bf16 (rows, N) matrix with row stride ld accumulated into f32 out[N] (bias gradients). */
int bb_colsum_bf16(const void* x, int64_t rows, int N, int64_t ld, float* out, void* stream);

/* Masked softmax over the last dim (vilmodel.py:117-127, 335-346; transformer.py MHA):
 * scores f32 (nbatch, H, nq, ld) already scaled; kmask f32 (nbatch, nk) additive (0 / -10000 / -inf) or NULL;
 * bias f32 (nbatch, nq, nk) additive, shared by heads (graph_sprels, vilmodel.py:391-392) or NULL.
 * probs bf16 (same layout); probs_drop bf16 = dropout(probs) when thresh != 0 (else may be NULL).
 * Columns [nk, ld) of the outputs are written as zeros. */
int bb_softmax_fwd(const float* scores, const float* kmask, const float* bias, int nbatch, int H, int nq, int nk,
                   int ld, uint64_t seed, uint32_t thresh, float scale, void* probs, void* probs_drop, void* stream);
/* dS = P * (dPd*keep*scale - sum_k(P * dPd*keep*scale)) * out_scale ; dP f32 (.., ld) wrt dropped probs;
 * ds bf16; optional dbias f32 (nbatch, nq, nk) += sum over heads (atomics, caller zeroes). */
int bb_softmax_bwd(const void* probs, const float* dprobs, int nbatch, int H, int nq, int nk, int ld, uint64_t seed,
                   uint32_t thresh, float scale, float out_scale, void* ds, float* dbias, void* stream);

/* Text embeddings: out f32 (ntok, H) = word[ids] + pos[tok % L] + type[0] (vilmodel.py:62-74; the LayerNorm
 * that follows is bb_layernorm_fwd with x_f32=1). Backward scatters dz f32 (ntok, H) into the three
 * embedding-table gradients with f32 atomics; rows with id == padding_idx get no word gradient
 * (nn.Embedding(padding_idx=0), vilmodel.py:53). Any of dword/dpos/dtype0 may be NULL. */
int bb_embed_sum(const int64_t* ids, const float* word, const float* pos, const float* type0, int64_t ntok, int L,
                 int H, float* out, void* stream);
int bb_embed_scatter_grad(const int64_t* ids, const float* dz, int64_t ntok, int L, int H, int64_t padding_idx,
                          float* dword, float* dpos, float* dtype0, void* stream);

/* out[r, :] = in[idx[r], :] (bf16 rows of width H); idx < 0 writes zeros. And the adjoint
 * out[idx[r], :] += in[r, :] in f32. */
int bb_gather_rows_bf16(const void* in, const int64_t* idx, int64_t nout, int H, void* out, void* stream);
int bb_scatter_add_rows(const void* in_bf16, const int64_t* idx, int64_t nin, int H, float* out_f32, void* stream);
/* Deterministic scatter-add by destination.  dst_sorted (n,) is sorted ascending and stable, so entries with the same
 * destination keep ascending source order; for each run of entries e1 < e2 < ... with dst_sorted == d >= 0:
 *   out_f32[d, :] += ((t_e1 + t_e2) + ...),   t_e = w[e] * src[src_row[e], :]  (one rounded fp32 product, no FMA),
 * or t_e = src[src_row[e], :] when w is NULL; entries with dst_sorted < 0 are dropped.  src is f32 (src_f32 = 1) or
 * the activation type, rows of width H (a multiple of 8); src and out 16-byte aligned.  With a stable sort of the
 * destinations, this is the deterministic form of bb_scatter_add_rows, bb_segment_wsum_bwd and the word-table gradient
 * of bb_embed_scatter_grad. */
int bb_scatter_rows_sorted(const void* src, int src_f32, const int64_t* src_row, const float* w,
                           const int64_t* dst_sorted, int64_t n, int H, float* out_f32, void* stream);

/* bf16 -> bf16 inverted dropout with the same counter-based RNG as everywhere else (element index = counter):
 * regenerates a forward mask in backward.  src may equal dst. */
int bb_dropout_bf16(const void* src, void* dst, int64_t n, uint64_t seed, uint32_t thresh, float scale, void* stream);
/* out[r,:] = a[r,:] (+ b[r,:]) (+ table[idx[r],:]) (+ vec[:]) ; a,b,out bf16 (rows,H); table,vec f32; idx int64.
 * (embedding sums of vilmodel.py:521-524, 590-592, 675-677). b/table/idx/vec may be NULL. */
int bb_add_rows(const void* a, const void* b, const float* table, const int64_t* idx, const float* vec, int64_t rows,
                int H, void* out, void* stream);
/* in-place x[r,:] *= g[r] on a bf16 (rows, ld) matrix. */
int bb_scale_rows_bf16(void* x, const float* g, int64_t rows, int64_t ld, void* stream);
/* Segment weighted sum (vilmodel.py:632-666 _aggregate_gmap_features, host loops turned into CSR lists):
 * out[s,:] = sum_{e in [seg_off[s], seg_off[s+1])} w[e] * src[idx[e],:]  (src,out bf16; f32 accumulate).
 * Backward: dsrc_f32[idx[e],:] += w[e] * dout[s,:] (atomics; caller zeroes dsrc). */
int bb_segment_wsum(const void* src, const int32_t* seg_off, const int32_t* idx, const float* w, int64_t nseg, int H,
                    void* out, void* stream);
int bb_segment_wsum_bwd(const void* dout, const int32_t* seg_off, const int32_t* idx, const float* w, int64_t nseg,
                        int H, float* dsrc_f32, void* stream);

/* out = dy * f'(aux): mode 1 = exact-erf GELU derivative at aux (pre-activation), mode 2 = (aux > 0) (ReLU). */
int bb_act_bwd_bf16(const void* dy, const void* aux, int mode, void* out, int64_t n, void* stream);

/* Generic small elementwise helpers on bf16 tensors. */
int bb_add_bf16(const void* a, const void* b, void* out, int64_t n, void* stream);       /* out = a + b */
int bb_axpy_f32_from_bf16(const void* x, float* y, int64_t n, void* stream);             /* y += x */

/* Fused softmax cross-entropy over logits f32 (rows, ld) with V valid columns (pretrain_cmt.py:259):
 * loss[r] = logsumexp - logit[label]; dlogits (bf16, same ld) = (softmax - onehot) * gscale[r] (may be NULL).
 * label < 0 -> loss 0, zero gradient. */
int bb_softmax_xent(const float* logits, const int64_t* labels, int64_t rows, int V, int64_t ld, float* loss,
                    const float* gscale, void* dlogits, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused attention scores (keys per row <= 512, head dim 64): the 128 x nk product of one (sample, head, query
 * tile) is formed by wgmma in registers, 64 keys at a time, and the row softmax / softmax-backward runs on the
 * accumulators; no fp32 score matrix in HBM.  A = Q (mode 0) or dO (mode 1): element (b,h,q,d) at A + b*a_s2 + h*a_s1 + q*lda + d;
 * Bm = K (mode 0) or V (mode 1) likewise with nk rows.  P / Pd / Pin / dS are bf16 (B,H,nq,ldp).
 *   mode 0: P = softmax(alpha*A Bm^T + kmask + bias), Pd = dropout(P) (Pd may be NULL)
 *   mode 1: dS = Pin o (g - sum_k Pin g) * out_scale with g = dropout-mask(A Bm^T); dbias (B,nq,nk) f32 += unscaled
 * Same dropout counters as bb_softmax_fwd/bwd (vilmodel.py:117-127, 335-346).
 * ------------------------------------------------------------------------------------------- */
typedef struct bb_attn_scores_args {
  const void* A; int64_t lda, a_s1, a_s2;
  const void* Bm; int64_t ldb, b_s1, b_s2;
  int32_t B, H, nq, nk, ldp, mode;
  float alpha, out_scale;
  const float* kmask; const float* bias;
  uint64_t seed; uint32_t thresh; float scale;
  void* P; void* Pd;
  const void* Pin; void* dS; float* dbias;
} bb_attn_scores_args;
int bb_attn_scores(const bb_attn_scores_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fused attention core, head dim 64 (csrc/attn_flash.cu): O = dropout(softmax(alpha Q K^T + kmask + bias)) V for
 * B x H independent (sample, head) problems without materialising scores or probabilities in HBM
 * (vilmodel.py:103-154 BertSelfAttention, 325-363 BertOutAttention; transformer.py:170-182 panorama encoder).
 * Element (b, row, h, d) of q / k / v / o / dout / dq / dk / dv is at  ptr + b*X_bs + row*ldX + h*64 + d  (bf16), so
 * per-head views into packed Q|K|V buffers need no copies.  q / k / v / o / dout / dq / dk / dv must be 16-byte aligned
 * and every row stride ld* and batch stride *_bs a multiple of 8 elements; other calls are rejected.  kmask (B,nk) and bias (B,nq,nk) are additive fp32
 * (may be NULL); lse (B,H,nq) receives the row log-sum-exp (log2 domain) and is the only tensor saved for backward
 * besides o; rows whose keys are all -inf give zeros.  Dropout: element (b,h,q,k) is kept iff a 16-bit half of
 * mix(hash(seed, (b*H+h)*nq+q), k/2) is >= thresh >> 16 (one row hash, one mix per pair of adjacent keys); kept
 * values are scaled by `scale`; backward replays the same mask.
 * bb_flash_bwd: dsum (B,H,nq) is scratch; dq / dk / dv are overwritten; dbias (B,nq,nk) f32 is accumulated (+=,
 * summed over heads) when not NULL.
 * ------------------------------------------------------------------------------------------- */
typedef struct bb_flash_args {
  const void* q; const void* k; const void* v; void* o;
  int64_t q_bs, k_bs, v_bs, o_bs;
  int32_t ldq, ldk, ldv, ldo;
  int32_t B, H, nq, nk, dh;
  float alpha;
  const float* kmask; const float* bias;
  float* lse;
  uint64_t seed; uint32_t thresh; float scale;
  /* backward only */
  const void* dout; int64_t do_bs; int32_t lddo; int32_t pad0_;
  float* dsum;
  void* dq; void* dk; void* dv;
  int64_t dq_bs, dk_bs, dv_bs;
  int32_t lddq, lddk, lddv; int32_t pad1_;
  float* dbias;
} bb_flash_args;
int bb_flash_fwd(const bb_flash_args* args, void* stream);
/* Which core serves bb_flash_fwd / bb_flash_bwd: 0 = always the warp-level mma.sync kernels (csrc/attn_flash.cu),
 * 1 (default, or env BB_ATTN_TC) = the wgmma / TMA kernels (csrc/attn_tc.cu) when nk >= 64 and bias == NULL,
 * 2 = the wgmma kernels whenever they support the call (any nk; tests).  Returns the previous mode. */
int bb_set_attn_tc(int mode);
/* Kept for ABI compatibility: accepts and ignores a trace buffer (the wgmma attention kernels record no trace). */
int bb_attn_tc_trace(long long* device_buf);
int bb_flash_bwd(const bb_flash_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Native sub-layer executors: ONE call enqueues the whole kernel sequence of a sub-layer on `stream`.
 *   attention sub-layer = LN(dropout(dense(attention(x, c))) + x)     (vilmodel.py:103-166, 325-363)
 *   FFN sub-layer       = LN(dropout(W2 gelu(W1 a + b1) + b2) + a)     (vilmodel.py:168-193)
 * The caller provides a forward workspace `ws` (kept until backward) and a backward scratch `gws`, sized by
 * bb_*_ws_bytes; parameter-gradient buffers are fp32, zero-filled by the caller and accumulated into.
 * Weights are bf16 (out,in) row-major; self-attention uses the row-stacked Q|K|V weight (3Hd,Hd) in w_qkv,
 * cross-attention Wq in w_qkv and the stacked K|V weight (2Hd,Hd) in w_kv.
 * ------------------------------------------------------------------------------------------- */
/* Optional: the backward executors (bb_attn_bwd / bb_ffn_bwd / bb_pano_bwd) launch their weight-gradient GEMMs and
 * bias column sums on `side_stream` (forked from the caller's stream with an event each time) so that they overlap the
 * dX chain.  The caller must (1) keep every buffer of a backward call (workspaces, dy, the forward workspace) alive
 * until it has called bb_side_join(stream), which makes `stream` wait for the side stream, and (2) join before anything
 * reads the parameter gradients.  NULL (default) = everything on the caller's stream. */
int bb_set_side_stream(void* side_stream);
int bb_side_join(void* stream);

typedef struct bb_attn_desc {
  int32_t B, nq, nk, Hd, heads;
  int32_t cross;      /* 0: self-attention (c unused, nk == nq), 1: cross-attention over context c */
  int32_t want_dbias; /* backward: accumulate d(bias) (graph bias of the global map encoder) */
  float eps;
  const void* x;      /* (B*nq, Hd) bf16 queries / residual */
  const void* c;      /* (B*nk, Hd) bf16 context or NULL */
  const float* kmask; /* (B, nk) additive key mask or NULL */
  const float* bias;  /* (B, nq, nk) additive bias shared by heads or NULL */
  const void* w_qkv; const void* w_kv; const void* w_o;
  const float* b_qkv; const float* b_kv; const float* b_o; const float* gamma; const float* beta;
  uint64_t seed_attn; uint32_t th_attn; float sc_attn; /* attention-probability dropout */
  uint64_t seed_h; uint32_t th_h; float sc_h;          /* hidden dropout before the residual add */
  void* ws;  /* forward workspace */
  void* y;   /* (B*nq, Hd) bf16 output */
  /* backward only */
  const void* dy; void* gws; void* dx; void* dc;
  float* dw_qkv; float* db_qkv; float* dw_kv; float* db_kv; float* dw_o; float* db_o; float* dgamma; float* dbeta;
  float* dbias;
} bb_attn_desc;
int bb_attn_ws_bytes(const bb_attn_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes);
int bb_attn_fwd(const bb_attn_desc* d, void* stream);
int bb_attn_bwd(const bb_attn_desc* d, void* stream);

typedef struct bb_ffn_desc {
  int64_t M;          /* rows (tokens) */
  int32_t Hd, Fd;     /* hidden and intermediate sizes */
  float eps;
  const void* a;      /* (M, Hd) bf16 input / residual */
  const void* w1; const void* w2; const float* b1; const float* b2; const float* gamma; const float* beta;
  uint64_t seed_h; uint32_t th_h; float sc_h;
  void* ws; void* y;
  /* backward only */
  const void* dy; void* gws; void* da;
  float* dw1; float* db1; float* dw2; float* db2; float* dgamma; float* dbeta;
} bb_ffn_desc;
int bb_ffn_ws_bytes(const bb_ffn_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes);
int bb_ffn_fwd(const bb_ffn_desc* d, void* stream);
int bb_ffn_bwd(const bb_ffn_desc* d, void* stream);

/* Pre-norm panorama encoder layer (transformer.py:170-182 with nn.MultiheadAttention's packed in_proj):
 *   x1 = x + drop(out_proj(attention(LN1(x))));  y = x1 + drop(W2 drop(gelu(W1 LN2(x1) + b1)) + b2)
 * x, y (N*V, Hd) bf16; kmask (N, V) additive (-inf on padding); LayerNorm eps fixed at 1e-5 like nn.LayerNorm. */
typedef struct bb_pano_desc {
  int32_t N, V, Hd, heads, Fd;
  int32_t pad_;
  const void* x; const float* kmask;
  const void* w_in; const void* w_out; const void* w1; const void* w2;
  const float* b_in; const float* b_out; const float* b1; const float* b2;
  const float* g1; const float* be1; const float* g2; const float* be2;
  uint64_t seed_attn; uint32_t th_attn; float sc_attn;
  uint64_t seed1; uint64_t seed2; uint64_t seed3; uint32_t th_h; float sc_h;
  void* ws; void* y;
  /* backward only */
  const void* dy; void* gws; void* dx;
  float* dw_in; float* db_in; float* dw_out; float* db_out; float* dw1; float* db1; float* dw2; float* db2;
  float* dg1; float* dbe1; float* dg2; float* dbe2;
} bb_pano_desc;
int bb_pano_ws_bytes(const bb_pano_desc* d, int64_t* fwd_bytes, int64_t* bwd_bytes);
int bb_pano_fwd(const bb_pano_desc* d, void* stream);
int bb_pano_bwd(const bb_pano_desc* d, void* stream);


/* ---------------------------------------------------------------------------------------------
 * Multi-tensor optimizer step on a DEVICE table of tensors (csrc/optim.cu): one launch for all parameters.
 * Replaces the per-tensor python loop of pretrain_src/optim/adamw.py:53-112 (AdamW.step: eps inside the sqrt
 * denominator sum, bias-corrected step size, decoupled weight decay applied AFTER the Adam update) and
 * torch.nn.utils.clip_grad_norm_ at pretrain_src/train_r2r.py:295-300.
 * A tensor occupies ceil(n / bb_mt_chunk_elems()) consecutive chunks starting at chunk0; the table is sorted by
 * chunk0 and chunk0 of entry 0 is 0.  step_size = lr * sqrt(1-beta2^t) / (1-beta1^t) (or lr when correct_bias is
 * off), decay = lr * weight_decay, both per tensor because each parameter has its own step counter t.
 * ------------------------------------------------------------------------------------------- */
typedef struct bb_mt_tensor {
  float* p;        /* fp32 parameter (bb_adamw_step: updated in place; bb_mt_cast_bf16: source) */
  const float* g;  /* fp32 gradient (bb_mt_sumsq, bb_adamw_step) */
  float* m;        /* exp_avg */
  float* v;        /* exp_avg_sq */
  void* p16;       /* bf16 shadow of p, written after the update (may be NULL in bb_adamw_step) */
  int64_t n;       /* elements */
  float step_size;
  float decay;
  int64_t chunk0;
} bb_mt_tensor;
int bb_mt_chunk_elems(void);
/* *out = sum over all tensors of sum(g^2)  (zeroed on the stream first; fp32 atomics across CTAs) */
int bb_mt_sumsq(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, float* out, void* stream);
/* g' = g * grad_scale * min(1, max_norm / (grad_scale*sqrt(*sumsq) + 1e-6))   (no clipping when sumsq == NULL or
 * max_norm <= 0); m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; p -= step_size * m / (sqrt(v) + eps); p -= decay * p;
 * p16 = bf16(p).  No host synchronisation: the norm is read on the device. */
int bb_adamw_step(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, float beta1, float beta2, float eps,
                  const float* sumsq, float max_norm, float grad_scale, void* stream);
/* p16 = bf16(p) for every table entry (refresh of the bf16 weight shadows in one launch). */
int bb_mt_cast_bf16(const bb_mt_tensor* table_dev, int ntensors, int64_t total_chunks, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BEVBERT_B200_H */
