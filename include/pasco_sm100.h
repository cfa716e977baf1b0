/* pasco_sm100.h — C ABI of libpasco_sm100.so, the sm_90a sparse-voxel engine that sits
 * underneath PaSCo's operator surface.
 *
 * Every entry point replaces one granule of the MinkowskiEngine 0.5.4 pybind backend
 * (`MinkowskiEngineBackend._C`, not vendored in /root/reference) that the reference reaches
 * through `import MinkowskiEngine as ME`; the reference call site each one serves is cited
 * as pasco/<file>:<line> (paths relative to /root/reference).
 *
 * Conventions
 *   - plain C types, raw DEVICE pointers; inputs and outputs are caller-owned memory;
 *   - scratch a call needs for itself comes from a stream-ordered memory pool of the library's own and is released
 *     on the call's stream; the one exception is the split-K convolution, whose caller passes its workspace
 *     (pasco_conv_splitk_workspace_bytes also tells the caller whether a shape is split at all);
 *   - every call takes the CUDA stream to launch on (pass torch's current stream);
 *   - returns 0 on success, negative on error; pasco_last_error() gives the message of the
 *     last failure on the calling thread;
 *   - coordinates are int32 rows (b, x, y, z), each component in [-32768, 32767];
 *   - features are row-major float32 [N, C]; row indices are int32, −1 == "no row";
 *   - a neighbour table `nbr` is int32 [K, N_out]: nbr[k*N_out + o] = input row feeding
 *     output row o through kernel offset k, or −1.  Offsets enumerate x fastest; odd kernel
 *     sizes are centred, even ones span [0, k)·stride  (ME convention, SURVEY.md §8b).
 */
#ifndef PASCO_SM100_H_
#define PASCO_SM100_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* pasco_stream_t; /* cudaStream_t */

const char* pasco_last_error(void);
int pasco_abi_version(void);
/* fills sm count / smem per block opt-in / compute capability major*10+minor of the current device */
int pasco_device_info(int* sm_count, int* smem_optin, int* cc);

/* ---- coordinate maps (ME CoordinateMapManager::insert_and_map / stride / kernel_map) ----
 * Hash table = open addressing over `capacity` (power of two ≥ 2N) slots:
 *   table_keys  uint64[capacity]  (caller fills with 0xFF bytes before the first insert)
 *   table_vals  int32 [capacity]  (caller fills with 0x7F bytes)                            */

/* ME.SparseTensor(F, C) — pasco/models/net_panoptic_sparse.py:323, unet3d_sparse_v2.py:207.
 * Inserts n rows; on return table_vals[slot(key)] = smallest row index holding that key and
 * first_row[i] = that winning row for input row i (first_row[i]==i ⇔ row i is kept).
 * Keys pack 16 bits per component: a coordinate or batch index outside [-32768, 32767] sets *err_flag = 2 on the
 * device (err_flag may be NULL) and the host wrapper raises; MinkowskiEngine accepts the full int32 range.          */
int pasco_hash_insert(const int32_t* coords, int64_t n, uint64_t* table_keys, int32_t* table_vals,
                      int64_t capacity, int32_t* first_row, int32_t* err_flag, pasco_stream_t s);

/* After compaction: rewrite table values old_row → new_row[old_row] (new_row[i] = −1 for dropped rows). */
int pasco_hash_remap(int32_t* table_vals, int64_t capacity, const int32_t* new_row, pasco_stream_t s);

/* row of each query coordinate (−1 if absent) — union map (decoder_v3.py:163) and tests */
int pasco_hash_lookup(const int32_t* query, int64_t nq, const uint64_t* table_keys, const int32_t* table_vals,
                      int64_t capacity, int32_t* out_row, pasco_stream_t s);

/* out[i] = (b, floor(x/s)*s, ...) — ME stride map for k=2,s=2 convs (pasco/maskpls/mink.py:509-511)
 * and max-pool (transformer_predictor_v2.py:100-102).  Floors toward −inf.                     */
int pasco_coords_floor(const int32_t* coords, int64_t n, int32_t sx, int32_t sy, int32_t sz, int32_t* out,
                       pasco_stream_t s);

/* generative transposed conv output coordinates (mink.py:524-527): child row 8*p + k =
 * parent p + offset_k * out_stride, offsets x fastest in {0,1}^3; kernel_size fixed to 2.     */
int pasco_coords_generate_k2(const int32_t* coords, int64_t n, int32_t out_sx, int32_t out_sy, int32_t out_sz,
                             int32_t* out, pasco_stream_t s);

/* nbr[k, o] for an odd kernel (k=3) between an input map (hash table) and output coords:
 * probes out + offset_k*dilation*stride  (every ME.MinkowskiConvolution k=3: mink.py:625-638,
 * decoder_v3.py:267-282).                                                                      */
int pasco_kernel_map_probe(const int32_t* out_coords, int64_t n_out, const uint64_t* table_keys,
                           const int32_t* table_vals, int64_t capacity, int32_t kernel_size, int32_t sx,
                           int32_t sy, int32_t sz, int32_t* nbr, pasco_stream_t s);

/* same for an anisotropic odd box kernel (kx,ky,kz), K = kx*ky*kz offsets x fastest — the dense bottleneck
 * kernels (3,3,1), (5,5,3), (7,7,5) of pasco/models/layers.py:656-702 run as sparse convs over the full
 * stride-8 grid.                                                                                  */
int pasco_kernel_map_box(const int32_t* out_coords, int64_t n_out, const uint64_t* table_keys,
                         const int32_t* table_vals, int64_t capacity, int32_t kx, int32_t ky, int32_t kz,
                         int32_t sx, int32_t sy, int32_t sz, int32_t* nbr, pasco_stream_t s);

/* even kernel == stride (k=2 s=2 conv, k=s max-pool): every child has one parent.
 *   parent_of[i] = row of floor(child_i) in the parent table
 *   slot_of[i]   = kernel offset index of the child inside its parent block (x fastest)
 *   nbr[k, p]    = child row (written when nbr != NULL; K = ks^3 rows of n_parent)              */
int pasco_kernel_map_down(const int32_t* child_coords, int64_t n_child, const uint64_t* table_keys,
                          const int32_t* table_vals, int64_t capacity, int32_t ks, int32_t child_sx,
                          int32_t child_sy, int32_t child_sz, int32_t* parent_of, int32_t* slot_of, int32_t* nbr,
                          int64_t n_parent, pasco_stream_t s);

/* ---- row compaction (ME.MinkowskiPruning: decoder_v3.py:159,421,496; misc.py:17-26) ----------
 * step 1: block_counts[b] = popcount of mask over rows [b*1024, (b+1)*1024)
 * (caller turns counts into exclusive offsets — a length-ceil(n/1024) scan)
 * step 2: new_row[i] = compacted index or −1, kept_rows[new] = i (order preserving)             */
int pasco_mask_block_counts(const uint8_t* mask, int64_t n, int32_t* block_counts, pasco_stream_t s);
int pasco_mask_compact(const uint8_t* mask, int64_t n, const int32_t* block_offsets, int32_t* new_row,
                       int32_t* kept_rows, pasco_stream_t s);

/* out[r, :] = rows[r] >= 0 ? src[rows[r], :] : 0   (row gather; also the backward of scatter) */
int pasco_gather_rows(const float* src, const int32_t* rows, int64_t n_rows, int32_t C, float* out,
                      pasco_stream_t s);
/* dst[rows[r], :] (+)= src[r, :]; rows unique, −1 skipped (union add, decoder_v3.py:163) */
int pasco_scatter_rows(const float* src, const int32_t* rows, int64_t n_rows, int32_t C, float* dst,
                       int32_t accumulate, pasco_stream_t s);
/* same for int32 [N,4] coordinate rows */
int pasco_gather_coords(const int32_t* src, const int32_t* rows, int64_t n_rows, int32_t* out, pasco_stream_t s);

/* ---- dense <-> sparse (SparseTensor.dense / ME.to_sparse: augmenter.py:15-22,
 *      unet3d_sparse_v2.py:196-202, transformer_predictor_v2.py:263-274) ----------------------
 * dense is [B, C, X, Y, Z] float32; cell = (coord - min) / stride.  A row whose cell lies outside the volume is
 * skipped (to_dense) / reads as zero (from_dense) and sets *err_flag = 1 on the device (err_flag may be NULL); the
 * host wrapper raises at its next synchronisation point, where MinkowskiEngine raises immediately.              */
int pasco_to_dense(const float* feats, const int32_t* coords, int64_t n, int32_t C, const int32_t min_c[3],
                   const int32_t stride[3], float* dense, int32_t B, int32_t X, int32_t Y, int32_t Z,
                   int32_t* err_flag, pasco_stream_t s);
int pasco_from_dense(const float* dense, const int32_t* coords, int64_t n, int32_t C, const int32_t min_c[3],
                     const int32_t stride[3], float* feats, int32_t B, int32_t X, int32_t Y, int32_t Z,
                     int32_t* err_flag, pasco_stream_t s);
/* occupancy[b,x,y,z] = (sum_c |dense[b,c,x,y,z]|) != 0  → uint8 mask in (b,x,y,z) order */
int pasco_dense_occupancy(const float* dense, int32_t B, int32_t C, int64_t cells, uint8_t* mask,
                          pasco_stream_t s);

/* ---- sparse convolution (ME ConvolutionForward/Backward: every conv on the path) -------------
 * out[o,:] = sum_k in[nbr[k,o],:] @ W[k]        W: float32 [K, Cin, Cout]
 *
 * Tensor-core path (wgmma, bf16 split operands, fp32 accumulate in registers):
 *   precision 1 = bf16 operands (1 MMA / k-step), 3 = bf16x3 split (hi·hi + lo·hi + hi·lo,
 *   ~2^-16 relative: the "fp32" mode of BASELINE.json configs[1]).
 *   Requires Cin % 16 == 0 (Cin >= 16), Cout % 16 == 0, 16 <= Cout <= 512 (forward, input gradient, planes and weight
 *   gradient alike).  The contraction runs in blocks of 64 channels; a last block past Cin is zero-padded in the
 *   kernels and never read from memory.
 * Weights are first packed into the swizzled shared-memory operand image:
 *   transpose=0: B[n=co][k=ci] = W[k][ci][co]      (forward)
 *   transpose=1: B[n=ci][k=co] = W[k][ci][co]      (input gradient; swap Cin/Cout in the conv call)
 * packed size in bytes = pasco_conv_packed_bytes(K, Cin, Cout): K x Cout x Cin x 4 with the contraction rounded up to
 * a multiple of 64, large enough for either transpose (= K * Cin * Cout * 4 when both are multiples of 64).         */
int64_t pasco_conv_packed_bytes(int32_t K, int32_t Cin, int32_t Cout);
int pasco_conv_pack_weights(const float* W, int32_t K, int32_t Cin, int32_t Cout, int32_t transpose, void* packed,
                            pasco_stream_t s);
/* koff_map (host int32[K] or NULL): packed weight slice used for table row k; must be the identity
 * (NULL) or the reversal K-1-k (mirrored offsets of the input gradient).  K <= 1024.
 * bias: float32[Cout] or NULL.  The input rows are read as they are; a BatchNorm + activation in front of the
 * convolution is fused into pasco_split_planes instead (plane-gather path below).
 * stats: optional float64[2*Cout] accumulating column sum / sum of squares of the output.
 * in_pitch / out_pitch: row strides in floats (0 = Cin / Cout) so that a column block of a wider matrix can be
 * read / written in place — dense Linear layers run as K = 1, nbr = NULL convolutions in column chunks <= 256.  */
int pasco_conv_forward_tc(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out,
                          int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map,
                          const float* bias, double* stats, float* out, int32_t precision, int64_t in_pitch,
                          int64_t out_pitch, pasco_stream_t s);
/* Split-K form of the same convolution for shapes with few output tiles and many offsets (the dense bottleneck of
 * layers.py:646-726 runs as 32 tiles x 245 offsets: one CTA per tile would leave most SMs idle).  The offsets are
 * cut into ranges, every (tile, range) pair is a work item whose partial result goes to the caller's workspace, and a
 * second kernel adds the partials in a fixed order (+ bias) — still deterministic, no atomics.
 * pasco_conv_splitk_workspace_bytes returns 0 when the shape is not worth splitting (then call pasco_conv_forward_tc). */
int64_t pasco_conv_splitk_workspace_bytes(int32_t K, int64_t n_out, int32_t Cout);
int pasco_conv_forward_splitk(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin,
                              int32_t Cout, const void* packed_w, const int32_t* koff_map, const float* bias, float* out,
                              int32_t precision, int64_t in_pitch, int64_t out_pitch, void* workspace,
                              int64_t workspace_bytes, pasco_stream_t s);

/* Plane-gather path (the default for every gathered convolution): the activations are split ONCE per tensor into bf16
 * planes x = hi + lo (lo = NULL for precision 1) by pasco_split_planes — optionally fused with y = act(x*scale + shift),
 * the BatchNorm + activation of the producing layer — and the convolution / weight-gradient producers move plane rows
 * with 16-byte cp.async copies straight into the swizzled operand tiles (missing neighbours are zero-fill copies that touch
 * no memory).  Planes are bf16 [N, C] with a row pitch in ELEMENTS (0 = C); C % 8 == 0.  The convolutions read only the
 * C channels of a row: channels past C up to the next multiple of 64 are zero-fill copies.
 * pasco_conv_forward_planes: forward and input gradient (same contract as pasco_conv_forward_tc: koff_map, bias, fused
 * BatchNorm statistics of `out` in `stats`);  pasco_conv_wgrad_planes: dW (zeroed by the caller) from the planes of the
 * layer input and of the output gradient.                                                                          */
int pasco_split_planes(const float* x, int64_t n, int32_t C, int64_t pitch, const float* scale, const float* shift,
                       int32_t act, void* hi, void* lo, pasco_stream_t s);
int pasco_conv_forward_planes(const void* hi, const void* lo, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out,
                              int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map, const float* bias,
                              double* stats, float* out, int32_t precision, int64_t plane_pitch, int64_t out_pitch,
                              pasco_stream_t s);
/* Inference form of pasco_conv_forward_planes (eval-mode forward without gradients): the same convolution with an
 * epilogue that, per element of row r < n_out and column c,
 *   v = acc + bias[c]
 *   residual != NULL:  v = act_out(residual[r][c] + v)             (a residual block's ReLU(skip + y))
 *   out != NULL:       out[r][c] = v
 *   next_hi != NULL:   z = act_next(v * next_scale[c] + next_shift[c])  (one fused multiply-add; no affine when next_scale
 *                      is NULL), next_hi[r][c] = bf16(z), next_lo[r][c] = bf16(z - hi) (next_lo in precision 3 only)
 * i.e. the next layer's eval-mode BatchNorm + activation written as the planes the next convolution gathers.  The
 * arithmetic is that of pasco_affine_act and pasco_split_planes, so the result is bit for bit the unfused sequence.
 * residual, out and the next planes are contiguous [n_out, Cout]; act_* as in pasco_affine_act (0 none, 1 ReLU,
 * 2 LeakyReLU 0.01).  At least one of out / next_hi is set.  No statistics are computed.                          */
int pasco_conv_forward_planes_infer(const void* hi, const void* lo, int64_t n_in, const int32_t* nbr, int32_t K,
                                    int64_t n_out, int32_t Cin, int32_t Cout, const void* packed_w, const int32_t* koff_map,
                                    const float* bias, const float* residual, int32_t act_out, float* out,
                                    const float* next_scale, const float* next_shift, int32_t act_next, void* next_hi,
                                    void* next_lo, int32_t precision, int64_t plane_pitch, pasco_stream_t s);
int pasco_conv_wgrad_planes(const void* in_hi, const void* in_lo, int64_t n_in, const int32_t* nbr, int32_t K,
                            int64_t n_out, int32_t Cin, int32_t Cout, const void* g_hi, const void* g_lo, float* dW,
                            int32_t precision, int64_t in_pitch, int64_t gout_pitch, pasco_stream_t s);

/* dW[k] = sum_o in[nbr[k,o],:]^T @ gout[o,:]   (wgmma, MN-major operands); dW float32 [K,Cin,Cout] zeroed by caller.
 * Cin % 16 == 0, Cout % 16 == 0, Cout <= 512 (this function and pasco_conv_wgrad_planes).                         */
int pasco_conv_wgrad_tc(const float* in, int64_t n_in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin,
                        int32_t Cout, const float* gout, float* dW, int32_t precision, int64_t in_pitch,
                        int64_t gout_pitch, pasco_stream_t s);

/* CUDA-core fp32 reference path of the same contraction (any Cin/Cout; validation + odd shapes) */
int pasco_conv_forward_simt(const float* in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin,
                            int32_t Cout, const float* W, int32_t w_transposed, const int32_t* koff_map,
                            const float* bias, float* out, pasco_stream_t s);
int pasco_conv_wgrad_simt(const float* in, const int32_t* nbr, int32_t K, int64_t n_out, int32_t Cin, int32_t Cout,
                          const float* gout, float* dW, pasco_stream_t s);

/* ---- pooling / reductions --------------------------------------------------------------------
 * ME.MinkowskiMaxPooling(k=s, stride=s) (transformer_predictor_v2.py:100-102): out rows
 * pre-filled with -inf by the caller; out[parent_of[i], c] = max(...)                            */
int pasco_maxpool_forward(const float* in, const int32_t* parent_of, int64_t n_in, int32_t C, float* out,
                          pasco_stream_t s);
/* torch_scatter.scatter_max(src, index, dim=0) (unet3d_sparse_v2.py:79): out pre-filled with -inf,
 * second pass writes argmax (smallest row attaining the max) and zero-fills empty segments        */
int pasco_scatter_max(const float* src, const int64_t* index, int64_t n, int32_t C, float* out, int64_t n_seg,
                      int64_t* argmax, pasco_stream_t s);

/* ---- BatchNorm over rows (ME.MinkowskiBatchNorm == BatchNorm1d on [N,C]; mink.py:512,623,631) ---
 * stats float64[2*C] (sum, sumsq) zeroed by the caller; apply: y = act(x*scale[c] + shift[c])      */
int pasco_bn_stats(const float* x, int64_t n, int32_t C, double* stats, pasco_stream_t s);
int pasco_affine_act(const float* x, int64_t n, int32_t C, const float* scale, const float* shift, int32_t act,
                     const float* residual, float* y, pasco_stream_t s);
/* per-channel coefficients in one launch each: stats -> scale/shift (+ mean, rstd, running-statistics update);
 * backward sums -> (ca, cb, cc) of dx = ca*dz + cb*x + cc and the gamma/beta gradients (divided by grad_div).
 * count_dev (device double, e.g. the all-reduced SyncBatchNorm row count) overrides `count` when not NULL.       */
int pasco_bn_finalize(const double* stats, const double* count_dev, double count, int32_t C, const float* gamma,
                      const float* beta, float eps, float momentum, float* scale, float* shift, float* mean, float* rstd,
                      float* running_mean, float* running_var, pasco_stream_t s);
int pasco_bn_bwd_coefs(const double* sums, const double* count_dev, double count, int32_t C, const float* gamma,
                       const float* mean, const float* rstd, float grad_div, float* ca, float* cb, float* cc, float* ggamma,
                       float* gbeta, pasco_stream_t s);
/* backward: given dy, x (pre-BN), scale/shift/act → sums float64[2*C] = (Σ dz, Σ dz·x̂·…) and dx */
int pasco_bn_bwd_reduce(const float* dy, const float* x, int64_t n, int32_t C, const float* scale,
                        const float* shift, int32_t act, double* sums, pasco_stream_t s);
int pasco_bn_bwd_apply(const float* dy, const float* x, int64_t n, int32_t C, const float* scale,
                       const float* shift, int32_t act, const float* coef_a, const float* coef_b,
                       const float* coef_c, float* dx, pasco_stream_t s);

/* ---- MaskPLS masked cross-attention (pasco/models/transformer/blocks.py:73-92 with the attention mask of
 *      transformer_predictor_v2.py:220-289): Q queries against all P voxels, H heads of width D <= 64 ----------
 * Any Q >= 1: the kernels work in blocks of 128 queries and stream K and V once per block (Q <= 128 is one block).
 * q [Q, H*D], k / v [P, H*D] float32 (already projected); logits = scale * q.k; mask = bit rows
 * uint32 [Q, 2*ceil(P/64)] (bit j of word 2t + j/32 set = key 64t + j masked) or NULL; out [Q, H*D] is overwritten
 * (the key chunks' shares are summed in a fixed order); lse [H, Q] receives log-sum-exp per row (needed by the
 * backward).  Two streaming passes over K (row statistics, then output), wgmma for both GEMMs, bf16x3 split operands. */
int pasco_xattn_forward(const float* q, const float* k, const float* v, const uint32_t* mask, int32_t Q, int64_t P,
                        int32_t H, int32_t D, float scale, float* out, float* lse, pasco_stream_t s);
/* backward of the above: recomputes the probabilities from lse; dq [Q, H*D] is overwritten (chunk shares, fixed order),
 * dk / dv [P, H*D] are fully overwritten (no atomics; at Q > 128 the query blocks' partials are added in block order,
 * through a workspace of (ceil(Q/128) - 1) * 2 * P * H * D floats from the library's pool).                       */
int pasco_xattn_backward(const float* q, const float* k, const float* v, const uint32_t* mask, const float* lse,
                         const float* out, const float* dout, int32_t Q, int64_t P, int32_t H, int32_t D, float scale,
                         float* dq, float* dk, float* dv, pasco_stream_t s);
/* the attention mask of transformer_predictor_v2.py:220-289 and line 164, built directly as the bit rows above:
 * key v of the P keys is masked for query q unless some scale-1 voxel u in v's stride-s block has logit[u, q] > 0.
 * logits [*, Q] float32 with row pitch ld; voxel u reads logit row rows[u] (NULL: row u) for u < n_child;
 * parent_of [n_child] = u's row among the n_parent stride-s voxels (NULL: identity, n_parent = n_child; −1 skipped);
 * key_parent [P] = key v's row among those n_parent voxels (−1: no voxel, masked).
 * Out: mask uint32 [Q, 2*ceil(P/64)]; keys beyond P masked; a query whose P keys are all masked gets those P bits
 * cleared (it attends everywhere) and keeps its padding bits.  Scratch from the caller, zero-filled: pooled uint32
 * [n_parent, ceil(Q/32)] and seen int32 [Q].  Integer atomicOr only: two calls give identical bits.               */
int pasco_attn_mask_bits(const float* logits, int64_t ld, int32_t Q, const int32_t* rows, int64_t n_child,
                         const int32_t* parent_of, int64_t n_parent, const int32_t* key_parent, int64_t P,
                         uint32_t* pooled, int32_t* seen, uint32_t* mask, pasco_stream_t s);

/* ---- test-time post-processing: the M-subnet ensemble (pasco/models/ensembler.py:20-187, reached from
 *      net_panoptic_sparse.py:245-294) and panoptic inference (pasco/models/helper.py:91-303, reached from
 *      Net.step_inference, net_panoptic_sparse.py:539-648), on sparse rows of the X x Y x Z reference grid -------------
 * A cell is the linear index (x*Y + y)*Z + z; cell maps are int32 [X*Y*Z] holding a row index or −1.                */

/* transform_utils.py:55-76,160-181 (transform + sample_scene): cell_row[cell] = row of the subnet's hash table (keys
 * with batch index 0) at round((T·(cell*0.2 + 0.1 + lo) − lo − 0.1) / 0.2), lo = (0, −25.6, −2), in fp32 with
 * round-half-to-even, or −1; T = rows 0-2 of the 4x4 pose (host float[12], row-major).  cell_mask (NULL allowed)
 * receives cell_row >= 0 as a byte, ready for pasco_mask_block_counts / pasco_mask_compact.                        */
int pasco_pose_lookup(const uint64_t* table_keys, const int32_t* table_vals, int64_t capacity, const float T[12],
                      int32_t X, int32_t Y, int32_t Z, int32_t* cell_row, uint8_t* cell_mask, pasco_stream_t s);
/* mask[i] = 1 where cell_row[i] >= 0, other bytes untouched: the union of row sets (ensembler.py:100-112, 182-186) */
int pasco_cell_mask_or(const int32_t* cell_row, int64_t n, uint8_t* mask, pasco_stream_t s);
/* out[r] = cell_row[lin[r]] */
int pasco_lookup_rows(const int32_t* cell_row, const int32_t* lin, int64_t n, int32_t* out, pasco_stream_t s);
/* Net.step's subnet box (net_panoptic_sparse.py:430-459): every row r of coords int32 [n, 4] (b, x, y, z; b ignored)
 * with lo <= (x, y, z) <= hi sets cell_row[cell] = r at cell (x, y, z) − lo of the X x Y x Z box (cell_row filled with
 * −1 by the caller; hi − lo below the box size) and cell_mask[cell] = 1 (zeroed by the caller); counts int32 [2]
 * (zeroed) += the rows outside [lo, hi], the rows at a cell another row already holds (which row holds it is then
 * unspecified).  Integer atomics only.                                                                             */
int pasco_box_cells(const int32_t* coords, int64_t n, const int32_t lo[3], const int32_t hi[3], int32_t X, int32_t Y,
                    int32_t Z, int32_t* cell_row, uint8_t* cell_mask, int32_t* counts, pasco_stream_t s);

/* ensembler.py:40-58 for the masks: out[r, q] = sigmoid(logits[rows[r], q]) fp32 [n, Q]; optionally (hi != NULL) the
 * bf16 planes hi = bf16(out), lo = bf16(out − hi) [n, Qp], Qp % 16 == 0, columns past Q zero; colsum (NULL allowed)
 * [Q] = column sums, reduced from per-CTA partials in CTA order; nonzero (NULL allowed) [n] = row has a non-zero. */
int pasco_mask_rows_sigmoid(const float* logits, const int32_t* rows, int64_t n, int32_t Q, float* out, void* hi,
                            void* lo, int32_t Qp, float* colsum, uint8_t* nonzero, pasco_stream_t s);
/* ensembler.py:88-129: for output row r at cell lin[r] and column j,
 *   a = A[cell_a[cell], a_col[j]] (0 when there is no anchor row), b likewise from B, cell_b, b_col
 *   v = (b_col != NULL and b_col[j] >= 0) ? (a*weight + b) / (weight + 1) : a,  then v *= gate[cell] when gate != NULL
 * (b may be NULL when the subnet has no row: every b then reads as zero)
 * out fp32 [n, q_out]; planes, colsum and nonzero as in pasco_mask_rows_sigmoid.  The last step of the ensemble passes
 * the kept queries as a_col (the mean-IoU keep) and the ensembled occupancy as gate.                                */
int pasco_mask_merge(const float* a, const int32_t* cell_a, int32_t qa, const float* b, const int32_t* cell_b, int32_t qb,
                     const int32_t* lin, int64_t n, const int32_t* a_col, const int32_t* b_col, int32_t q_out,
                     int32_t weight, const uint8_t* gate, float* out, void* hi, void* lo, int32_t Qp, float* colsum,
                     uint8_t* nonzero, pasco_stream_t s);
/* ensembler.py:166-176: out[r, :] = softmax(logits[rows[r], :]) over K channels */
int pasco_softmax_rows(const float* logits, const int32_t* rows, int64_t n, int32_t K, float* out, pasco_stream_t s);
/* utils.py:153-198 + ensembler.py:78-86: from the intersections inter [Q, pitch] (pasco_conv_wgrad_planes with K = 1)
 * and the column sums, iou = inter / (sum_a + sum_b − inter) (0 where the union is 0); gated [Q, Q] = iou > threshold
 * ? iou : 0 — the matrix the host hands to linear_sum_assignment.                                                   */
int pasco_soft_iou(const float* inter, int32_t Q, int64_t pitch, const float* sum_a, const float* sum_b, float threshold,
                   float* gated, pasco_stream_t s);
/* ensembler.py:160-187 + net_panoptic_sparse.py:278-294 (max_prob): per row r at cell lin[r], the mean over the M <= 8
 * subnets of probs[m][cell_rows[m][cell]] (a subnet without a row there counts as one-hot class 0); pred[r] = its first
 * argmax, conf[r] = its max; gate (NULL allowed) [cells] receives pred != 0 at the cell.  probs / cell_rows are host
 * arrays of device pointers.                                                                                         */
int pasco_sem_ensemble(int32_t M, const float* const probs[], const int32_t* const cell_rows[], const int32_t* lin,
                       int64_t n, int32_t K, int32_t* pred, float* conf, uint8_t* gate, pasco_stream_t s);
/* helper.py:135-186 pass 1 over the mask probabilities probs [n, Q] with class probabilities query_probs [Q, K1]:
 * a query is kept when its first-argmax label is neither 0 nor K1 − 1 and its max > object_mask_threshold; per row,
 * win = (q << 1) | (m_q >= vox_occ_threshold) for the kept q maximising prob_q * m_q (lowest q on ties), −1 without a
 * kept query; m_win = m_q, m_sum = the sum of m over kept queries; c_sum (NULL allowed) = the sum of prob_q * m_q over
 * kept queries.  areas int32 [2Q], zeroed by the caller: [0, Q) the mask_area and [Q, 2Q) the original_area of every
 * query (integer counts).                                                                                           */
int pasco_panoptic_pass1(const float* probs, int64_t n, int32_t Q, const float* query_probs, int32_t K1,
                         float object_mask_threshold, float vox_occ_threshold, int32_t* win, float* m_win, float* m_sum,
                         float* c_sum, int32_t* areas, pasco_stream_t s);
/* helper.py:187-250 on one thread: the walk over kept queries in ascending order (overlap filter mask_area /
 * original_area in double, stuff classes merged into their first segment, sequential ids).  seg_of / cls_of int32 [Q]:
 * the segment id a query paints (0 none) and its semantic class (−1 for merged stuff, which keeps semantic 0).
 * records int32 [1 + 4Q]: the segment count, then per segment (query, class, float bits of the class probability,
 * isthing).  kept (NULL allowed) int32 [1 + Q]: the kept-query count kq, then the kept queries in ascending order.
 * thing_mask bit c = class c is a thing class; K1 <= 65.                                                           */
int pasco_panoptic_segments(const float* query_probs, int32_t Q, int32_t K1, float object_mask_threshold,
                            double overlap_threshold, uint64_t thing_mask, const int32_t* areas, int32_t* seg_of,
                            int32_t* cls_of, int32_t* records, int32_t* kept, pasco_stream_t s);
/* helper.py:236-247 pass 2 from the pass-1 records: panoptic / semantic int32 [n] and the confidence fp32 [n] =
 * m_win / (m_sum + 1e-8) on rows painted by a non-merged segment, 0 elsewhere.                                     */
int pasco_panoptic_pass2(const int32_t* win, const float* m_win, const float* m_sum, int64_t n, const int32_t* seg_of,
                         const int32_t* cls_of, int32_t* panoptic, int32_t* semantic, float* confidence, pasco_stream_t s);
/* helper.py:246-281: the dense volumes of panoptic_inference from the rows of passes 1 and 2.  Row r (coords int32
 * [n, 4], batch 0) lands at cell coord − min_c of the X x Y x Z box; every output is zeroed by the caller.  panoptic /
 * semantic int32 and confidence fp32 [X, Y, Z] take the pass-2 rows; on rows with semantic != 0 (painted by a segment
 * of its own), ins_uncertainty = the winner's class probability, vox_uncertainty = prob_q * m_q / c_sum and
 * all_mask_probs fp32 [kq, X, Y, Z] = probs[r, kept[k]] (kept int32 [kq]: the kept queries, as pass 1 orders them).
 * A row outside the box or of another batch sets *err_flag = 1 and is skipped.                                     */
int pasco_panoptic_dense(const int32_t* coords, int64_t n, const int32_t min_c[3], int32_t X, int32_t Y, int32_t Z,
                         const int32_t* panoptic_rows, const int32_t* semantic_rows, const float* confidence_rows,
                         const int32_t* win, const float* m_win, const float* c_sum, const float* query_probs, int32_t K1,
                         const float* probs, int32_t Q, const int32_t* kept, int32_t kq, int32_t* panoptic,
                         int32_t* semantic, float* confidence, float* ins_uncertainty, float* vox_uncertainty,
                         float* all_mask_probs, int32_t* err_flag, pasco_stream_t s);
/* ensembler.py:159-187: the dense class distributions [K, cells] of ensemble_sem_compl.  subnet_out (NULL allowed, or a
 * host array of M device pointers, each NULL allowed) [m] = subnet m's softmax row at every cell where it has one and
 * one-hot class 0 elsewhere; ensemble_out (NULL allowed) = their mean, computed as pasco_sem_ensemble computes it; gate
 * (NULL allowed) [cells] = first argmax of that mean != 0.  probs / cell_rows as in pasco_sem_ensemble.             */
int pasco_sem_dense(int32_t M, const float* const probs[], const int32_t* const cell_rows[], int64_t cells, int32_t K,
                    float* const subnet_out[], float* ensemble_out, uint8_t* gate, pasco_stream_t s);
/* ensembler.py:102-105: gate [cells] = first argmax over the K channels of dense [K, cells] != 0.                   */
int pasco_class_gate(const float* dense, int64_t cells, int32_t K, uint8_t* gate, pasco_stream_t s);

/* ---- evaluation of the predictions against a scene's ground truth: the counting passes of Net.evaluate_all
 *      (net_panoptic_sparse.py:650-765), finished on the host by pasco_b200/metrics.py --------------------------------
 * label uint8 [cells] is the semantic ground truth (255 = unknown).  Counts are integer atomics; float sums are double,
 * reduced per CTA in thread order and over CTAs in CTA order (bit-identical repeat calls).  bounds = the 16 fp32 bin
 * boundaries torch.linspace(0, 1, 16); a confidence falls in slot (number of boundaries <= conf) − 1, as
 * torch.bucketize(conf, bounds, right=True) − 1, so 1.0 has slot 15 of its own.  Every output is zeroed by the caller. */

/* panoptic_quality.py:357-390 + net_panoptic_sparse.py:719-726: masks uint8 [n_masks, cells], seg_of_mask int32
 * [n_masks] = the segment id each mask paints (0 = none; from the host walk over the labels).  gt_id int32 [cells] =
 * the id of the last mask covering the cell (0 at unknown cells); mask_count [n_masks] = every mask's sum; gt_area
 * [G + 1] = cells of each id after the zeroing; hist [K + 1] = known cells per class, hist[K] = labels >= K.         */
int pasco_eval_gt(const uint8_t* masks, int32_t n_masks, const int32_t* seg_of_mask, const uint8_t* label, int64_t cells,
                  int32_t G, int32_t K, int32_t* gt_id, int32_t* mask_count, int32_t* gt_area, int32_t* hist,
                  pasco_stream_t s);
/* panoptic_quality.py:189-216 over an entry's rows (lin int64 ascending cells, panoptic int32 ids in [0, S]), known
 * cells only: pairs int32 [(G + 1) x (S + 1)] = cells per (gt id, pred id) with pred id != 0; pred_area [S + 1] = cells
 * per pred id, pred_area[0] = rows with a cell outside [0, cells) or an id outside [0, S].  Privatised in shared
 * memory when the table fits.                                                                                      */
int pasco_eval_pairs(const int64_t* lin, const int32_t* panoptic, int64_t n, const int32_t* gt_id, const uint8_t* label,
                     int64_t cells, int32_t G, int32_t S, int32_t* pairs, int32_t* pred_area, pasco_stream_t s);
/* metrics.py:480-547 over an entry's semantic rows (lin int64, pred int32, conf fp32) at known cells: confmat int32
 * [K x K] (gt row, pred column); cal int32 [2][2][16] = per partition (0: pred == 0, 1: pred != 0) the count and the
 * correct count per slot; pred_bad = rows with a cell outside [0, cells) or, at known cells, a pred or label outside
 * [0, K); sums double [34] = per partition the 16
 * slot confidence sums, then per partition Σ −log(p[label] + 1e-12) with p the mean of the M <= 8 subnets' softmax
 * rows (probs / cell_rows host arrays of device pointers, as in pasco_sem_ensemble; M = 0: no NLL).  1 <= K <= 64.  */
int pasco_eval_ssc(const int64_t* lin, const int32_t* pred, const float* conf, int64_t n, const uint8_t* label,
                   int64_t cells, int32_t K, const float bounds[16], int32_t M, const float* const probs[], const int32_t* const cell_rows[],
                   int32_t* confmat, int32_t* cal, int32_t* pred_bad, double* sums, pasco_stream_t s);
/* metrics.py:137-165 over an entry's rows with gt_id[cell] != 0 and confidence != 0: correct when match[pred id] (int32
 * [S + 1], 0 = unmatched) equals the gt id; rows with a cell outside [0, cells) are skipped.  cal int32 [2][16]
 * (count, correct per slot), sums double [16].                                                                      */
int pasco_eval_vox(const int64_t* lin, const int32_t* panoptic, const float* confidence, int64_t n, const int32_t* gt_id,
                   int64_t cells, const int32_t* match, int32_t S, const float bounds[16], int32_t* cal, double* sums, pasco_stream_t s);

/* ---- dense forms: the volumes the reference's Net.evaluate_all is given (net_panoptic_sparse.py:650-695), cell i of
 *      an [X, Y, Z] volume is row i; no cell array is read ------------------------------------------------------------
 * panoptic_quality.py:359: out fp32 [cells] = gt_id as float (pasco_eval_gt's ids, 0 at unknown cells), the
 * gt_panoptic_seg volume evaluate_all returns.                                                                      */
int pasco_eval_gt_volume(const int32_t* gt_id, int64_t cells, float* out, pasco_stream_t s);
/* pasco_eval_pairs over a dense id volume panoptic int32 [cells]: pred_area[0] = cells with an id outside [0, S].    */
int pasco_eval_pairs_dense(const int32_t* panoptic, const int32_t* gt_id, const uint8_t* label, int64_t cells, int32_t G,
                           int32_t S, int32_t* pairs, int32_t* pred_area, pasco_stream_t s);
/* net_panoptic_sparse.py:682-694 + metrics.py:480-547 over class planes prob fp32 [K][cells] (channel-major): pred int64
 * [cells] = first argmax over K as torch.argmax (a NaN wins, the first NaN); confmat int32 [K x K] at known cells; with
 * confidence fp32 [cells] (NULL: no calibration, cal / sums untouched, sums may be NULL) cal int32 [2][2][16] and sums
 * double [34] as pasco_eval_ssc's, the NLL of the label's own plane.  bad = known cells with a label >= K, or with a
 * confidence outside [0, 1] (NaN included).  1 <= K <= 64.                                                          */
int pasco_eval_ssc_planes(const float* prob, int32_t K, int64_t cells, const uint8_t* label, const float* confidence,
                          const float bounds[16], int64_t* pred, int32_t* confmat, int32_t* cal, int32_t* bad,
                          double* sums, pasco_stream_t s);
/* pasco_eval_vox over dense volumes panoptic int32 / confidence fp32 [cells]; bad = counted cells (gt id != 0,
 * confidence != 0) whose confidence lies outside [0, 1], left out of cal and sums.                                  */
int pasco_eval_vox_dense(const int32_t* panoptic, const float* confidence, const int32_t* gt_id, int64_t cells,
                         const int32_t* match, int32_t S, const float bounds[16], int32_t* cal, int32_t* bad,
                         double* sums, pasco_stream_t s);

/* ---- training criterion of the reference's SetCriterion (criterion_sparse.py, matcher_sparse.py, helper.py:7-37,
 *      lovasz.py:186-219) on one output level's rows; fp32, float sums in a fixed order ------------------------------
 * Samples the T mask volumes masks uint8 [T][X·Y·Z], unknown uint8 [X·Y·Z] and (label != NULL) the class volume at
 * the rows (b, x, y, z) of xyz int32 [n][4] with b = 0, at (x, y, z) − min_c (int32 [3], device); rows with b != 0 get
 * no bit, flag or label and are not counted.  bits uint32 [n][max(1, ceil(T/32))], flags uint8 [n] (1: not
 * unknown, 2: also at least one target bit), lab int32 [n] (−1 for 255).  stats int32 [T + 5], zeroed by the caller:
 * per-target bit counts over the valid rows, the valid-row count, rows outside the volume or with a label outside
 * [0, K) other than 255, two words of present-class bits, the known-row count.  1 <= K <= 64.                      */
int pasco_setloss_sample(const int32_t* xyz, int64_t n, const int32_t* min_c, const uint8_t* masks, int32_t T,
                         const uint8_t* unknown, const uint8_t* label, int32_t X, int32_t Y, int32_t Z, int32_t K,
                         uint32_t* bits, uint8_t* flags, int32_t* lab, int32_t* stats, pasco_stream_t s);
/* matcher_sparse.py:96-157: C fp32 [Q][T] from F fp32 [n][Q] read once over the valid rows, query_logits fp32 [Q][K1],
 * target class ids int32 [T] and class_weight fp32 [K1]; the focal part is 0 without valid rows.                    */
int pasco_setloss_match_cost(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                             const uint8_t* flags, const int32_t* stats, const float* query_logits, int32_t K1,
                             const int32_t* ids, const float* class_weight, float cost_mask, float cost_class,
                             float cost_dice, float* C, pasco_stream_t s);
/* criterion_sparse.py:83-112 over the known rows, per matched pair (query qi[k], target tj[k]): sums fp32 [P][4] =
 * Σ focal(F, t), Σ σ(F)·t, Σ σ(F), Σ t.  The backward writes dL/dF of the pairs' columns from g fp32 [P][4] (the
 * gradient of those sums) into gF fp32 [n][Q]; other columns are left as they are.                                 */
int pasco_setloss_pair_sums(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                            const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P, float* sums,
                            pasco_stream_t s);
int pasco_setloss_pair_backward(const float* F, int64_t n, int32_t Q, const uint32_t* bits, int32_t T,
                                const uint8_t* flags, const int32_t* qi, const int32_t* tj, int32_t P, const float* g,
                                float* gF, pasco_stream_t s);
/* helper.py:7-37: out fp32 [n][K] = Σ_j a_nj · L[j], a_nj = (σ(F[n, keep[j]]) + 1e-8) normalised over the kq kept
 * queries, L fp32 [kq][K].  The backward writes gF's kept columns and gL fp32 [kq][K] from g fp32 [n][K].
 * 1 <= kq <= 128, 1 <= K <= 64.                                                                                    */
int pasco_setloss_ssc_forward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq, const float* L,
                              int32_t K, float* out, pasco_stream_t s);
int pasco_setloss_ssc_backward(const float* F, int64_t n, int32_t Q, const int32_t* keep, int32_t kq, const float* L,
                               int32_t K, const float* out, const float* g, float* gF, float* gL, pasco_stream_t s);
/* lovasz.py:186-219 for every class at once.  labels int32 [P]: −1 leaves the row out, c in [0, C) is class c, >= C
 * is background of every class.  errors: probs fp32 [P][C] = softmax, err fp32 [C][P] = |fg − p| (−1 for a row left
 * out); the caller sorts each class's row descending (perm int64 [C][P]).  grad: lovasz_grad at every sorted
 * position into grad fp32 [C][P] and loss fp32 [C] = Σ err·grad per class.  backward: dx fp32 [P][C] from g fp32 [C]
 * = dL/dloss.  1 <= C <= 64.                                                                                       */
int pasco_lovasz_errors(const float* logits, int64_t P, int32_t C, const int32_t* labels, float* probs, float* err,
                        pasco_stream_t s);
int pasco_lovasz_grad(const float* err_sorted, const int64_t* perm, const int32_t* labels, int64_t P, int32_t C,
                      float* grad, float* loss, pasco_stream_t s);
int pasco_lovasz_backward(const float* probs, const int32_t* labels, const int64_t* perm, const float* grad,
                          const float* g, int64_t P, int32_t C, float* dx, pasco_stream_t s);

/* ---- the same criterion over a table of levels: each pass is one launch for every level (up to 24 per launch) -----
 * A level is one output level of one subnet: its mask logits F fp32 [n][Q], its subnet's sampled bits / flags / stats
 * (pasco_setloss_sample), its query logits [Q][K1], target class ids [T] and class weights [K1].  Each level keeps the
 * row chunking and the fixed-order partial sums of the one-level calls above, so a grouped call gives the same bits as
 * one call per level.  Each pass reads only the fields it names; the others may be zero.                            */
typedef struct {
  const float* F;                /* [n][Q] */
  int64_t n;
  int32_t Q, T;
  const uint32_t* bits;
  const uint8_t* flags;
  const int32_t* stats;
  const float* query_logits;     /* [Q][K1] */
  int32_t K1;
  const int32_t* ids;            /* [T] */
  const float* class_weight;     /* [K1] */
  float* C;                      /* match cost: [Q][T] */
  const int32_t* qi;             /* pair sums: P matched pairs */
  const int32_t* tj;
  int32_t P;
  float* sums;                   /* [P][4] */
  const float* g_sums;           /* pair backward: [P][4] */
  float* gF_pairs;               /* [n][Q], the pairs' columns written */
  int32_t* keep;                 /* keep: queries whose arg-max is not the last class, ascending, [Q] */
  int32_t* kept;                 /* keep: their count, [1] */
  int32_t kq;                    /* ssc: kept queries (0: the level has no ssc term) */
  const float* L;                /* ssc: row j of the class logits at L + rows[j]·ldL (rows NULL: j), K columns */
  const int32_t* L_rows;
  int32_t ldL, K;
  float* ssc;                    /* [n][K] */
  const float* g_ssc;            /* ssc backward: [n][K] */
  float* gF_ssc;                 /* [n][Q], the kept columns written */
  float* gL;                     /* [kq][K] */
} pasco_setloss_level;

/* keep: helper.py:20-23's kept queries of every level, built on the device.  1 <= Q <= 4096, 2 <= K1 <= 65.      */
int pasco_setloss_keep_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s);
/* pasco_setloss_match_cost for every level with T >= 1.                                                             */
int pasco_setloss_match_cost_group(const pasco_setloss_level* lv, int32_t count, float cost_mask, float cost_class,
                                   float cost_dice, pasco_stream_t s);
/* pasco_setloss_pair_sums / _pair_backward for every level with P >= 1.                                             */
int pasco_setloss_pair_sums_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s);
int pasco_setloss_pair_backward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s);
/* pasco_setloss_ssc_forward / _ssc_backward for every level with kq >= 1.                                           */
int pasco_setloss_ssc_forward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s);
int pasco_setloss_ssc_backward_group(const pasco_setloss_level* lv, int32_t count, pasco_stream_t s);

/* One Lovász-softmax term: the fields of pasco_lovasz_errors / _grad / _backward.  perm holds row indices within the
 * term, as in the one-term calls.                                                                                   */
typedef struct {
  const float* logits;           /* [P][C] */
  int64_t P;
  int32_t C;
  const int32_t* labels;         /* [P] */
  float* probs;                  /* [P][C] */
  float* err;                    /* [C][P] */
  const float* err_sorted;       /* [C][P] */
  const int64_t* perm;           /* [C][P] */
  float* grad;                   /* [C][P] */
  float* loss;                   /* [C] */
  const float* g;                /* [C] */
  float* dx;                     /* [P][C] */
} pasco_lovasz_term;

int pasco_lovasz_errors_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s);
int pasco_lovasz_grad_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s);
int pasco_lovasz_backward_group(const pasco_lovasz_term* t, int32_t count, pasco_stream_t s);

/* ---- point voxeliser grouping and the MIMO merge (csrc/voxel.cu); keys pack as the hash table's ---------------------
 * voxel_group: torch.unique(rows, dim=0, return_inverse=True) for rows [n][4] (int32, or int64 when is_i64)
 * (unet3d_sparse_v2.py:72-75).  Pass 1 inserts every row's key into table_keys (capacity, power of two >= 2n, filled
 * with 0xFF bytes) and writes the U unique keys, unordered, to ukeys [n]; stats int32 [2], zeroed by the caller: U and
 * an error flag (a component outside [-32768, 32767]; the other outputs are then undefined and _order must not run).
 * _order sorts the keys, writes unique_rows [U][4] (the input's integer type) in ascending lexicographic order of the
 * signed rows and inverse int64 [n]; table_vals int32 [capacity] is scratch.                                       */
int pasco_voxel_group(const void* rows, int32_t is_i64, int64_t n, uint64_t* table_keys, int64_t capacity,
                      uint64_t* ukeys, int32_t* stats, pasco_stream_t s);
int pasco_voxel_group_order(const void* rows, int32_t is_i64, int64_t n, const uint64_t* table_keys,
                            int32_t* table_vals, int64_t capacity, const uint64_t* ukeys, int64_t U, void* unique_rows,
                            int64_t* inverse, pasco_stream_t s);
/* Augmenter.merge (augmenter.py:13-27) without the dense volume.  coords int32 [n][4] (t, x, y, z) with t the subnet,
 * F fp32 [n][f].  _cells inserts the (x, y, z) cells (table_vals int32 [capacity] zeroed by the caller) and writes the
 * U cells that have a feature other than ±0 to ukeys [n], unordered; stats int32 [3], zeroed by the caller: U, the
 * largest t, an error flag (t < 0 or x, y, z outside [-32768, 32767]; _forward must not run).  _forward writes
 * out_coords int32 [U][4] = (0, x, y, z) in ascending (x, y, z) order, out_F fp32 [U][M·f] (subnet t's channels at
 * t·f, 0 where t has no row; t < M) and row_of int32 [n] (the output row of each input row, −1 for a dropped cell).
 * _backward: gin fp32 [n][f] = g [U][M·f] at the row's output row and channels, 0 for a dropped cell.            */
int pasco_mimo_merge_cells(const int32_t* coords, const float* F, int64_t n, int32_t f, uint64_t* table_keys,
                           int32_t* table_vals, int64_t capacity, uint64_t* ukeys, int32_t* stats, pasco_stream_t s);
int pasco_mimo_merge_forward(const int32_t* coords, const float* F, int64_t n, int32_t f, int32_t M,
                             const uint64_t* table_keys, int32_t* table_vals, int64_t capacity, const uint64_t* ukeys,
                             int64_t U, int32_t* out_coords, float* out_F, int32_t* row_of, pasco_stream_t s);
int pasco_mimo_merge_backward(const int32_t* coords, const int32_t* row_of, int64_t n, int32_t f, int32_t M,
                              const float* g, float* gin, pasco_stream_t s);

/* ---- the reference decoder's glue (csrc/decoder.cu; decoder_v3.py) -------------------------------------------------
 * completion_rows: probs = host array of M (<= 8) device pointers to fp32 softmax rows [n][K] (K <= 64).  Writes
 * cls int32 [M][n] (torch's max(-1) index: the first maximal value, a NaN at its first index), keep uint8 [M][n] =
 * cls != 0, votes int32 [n] = sum over m of keep, and with w fp32 [K] (may be null) weight fp32 [M][n] = p_max * w[cls]
 * as one fp32 multiply.  counts int32 [3M + 1], zeroed by the caller: kept rows per subnet, labelled cells per subnet
 * ((label != 0) & (label != 255) over labels = host array of M device volumes of n_label signed integers of
 * label_bytes bytes; may be null), rows whose weight is not a finite value >= 0 per subnet, rows with a vote.
 * topk_mask: keep uint8 [n] = the k largest w / q (IEEE fp32 division, w / q >= 0, not NaN), ties at the k-th value
 * taken by lowest row: torch.multinomial(w, k, replacement=False)'s set when q is its Exp(1) draw.
 * panop_crop: mask uint8 [n] = argmax(logits row) != 0 AND min <= (x, y, z) <= max with box int32 [6] = (min, max);
 * counts int32 [2], zeroed by the caller: rows with argmax != 0, rows kept.  With no argmax != 0, the first 1000 rows
 * inside the box are kept (decoder_v3.py:415-417).
 * mimo_batch: feats / coords = host arrays of M device pointers to fp32 [len_m][C] / int32 [len_m][4], len_m <= L.
 * out_F fp32 [M][L][C] and out_C int32 [M][L][4] zero-padded; keep_pad uint8 [M][L] (may be null) = any feature or
 * coordinate of the padded row != 0.                                                                             */
int pasco_completion_rows(const float* const* probs, int32_t M, int64_t n, int32_t K, const float* w,
                          const void* const* labels, int64_t n_label, int32_t label_bytes, int32_t* cls, uint8_t* keep,
                          float* weight, int32_t* votes, int32_t* counts, pasco_stream_t s);
int pasco_topk_mask(const float* w, const float* q, int64_t n, int64_t k, uint8_t* keep, pasco_stream_t s);
int pasco_panop_crop(const float* logits, int64_t n, int32_t K, const int32_t* coords, const int32_t* box,
                     uint8_t* mask, int32_t* counts, pasco_stream_t s);
int pasco_mimo_batch(const float* const* feats, const int32_t* const* coords, const int64_t* lengths, int32_t M,
                     int64_t L, int32_t C, float* out_F, int32_t* out_C, uint8_t* keep_pad, pasco_stream_t s);

/* ---- the reference transformer's sine position encoding (csrc/posenc.cu; transformer/position_encoding.py) ----------
 * sine_pos: PositionEmbeddingSineSparse(n, normalize=True) of P coordinate rows.  coords points at row 0's x; rows are
 * coord_pitch integers apart (int32, or int64 when is_i64), x, y, z adjacent.  table fp32 [rows][n] = the per-axis
 * encoding of coordinates lo .. lo + rows - 1; a coordinate beyond either end reads that end's row, so the table must
 * span every coordinate whose encoding differs from its ends' (|x| < 32 for the reference's eps and scale).  Writes
 * out fp32 [P][3n] (x, y, z blocks of n), rows out_pitch floats apart: out = pe (add = 0) or out += pe (add = 1).
 * n even, 2 <= n <= 256.                                                                                           */
int pasco_sine_pos(const void* coords, int32_t is_i64, int64_t P, int64_t coord_pitch, const float* table, int32_t lo,
                   int32_t rows, int32_t n, float* out, int64_t out_pitch, int32_t add, pasco_stream_t s);

/* ---- SemanticKITTI scene preparation (pasco/data/semantic_kitti/kitti_dataset.py:142-490, collate.py) ----
 * One item: label volumes sem / inst uint8 [X, Y, Z] (C order), a pose T and its inverse Ti (fp32 row-major 4x4, host
 * arrays), points fp32 [N, pitch] (x, y, z, then intensity columns).  Cells are transformed as transform_utils.transform
 * does, in fp32 (c * 0.2 + 0.1 + min_bound, T with fused multiply-adds in k order, (p − min_bound − 0.1) / 0.2,
 * round half to even); points as load_data_v3 does (numpy floor_divide in fp64, then transform).  stats int32
 * [PASCO_SCENE_STATS] collects each phase's integer results at the offsets below (pasco_scene_source initialises it);
 * bounds fp64 [4] are the crop's (new_min x, new_min y, new_max x, new_max y), ±inf without a crop.              */
enum {
  PASCO_SCENE_BND = 0,            /* min[3], max[3] of transform(nonzero(sem != 255), T)                   */
  PASCO_SCENE_N_LABELLED = 6,     /* source cells with sem != 255                                           */
  PASCO_SCENE_N_INSTANCE = 7,     /* source cells with inst != 0                                            */
  PASCO_SCENE_SEM_EXT = 8,        /* min[3], max[3] of the semantic rows of the transformed box             */
  PASCO_SCENE_N_SEM_ROWS = 14,    /* semantic rows of the transformed box                                   */
  PASCO_SCENE_BOX = 16,           /* min[3], max[3] of the semantic and instance rows the crop keeps        */
  PASCO_SCENE_N_SEM_KEPT = 22,    /* semantic rows the crop keeps                                           */
  PASCO_SCENE_N_POINTS = 23,      /* points inside the extent                                               */
  PASCO_SCENE_N_POINTS_KEPT = 24, /* of those, points the crop keeps                                        */
  PASCO_SCENE_CLS_ORIGIN = 256,   /* [256] flags: classes of the source semantic volume                     */
  PASCO_SCENE_INST_ORIGIN = 512,  /* [256] flags: ids of the source instance volume other than 0            */
  PASCO_SCENE_CLS = 768,          /* [256] flags: classes of the kept semantic rows                         */
  PASCO_SCENE_INST = 1024,        /* [256] flags: ids of the kept instance rows                             */
  PASCO_SCENE_STATS = 1280
};
/* initialises stats; BND, N_LABELLED, N_INSTANCE and the *_ORIGIN flags.  X, Y, Z >= 2.                              */
int pasco_scene_source(const uint8_t* sem, const uint8_t* inst, int32_t X, int32_t Y, int32_t Z, const float T[16],
                       int32_t* stats, pasco_stream_t s);
/* transform_scene over the box [lo, lo + G) (lo, G host arrays): gs / gi uint8 [G0, G1, G2] = source label + 1 (uint8,
 * so 255 → 0 = no row) at grid_sample's nearest source cell of Ti · centre, 0 outside; gi only with with_inst (the
 * source has an instance id other than 0).  SEM_EXT and N_SEM_ROWS.                                                   */
int pasco_scene_resample(const uint8_t* sem, const uint8_t* inst, int32_t X, int32_t Y, int32_t Z, const float Ti[16],
                         const int32_t lo[3], const int32_t G[3], int32_t with_inst, uint8_t* gs, uint8_t* gi,
                         int32_t* stats, pasco_stream_t s);
/* KittiDataset.crop's bounds from SEM_EXT and draw (np.random.rand(3), host array; NULL without a crop): crop_size =
 * (max − min) · 0.8 in fp32, new_min = min + (max − min − crop_size) · draw in fp64.  train = 0: ±inf.                 */
int pasco_scene_crop(const int32_t* stats, const double draw[3], int32_t train, double* bounds, pasco_stream_t s);
/* BOX, N_SEM_KEPT, CLS and INST over the rows of gs / gi inside the crop                                              */
int pasco_scene_crop_stats(const uint8_t* gs, const uint8_t* gi, const int32_t lo[3], const int32_t G[3],
                           int32_t with_inst, const double* bounds, int32_t* stats, pasco_stream_t s);
/* per point: ext[i] = inside the extent, keep[i] = ext and its transformed voxel inside the crop; N_POINTS and
 * N_POINTS_KEPT.                                                                                                       */
int pasco_scene_points(const float* pts, int64_t N, int32_t pitch, const float T[16], const double* bounds, uint8_t* ext,
                       uint8_t* keep, int32_t* stats, pasco_stream_t s);
/* keep_rows int32 [n_keep] (ascending point indices): feats fp32 [n_keep, V + pitch − 3 + 1 + E + 6] = (vote fp32 [N, V],
 * intensity, radius, embedding emb fp32 [E, N] transposed, xyz − voxel centre, xyz) and coords int64 [n_keep, 3];
 * ext_rows int32 [n_ext]: xyz fp64 [n_ext, 3] = xyz − vox_origin and label_out [n_ext] = label & 0xFFFF.             */
int pasco_scene_point_rows(const float* pts, int32_t pitch, const float* vote, int32_t V, const float* emb, int32_t E,
                           int64_t N, const int32_t* keep_rows, int64_t n_keep, const float T[16], float* feats,
                           int64_t* coords, const int32_t* label, const int32_t* ext_rows, int64_t n_ext, double* xyz,
                           int32_t* label_out, pasco_stream_t s);
/* the item's volumes on the box [box_lo, box_lo + size) (host arrays) from the kept rows of gs / gi: sem (255 where no
 * row), inst (0 where no row) and geo = complete_voxel as uint8 (0 empty, 1 labelled, 255 unknown), all uint8.        */
int pasco_scene_box(const uint8_t* gs, const uint8_t* gi, const int32_t lo[3], const int32_t G[3], int32_t with_inst,
                    const double* bounds, const int32_t box_lo[3], const int32_t size[3], uint8_t* sem, uint8_t* inst,
                    uint8_t* geo, pasco_stream_t s);
/* sem_labels / geo_labels at scale 2 or 4 (kitti_dataset.py:217-266) of sem uint8 [X, Y, Z] (multiples of the scale):
 * geo = 255 if the whole block is 255, else whether a cell is labelled 1-254; sem = the first class of 1-19 with the
 * most cells, and without one 0 if the whole block is 255, else 255.  Outputs uint8 [X/s, Y/s, Z/s].                 */
int pasco_scene_scale(const uint8_t* sem, int32_t X, int32_t Y, int32_t Z, int32_t scale, uint8_t* sem_out,
                      uint8_t* geo_out, pasco_stream_t s);
/* prepare_mask_label of sem / inst uint8 [cells]: slot int32 [512] (device) gives the mask of class c at slot[c] and of
 * instance id at slot[256 + id], −1 for none.  masks bool [n_masks, cells] (zero-filled here), labels uint8 [n_masks]:
 * the class of a class mask, sem at the first cell in C order of an instance mask.  cells < 2^31.                     */
int pasco_scene_masks(const uint8_t* sem, const uint8_t* inst, int64_t cells, const int32_t* slot, int32_t n_masks,
                      uint8_t* masks, uint8_t* labels, pasco_stream_t s);

#ifdef __cplusplus
}
#endif
#endif /* PASCO_SM100_H_ */
