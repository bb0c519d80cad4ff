/*
 * tio_b200.h — C-ABI of the CUDA-native (sm_90a) 3-D augmentation hot path.
 *
 * Drop-in boundary for the TorchIO v2 (2.0.0a2 @ 2b019d2) transform kernels.
 * The reference has no FFI layer: its seam is the Python method
 *   Transform.apply_transform(batch, params)        transforms/transform.py:408-427
 * and, one level down, the plain-tensor helpers each entry point below
 * replaces (cited per function; paths relative to src/torchio/).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - Volumes are contiguous (B, C, I, J, K), K fastest, in DEVICE memory.
 *   - Parameter tables are DEVICE pointers unless marked "host"; callers pack
 *     them into one pinned staging buffer and upload it once per launch.
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default).
 *   - Every function returns 0 on success, non-zero on error;
 *     tio_last_error() returns a thread-local message.  No exceptions cross
 *     the boundary, no global mutable state, re-entrant from several threads
 *     (the reference calls transforms from Queue's ThreadPoolExecutor,
 *     data/queue.py:119-123).
 *   - Outputs are caller-allocated; the library keeps no pointer after return.
 */
#ifndef TIO_B200_H
#define TIO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TIO_ABI_VERSION 2

/* element types accepted by tio_resample (images: F32; label maps: the rest) */
enum tio_dtype {
  TIO_F32 = 0,
  TIO_U8 = 1,
  TIO_I8 = 2,
  TIO_I16 = 3,
  TIO_I32 = 4,
  TIO_I64 = 5,
  /* images accepted by tio_interpolate / tio_axis_resample only */
  TIO_F16 = 6,
  TIO_BF16 = 7,
  TIO_F64 = 8
};

enum tio_interp { TIO_NEAREST = 0, TIO_LINEAR = 1, TIO_LABEL_PV = 2 };
/* OR into `mode`: keep the reference's fp32 rounding sequence of the sampling coordinates on
 * every tile.  Without it, fp32 trilinear tiles whose taps all lie inside the volume evaluate the
 * same mapping with one fma per axis (differs from the reference's own coordinate noise by
 * <= ~2e-5 voxel); label maps, border tiles and fill decisions are always exact. */
#define TIO_EXACT_COORDS 0x100

/* per-element flag bits for tio_resample */
#define TIO_FLAG_PASSTHROUGH 1u /* copy the row bit-exactly (spatial.py:1101-1106) */
#define TIO_FLAG_ELASTIC 2u     /* the element has a control-point grid */

const char* tio_last_error(void);
int tio_abi_version(void);
/* Number of kernels the calling thread has launched through the library, counted at each launch
 * (cudaMemsetAsync / cudaMemcpyAsync are not kernels and are not counted).  Thread-local, like
 * tio_last_error(). */
uint64_t tio_launch_count(void);

/*
 * K1 — fused resample: affine matrix + trilinear control-point displacement +
 * 8-tap / nearest gather + out-of-bounds fill + pass-through rows, one pass.
 *
 * Replaces _build_sampling_grid + _sample_batch[_per_sample]
 *   (transforms/spatial/spatial.py:1504-1579, 1651-1731, 1764-1857)
 * i.e. arange/meshgrid/cat/matmul, F.interpolate(trilinear, align_corners),
 * two F.grid_sample(zeros, align_corners=True) passes and torch.where.
 *
 *   src, dst   (B, C, I, J, K) / (B, C, OI, OJ, OK) of `dtype`
 *   mat        [B][12] fp32: rows 0..2 of inv(A_in) @ inv(T) @ A_out
 *              (float64 product cast to fp32, spatial.py:1594-1601)
 *   cp         [B][ni][nj][nk][3] fp32 displacements in mm, or NULL
 *   flags      [B] bytes (TIO_FLAG_*), or NULL (= 0 for every element)
 *   spacing_in/out  host float[3]: fp32 casts of the affine column norms
 *              (spatial.py:1559-1568)
 *   affine_first    spatial.py:1570-1577
 *   mode       TIO_NEAREST | TIO_LINEAR (spatial.py:150-153), optionally | TIO_EXACT_COORDS;
 *              TIO_LABEL_PV = label_interpolation="label" with the default linear one-hot
 *              interpolation, fused (spatial.py:1275-1389 without materialising the one-hot
 *              channels): C must be 1, fill[0] = default_pad_label (required); per output voxel
 *              the trilinear weight of every label among the 8 taps is accumulated in
 *              grid_sample's corner order, the largest wins (smallest label on ties, as
 *              argmax over torch.unique's ascending channels), and voxels whose in-bounds
 *              weight is not > 0.5 take the pad label.  u8 / i16 / i32 take the TMA tile path
 *              (box_hint >= 0 and a workspace), any other dtype the general gather kernel.
 *   fill       [C] fp32 per-channel fill, or NULL = skip the mask step
 *              (the reference skips it only for a python-float 0.0 fill,
 *              spatial.py:2072-2076).  The mask is always the TRILINEAR
 *              in-bounds weight sum, even for nearest data (:1722-1727).
 *   box_hint   host int selecting the kernel: < 0 = general gather kernel only
 *              (exact mul+add tap sum); 0 = TMA tile path with the default
 *              24^3 input box; 20 / 22 / 24 / 28 / 32 = TMA tile path with that box edge
 *              (callers that know the matrices pick the smallest box covering
 *              the pre-image of a 16^3 output tile).  The tile path applies to
 *              fp32 + TIO_LINEAR with K % 4 == 0; anything else, and any tile
 *              whose pre-image does not fit, uses the general kernel.
 *   workspace  device scratch of tio_resample_workspace_bytes(B, OI, OJ, OK) bytes,
 *              16-byte aligned (per-tile records of the TMA path); may be NULL,
 *              which selects the general kernel.  The library allocates nothing.
 * src and dst must not alias.
 */
size_t tio_resample_workspace_bytes(int B, int OI, int OJ, int OK);

/*
 * B-spline interpolation of orders 2-7 (image_interpolation / label_interpolation /
 * one_hot_label_interpolation "quadratic" ... "seventh"): the reference's
 *   interpol.grid_pull(data.float(), voxel_grid, interpolation=order, bound="dct2",
 *                      extrapolate=False, prefilter=True)
 * (transforms/spatial/spatial.py:1734-1761, 1860-1878), in two steps.
 *
 * tio_bspline_prefilter: coeff (B, C, I, J, K) fp32 = the interpolating B-spline coefficients of
 *   src (B, C, I, J, K) of `dtype` (TIO_F32 .. TIO_I64) under the half-sample-symmetric (dct2)
 *   boundary, per (b, c) volume: one pass per axis longer than 1 (at most three launches).
 *   Elements whose flags[b] has TIO_FLAG_PASSTHROUGH are skipped (flags may be NULL).  coeff may
 *   be src itself when dtype is TIO_F32 (in place); it must not overlap src otherwise.  A volume
 *   of 1 x 1 x 1 voxels is copied (converted to fp32) unless coeff is src.  Axes of up to 51199
 *   voxels: a CTA stages whole lines in 200 KiB of shared memory (32 lines per CTA up to 1599
 *   voxels, fewer above); a longer axis is refused.
 *
 * tio_bspline_resample: dst (B, C, OI, OJ, OK) of `dtype` = the spline of coeff at the input-voxel
 *   coordinates tio_resample computes from mat / cp / flags / spacings / affine_first (same
 *   arguments, same fp32 arithmetic) before its [-1, 1] normalisation.  A voxel with any
 *   coordinate outside (-0.05, n - 1 + 0.05) of its axis is 0; the sum is cast to `dtype` by
 *   truncation, as Tensor.to.  Passthrough elements copy src (the data coeff was made from)
 *   bit-exactly.  One launch.  dst must not overlap coeff or src.
 *
 * Both validate every argument before launching (order outside 2-7, null pointers, forbidden
 * aliasing: non-zero return, tio_last_error) and allocate nothing.
 */
int tio_bspline_prefilter(const void* src, int dtype, float* coeff, const uint8_t* flags,
                          int B, int C, int I, int J, int K, int order, void* stream);
int tio_bspline_resample(const float* coeff, const void* src, void* dst, int dtype,
                         int B, int C, int I, int J, int K,
                         int OI, int OJ, int OK,
                         const float* mat, const float* cp, const uint8_t* flags,
                         int ni, int nj, int nk,
                         const float* spacing_in, const float* spacing_out,
                         int affine_first, int order, void* stream);
int tio_resample(const void* src, void* dst, int dtype,
                 int B, int C, int I, int J, int K,
                 int OI, int OJ, int OK,
                 const float* mat, const float* cp, const uint8_t* flags,
                 int ni, int nj, int nk,
                 const float* spacing_in, const float* spacing_out,
                 int affine_first, int mode, const float* fill, int box_hint,
                 void* workspace, size_t workspace_bytes, void* stream);
/*
 * tio_resample with a box edge per batch element: fp32 + TIO_LINEAR (no TIO_EXACT_COORDS),
 * box_hint >= 0 and a workspace.  `elems` (device int[B]) lists every batch element once, and
 * `runs` (host int[2 * n_runs]: count, edge) splits that list into runs of ascending edges
 * (20 / 22 / 24 / 28 / 32, 1 <= n_runs <= 5, counts summing to B).  Each run is one bounds
 * pre-pass and one tile launch over its elements with that box, writing its elements' output.
 * A tile takes the staged box when its pre-image fits its run's box, so a caller that wants the
 * output of tio_resample(..., box_hint = E) picks for each element an edge that holds every
 * tile that fits E, and E itself for elements some of whose tiles need more.  Where the tile
 * path does not apply, the general kernel computes every element as tio_resample does.
 */
int tio_resample_tiered(const void* src, void* dst, int dtype,
                        int B, int C, int I, int J, int K,
                        int OI, int OJ, int OK,
                        const float* mat, const float* cp, const uint8_t* flags,
                        int ni, int nj, int nk,
                        const float* spacing_in, const float* spacing_out,
                        int affine_first, int mode, const float* fill, int box_hint,
                        const int* elems, const int* runs, int n_runs,
                        void* workspace, size_t workspace_bytes, void* stream);
/*
 * K1ᵀ — the adjoint of tio_resample with respect to src, for fp32 gradients: grad_in (B, C, I, J, K)
 * = K1ᵀ grad_out (B, C, OI, OJ, OK), with the geometry arguments of the forward call (mode
 * TIO_NEAREST or TIO_LINEAR, TIO_EXACT_COORDS accepted).  Replaces the backward of the reference's
 * F.grid_sample / torch.where (spatial.py:1651-1731, 1764-1857): each output voxel sends g * w to each
 * in-bounds trilinear tap (nearest: g to the rounded voxel), a voxel the forward filled (fill given
 * and mask <= 0.5) sends nothing, and TIO_FLAG_PASSTHROUGH elements copy g, which needs
 * (OI, OJ, OK) == (I, J, K) as in tio_resample (flags live on the device: the library cannot check).
 * Coordinates, weights and fill decisions follow the reference's fp32 chain in both coordinate
 * modes.  grad_in is zeroed (cudaMemsetAsync), then one bounds pre-pass and one tile launch add into
 * it with atomics: the result is not deterministic.  workspace: tio_resample_workspace_bytes(B, OI,
 * OJ, OK) bytes, 16-byte aligned, required.  box_hint > 24 selects 32^3 boxes, else 24^3.
 */
int tio_resample_backward(const float* grad_out, float* grad_in,
                          int B, int C, int I, int J, int K,
                          int OI, int OJ, int OK,
                          const float* mat, const float* cp, const uint8_t* flags,
                          int ni, int nj, int nk,
                          const float* spacing_in, const float* spacing_out,
                          int affine_first, int mode, const float* fill, int box_hint,
                          void* workspace, size_t workspace_bytes, void* stream);

/*
 * The materialised form of label_interpolation="label", for the combinations the fused mode
 * does not cover (antialias=True blurs the one-hot channels before they are sampled,
 * spatial.py:1367-1368):
 *   tio_onehot        dst (B, n, vox) fp32 = (src (B, vox) == labels[c])  (spatial.py:1362-1365);
 *                     `labels` = the n distinct values of the batch, ascending, as device
 *                     int64 (integer dtypes) or fp32 (TIO_F32) values
 *   tio_label_argmax  dst (B, vox) of `dtype` = labels[argmax_c sampled (B, n, vox)] (first maximum),
 *                     or pad_label where the sequential channel sum is not > 0.5 (spatial.py:1378-1389)
 */
int tio_onehot(const void* src, int dtype, int B, int64_t vox, const void* labels, int n,
               float* dst, void* stream);
int tio_label_argmax(const float* sampled, int B, int n, int64_t vox, const void* labels,
                     float pad_label, void* dst, int dtype, void* stream);

/*
 * Patch extraction for the Queue path: gathers `n` patches of size (pi,pj,pk) with
 * corners `corners[n][3]` (device int32, voxel indices, corner + size <= shape —
 * validated by the caller) from one volume `src` (C,I,J,K) into a dense block `dst`
 * (n,C,pi,pj,pk).  `elem_bytes` in {1,2,4,8} (any dtype; bytes are moved verbatim).
 * Replaces PatchSampler._extract_patch's per-patch views (data/sampler.py:54-67,
 * 198-223) + the per-patch copies of collate_subjects' torch.stack
 * (loader.py:15-24) with one pass over the patch bytes.
 */
int tio_crop_patches(const void* src, void* dst, int elem_bytes, int C, int I, int J, int K,
                     int n, const int32_t* corners, int pi, int pj, int pk, void* stream);

/*
 * Flip / Crop / Pad as one index-remap copy of a (B,C,I,J,K) batch into (B,C,OI,OJ,OK):
 * source index along an axis = output index - off (off = voxels padded before; negative =
 * voxels cropped), indices outside the volume follow `mode` (0 constant -> `*fill`,
 * `elem_bytes` bytes on the HOST; 1 replicate; 2 reflect; 3 circular — F.pad's modes),
 * then the axis is reversed when the element's bit in `flip[b]` is set (bit 0 I, 1 J, 2 K;
 * device array or NULL).  Replaces torch.flip + torch.where (spatial/flip.py:233-263),
 * the crop slice (crop.py:84-101) and F.pad (_padding.py:73-104).  Any dtype by size.
 */
int tio_remap(const void* src, void* dst, int elem_bytes, int B, int C, int I, int J, int K,
              int OI, int OJ, int OK, int off_i, int off_j, int off_k, int mode,
              const void* fill, const uint8_t* flip, void* stream);

/*
 * Axis permutation with flips of a (B,C,I,J,K) batch into (B,C,n[perm0],n[perm1],n[perm2]),
 * n = (I,J,K): out[b,c,o0,o1,o2] = in[b,c,s] with s[perm_d] = o_d, or n[perm_d]-1-o_d when bit
 * perm_d of `flip_bits` is set (flips are indexed by INPUT axis: flip first, then transpose).
 * Replaces torch.flip per axis + permute(...).contiguous() (spatial/reorient.py:63-91) and
 * permute(0,1,4,3,2).contiguous() (transpose.py:36-50) with one pass over the batch.  Any dtype by
 * size (`elem_bytes` in {1,2,4,8}).  `perm` must be a permutation of (0,1,2) other than the
 * identity (flips alone are tio_remap's), `flip_bits` in 0..7; src and dst must not overlap.
 */
int tio_permute(const void* src, void* dst, int elem_bytes, int B, int C, int I, int J, int K,
                int perm0, int perm1, int perm2, int flip_bits, void* stream);

/*
 * Parameter-table upload without the copy engine: an SM kernel reads `bytes`
 * from page-locked host memory (`host_pinned`, a cudaHostAlloc/cudaHostRegister
 * pointer, device-visible under unified addressing) and writes them to
 * `dst_device`, ordered on `stream` like any launch.  The reference builds these
 * tables on the host and moves them with `.to(device)` inside each transform
 * (e.g. spatial.py:1548-1551, blur.py:292-328); when a batch is streamed through
 * the device in slices, such small cudaMemcpyAsync calls queue behind the bulk
 * volume copies on the copy engine and stall the kernels that need them.
 */
int tio_upload(const void* host_pinned, void* dst_device, size_t bytes, void* stream);

/*
 * Per-channel minimum of batch element 0 -> fill[C] on the device, no host
 * sync.  Replaces _batch_fill_value("minimum") = tensor.min().item()
 * (spatial.py:2054-2060, 2094-2095).  `src` is (B, C, n) fp32, n = I*J*K.
 * As torch.amin: NaN when the channel holds a NaN, otherwise its least value.
 */
int tio_min_sample0(const float* src, int C, int64_t n, float* fill, void* stream);

/*
 * K3 — separable Gaussian blur with replicate (clamp) addressing, axes I, J,
 * K in that order.  Replaces _gaussian_smooth{,_shared,_per_element}
 * (transforms/intensity/blur.py:129-252) = 3 x (F.pad replicate + F.conv3d).
 *   taps      [3][B][2R+1] fp32, centred, normalised on the host exactly as
 *             blur.py:179-183 / 292-328 (zero beyond each element's radius,
 *             delta kernel where sigma <= 0)
 *   radius    [3][B] int32: the element's own radius on that axis (0 = skip)
 *   R         table half-width (max radius over the whole table), at most 6143;
 *             R > 16 runs one launch per blurred axis and then needs `scratch`
 *             whatever the axes
 *   axes_mask host int, bit a set = axis a is active for at least one element
 *             (lets the library skip whole passes without reading `radius`)
 *   identity  [B] bytes: rows with all sigma <= 0 are copied exactly
 *   scratch   device buffer of B*C*I*J*K floats (may be NULL when only the I
 *             axis is active)
 * src and dst must not alias.
 */
int tio_blur(const float* src, float* dst, float* scratch,
             int B, int C, int I, int J, int K,
             const float* taps, const int32_t* radius, int R, int axes_mask,
             const uint8_t* identity, void* stream);

/*
 * K4a — exact replay of torch's CPU `randn` stream on the device:
 * mt19937(seed) -> 24-bit uniforms -> 16-wide Box-Muller blocks (ATen normal_fill;
 * the stream the reference depends on through torch.randn(generator=CPU),
 * noise.py:166-178).
 * tio_randn_mt19937_window: outputs [lo, hi) of torch.randn(n) drawn at stream word
 * `offset` (after `offset` words of the generator were used), output i to z[i - lo].
 * Any offset, any n >= 16, lo < hi <= n.  The draw takes words [offset, offset+n)
 * in 16-groups relative to offset (u[j] pairs with u[j+8]); when n % 16 != 0 it then
 * takes 16 more words, which give outputs [n-16, n) anew, so it ends at word
 * offset + n + 16 (offset + n otherwise), at most 2^31.
 * tio_randn_mt19937: the [0, n) window, for offset % 16 == 0, n % 16 == 0, n >= 16.
 *   table      device copy of the jump-ahead table built once by
 *              tio_mt19937_build_table (host, ~2 s; depends only on MT19937, so
 *              callers cache it; tio_mt19937_table_bytes() gives its size)
 *   workspace  device scratch of tio_randn_mt19937_workspace_bytes(offset, n), or of
 *              tio_randn_mt19937_window_workspace_bytes(offset, n) for the window
 * The uniforms are bit-identical to torch.s; normals agree to <= 4e-6 absolute
 * (CUDA libm vs the host.s log/sin/cos).
 */
size_t tio_mt19937_table_bytes(void);
int tio_mt19937_build_table(void* host_blob, size_t bytes);
size_t tio_randn_mt19937_workspace_bytes(uint64_t offset, uint64_t n);
int tio_randn_mt19937(uint64_t seed, uint64_t offset, uint64_t n, float* z,
                      const void* table, void* workspace, size_t workspace_bytes,
                      void* stream);
size_t tio_randn_mt19937_window_workspace_bytes(uint64_t offset, uint64_t n);
int tio_randn_mt19937_window(uint64_t seed, uint64_t offset, uint64_t n, uint64_t lo, uint64_t hi,
                             float* z, const void* table, void* workspace, size_t workspace_bytes,
                             void* stream);

/*
 * Data-derived parameters of Standardize / Normalize, computed where the batch lives
 * (the reference reads batch element 0 on the host: standardize.py:52-79, normalize.py:121-139,
 * 332-366, _statistics.py:11-45).
 *   tio_moments    out3 (device doubles) = {sum, sum of (x - sum/count)^2, count} of the `n` values
 *                  at `src` for which mask[t] != 0 (mask NULL = all); fp64 accumulation, two passes
 *                  (the second reads the mean on the device), so a constant selection gives 0
 *   tio_quantiles  for each of the m <= 2 quantiles q (host doubles in [0,1]): index = q*(count-1),
 *                  lower = floor(index); values[2t], values[2t+1] = the order statistics of rank
 *                  lower and min(lower+1, count-1) (what torch.kthvalue(lower+1 / lower+2) returns),
 *                  weights[t] = index - lower, *count = number of selected values.  It is
 *                  tio_quantiles_batched with B = 1 on fp32 values.
 *                  workspace: tio_quantiles_workspace_bytes() device bytes, 16-byte aligned.
 *   tio_rescale    dst = ((clamp(src, lo, hi) - sub[b]) / div[b]) * mul[b] + add[b] over (B, per_elem),
 *                  each step rounded to fp32 like the reference's separate elementwise ops
 *                  (normalize.py:176-181, standardize.py:93; the inverses :271-297, :139-141).
 *                  `flags` selects the steps: 1 clamp, 2 sub, 4 div, 8 mul, 16 add (tables for
 *                  unselected steps may be NULL); keep[b] == 0 copies the row.  In-place allowed.
 */
int tio_moments(const float* src, const uint8_t* mask, int64_t n, double* out3, void* stream);
size_t tio_quantiles_workspace_bytes(void);
int tio_quantiles(const float* src, const uint8_t* mask, int64_t n, const double* q_host, int m,
                  float* values, double* weights, double* count, void* workspace,
                  size_t workspace_bytes, void* stream);
int tio_rescale(const float* src, float* dst, int B, int64_t per_elem, float lo, float hi,
                const float* sub, const float* div, const float* mul, const float* add,
                const uint8_t* keep, int flags, void* stream);

/*
 * Batched exact quantiles and histogram standardization
 * (transforms/intensity/histogram_standardization.py:216-303 of the reference, which copies every
 * element to the host for np.percentile and maps it with ~12 torch ops).
 *
 * tio_quantiles_batched: the tio_quantiles statistics for each of B elements of per_elem values
 *   (src (B, per_elem) of tio_dtype `dtype`, each value taken as `.float()` gives it; mask
 *   (B, per_elem) or NULL) and m >= 1 quantiles q_host[m] (host doubles in [0, 1]):
 *   values[B][2m] fp32, weights[B][m] fp64, count[B] fp64, has_nan[B] (NULL: not written) = 1 when
 *   a selected value is NaN.  Exact: a 3-level radix select over the order-preserving integer image
 *   of fp32, one launch per level for the whole batch; ranks with a common key prefix share a
 *   histogram; 13 quantiles per round over levels 1 and 2, more in further rounds.  No host sync.
 *   workspace: tio_quantiles_batched_workspace_bytes(B, m) device bytes, 16-byte aligned.
 *   Replaces np.percentile(flat.cpu().numpy(), ...) (histogram_standardization.py:279) and the
 *   per-image np.percentile of compute_histogram_landmarks (:100-108).
 * tio_histogram_tables: per element, np.percentile's linear value of each quantile from values /
 *   weights (d = b - a in fp32, the rest fp64, NaN when has_nan[b]), then the fp32 tables of
 *   histogram_standardization.py:283-300 for landmarks[m] (device fp32):
 *   tables[B][3(m-1)] = {slopes[m-1], intercepts[m-1], edges[m-2]}.
 * tio_histogram_map: dst[b] = slopes[bin] * x + intercepts[bin] (two roundings), bin =
 *   torch.bucketize(x, edges, right=False), x = src[b] as fp32, stored as torch's CUDA cast to
 *   `dtype` does; src == dst allowed (histogram_standardization.py:302-303 and the in-place
 *   `img_batch.data[i] = ...` of :216-227).
 */
size_t tio_quantiles_batched_workspace_bytes(int B, int m);
int tio_quantiles_batched(const void* src, int dtype, const uint8_t* mask, int B, int64_t per_elem,
                          const double* q_host, int m, float* values, double* weights, double* count,
                          uint8_t* has_nan, void* workspace, size_t workspace_bytes, void* stream);
int tio_histogram_tables(const float* values, const double* weights, const uint8_t* has_nan,
                         const float* landmarks, int B, int m, float* tables, void* stream);
int tio_histogram_map(const void* src, void* dst, int dtype, int B, int64_t per_elem,
                      const float* tables, int m, void* stream);

/*
 * Intensity chain: what Compose([BiasField, Blur, Noise, Gamma]) computes, in
 * at most two HBM passes.  Each stage is absent when its table is NULL (noise:
 * noise_mode 0), and an absent stage leaves v unchanged:
 *   K2  v   = src * exp(trilerp(coarse))   (/ when bias_divide)  if coarse != NULL
 *   K3  v   = blur_I(blur_J(blur_K(v)))                          if taps   != NULL
 *   K4  v   = v + (mean[b] + std[b] * n)   (or Rician)           if noise_mode != 0
 *   K5  dst = sign(v) |v|^gamma[b]                                if gamma  != NULL
 * A single transform runs as a call with only its own stage set.  The blur
 * passes commute up to fp32 summation order (the reference order is I, J, K).
 *   K2  replaces _apply_bias_per_element / _generate_bias_field
 *       (transforms/intensity/bias_field.py:201-255, 296-341); coarse is
 *       [B][C][si][sj][sk] fp32, drawn on the host by torch.normal from the
 *       recorded seeds (bias_field.py:281-293, 316-329)
 *   K3  see tio_blur for taps / radius / R / axes_mask
 *   K4  replaces _sample_noise + add + _restore_gated_out
 *       (transforms/intensity/noise.py:98-178); Rician:
 *       sqrt((v + n1)^2 + n2^2), n_i = mean + std * z_i
 *       noise_mode 1: standard normals supplied in z (z2 for the second Rician
 *                     draw), same shape as src; tio_randn_mt19937 replays the
 *                     reference's torch.randn(generator=CPU) stream
 *       noise_mode 2: Philox4x32-7 normals generated in registers, keyed by
 *                     philox_seed: statistically equivalent, NOT the reference stream
 *   K5  replaces data.sign() * data.abs().pow(gamma)
 *       (transforms/intensity/gamma.py:88-90)
 *   per-element identity rows (bias_identity[b], all radii 0, keep[b] == 0,
 *   gamma[b] == 1) pass through every stage as bit-exact copies
 *   scratch: B*C*I*J*K floats, required when axes_mask has bit 1 or 2 (J/K) together with
 *            bias or bit 0 (J/K alone reads src directly), or
 *            when R > 16 with blur and bias both active, or more than one axis
 * src, dst, scratch must be distinct when blur is active.
 */
int tio_intensity_fused(const float* src, float* dst, float* scratch,
                        int B, int C, int I, int J, int K,
                        const float* coarse, int si, int sj, int sk,
                        const uint8_t* bias_identity, int bias_divide,
                        const float* taps, const int32_t* radius, int R, int axes_mask,
                        const float* mean, const float* std, const uint8_t* keep,
                        const float* z, const float* z2,
                        uint64_t philox_seed, int noise_mode, int rician,
                        const float* gamma, void* stream);

/*
 * The first pass of the chain above (K2 bias and the I axis of K3: dst = what tio_intensity_fused
 * hands to its J/K pass) and z = stream elements [offset, offset+n) of tio_randn_mt19937(seed),
 * from one persistent kernel in which the two share every SM: the pass is bound by HBM, the
 * normals by instruction issue, so together they take little more than the slower one alone.
 * Both outputs are bit-identical to what tio_intensity_fused (axes_mask & 1, no noise, no gamma)
 * and tio_randn_mt19937 write.  The chain is finished by tio_intensity_fused(dst -> out) with
 * axes_mask & 6, no bias, and z as the supplied normals.
 *   taps / radius / R / axes_mask as for tio_blur; only bit 0 (the I axis) is read; R <= 6
 *   K % 4 == 0; src, dst, z 16-byte aligned; src != dst
 *   seed / offset / n / table as for tio_randn_mt19937; z holds n floats
 *   workspace  device scratch of tio_intensity_pass1_with_normals_workspace_bytes(offset, n)
 * Anything else (wider tables, ragged rows) is refused; callers then use the two calls above.
 */
size_t tio_intensity_pass1_with_normals_workspace_bytes(uint64_t offset, uint64_t n);
int tio_intensity_pass1_with_normals(const float* src, float* dst,
                                     int B, int C, int I, int J, int K,
                                     const float* coarse, int si, int sj, int sk,
                                     const uint8_t* bias_identity, int bias_divide,
                                     const float* taps, const int32_t* radius, int R, int axes_mask,
                                     uint64_t seed, uint64_t offset, uint64_t n, float* z,
                                     const void* table, void* workspace, size_t workspace_bytes,
                                     void* stream);

/*
 * LabelsToImage in one pass: dst (B, 1, vox) fp32 from channel 0 of `labels` (B, C, vox) of
 * `dtype`.  Replaces _generate_from_labels / _generate_per_element
 * (transforms/intensity/labels_to_image.py:182-290): per drawn label, in the reference's order,
 * result += (torch.randn_like(result) * std + mean) * (label == l) on a CUDA batch.
 *   label_values  [n] device int64, strictly ascending; a voxel matches l when `label == int(l)`
 *                 (fp32 maps: integral values only), n <= 2048
 *   mean, std     [B][n] device fp32 (per element; the shared form repeats one row)
 *   draw_offset   [n] device uint64: the Philox offset ATen's normal kernel would have been handed
 *                 for that label's randn_like draw, or ~0 when the label is not drawn
 *   seed          the CUDA generator's seed; grid_x the block count of ATen's launch
 *                 (min(SMs * maxThreadsPerSM / 256, ceil(B*vox / 256)))
 * Each voxel of a drawn label l is (((z + 0) * std) + mean) + 0 rounded step by step, z the
 * element ATen's draw wrote there; every other voxel is +0.  B*vox <= 2^29 (ATen splits larger
 * draws into several launches with other offsets).
 */
int tio_labels_to_image(const void* labels, int dtype, int C, int B, int64_t vox,
                        const int64_t* label_values, int n, const float* mean, const float* std,
                        const uint64_t* draw_offset, uint64_t seed, int grid_x, float* dst,
                        void* stream);

/*
 * Label-map utilities (transforms/label/ of the reference), one pass each.  Label dtypes are
 * tio_dtype codes; `src` is never modified.
 *
 * tio_label_lut: dst[e] = the value of src[e]'s key in the table, for `count` elements of `dtype`
 * (dst has the same dtype; in-place allowed).  Replaces the clone / zeros_like + one compare and one
 * masked index_put per entry of RemapLabels (remap_labels.py:50-58), RemoveLabels
 * (remove_labels.py:54-61), SequentialLabels (sequential_labels.py:53-61) and its inverse (:97-105).
 *   keys      [n] device, strictly ascending: int64 for integer maps (each key a value of the dtype),
 *             fp32 for fp32 maps (matched by value: -0 finds +0, NaN finds nothing)
 *   values    [n] device, `dtype`: what an element equal to keys[i] becomes
 *   identity  1: an element without a key is copied (RemapLabels); 0: it becomes 0 (zeros_like)
 * 8-bit maps hold at most 256 keys.
 *
 * tio_label_contour: dst (volumes, I, J, K) fp32 = 1 where the minimum of float(v) over the 3x3x3
 * neighbourhood (-1 outside the volume) differs from float(v) or is NaN, else 0; `src` is `volumes`
 * contiguous (I, J, K) volumes (B*C) of `dtype`.  Replaces _extract_contour (contour.py:52-71).
 *
 * tio_onehot_classes: dst (B, num_classes, vox) fp32 one-hot of channel 0 of `src` (B, C, vox):
 * channel c is 1 where long(v) == c (fp32: truncated as the device converts it; a class the dtype
 * cannot hold stays 0).  Replaces data.long(), F.one_hot, permute, .float() (one_hot.py:58-69).
 *
 * tio_label_range: range[0], range[1] (device int64) = the minimum and maximum of long(v) over
 * channel 0 of `src` (B, C, vox); what one_hot's range checks and num_classes=-1 read.
 *
 * tio_channel_argmax: dst (B, 1, vox) fp32 = the index of the first maximum over the C channels of
 * `src` (B, C, vox) of `dtype`, a NaN counting as the maximum (torch.argmax(dim=1)).  Replaces
 * _OneHotInverse (one_hot.py:87-97).
 */
int tio_label_lut(const void* src, void* dst, int dtype, int64_t count, const void* keys,
                  const void* values, int n, int identity, void* stream);
int tio_label_contour(const void* src, int dtype, int volumes, int I, int J, int K, float* dst,
                      void* stream);
int tio_onehot_classes(const void* src, int dtype, int B, int C, int64_t vox, int num_classes,
                       float* dst, void* stream);
int tio_label_range(const void* src, int dtype, int B, int C, int64_t vox, int64_t* range,
                    void* stream);
int tio_channel_argmax(const void* src, int dtype, int B, int C, int64_t vox, float* dst,
                       void* stream);

/*
 * Resolution changes (spatial/resize.py, spatial/anisotropy.py of the reference), one pass each on
 * the data's fp32 image: every tap is converted to fp32 and the result back to `dtype` as
 * `data.float()` ... `.to(dtype)` do.  `dtype` is any tio_dtype code (TIO_F16 / TIO_BF16 / TIO_F64
 * included); src and dst do not overlap.
 *
 * tio_interpolate: dst (volumes, OI, OJ, OK) from src (volumes, I, J, K), ATen's CUDA
 * upsample_trilinear3d (align_corners=True, `linear` = 1) or upsample_nearest3d (`linear` = 0).
 *   idx  [2*(OI+OJ+OK)] int32 device: per axis (I, then J, then K) the lower source index of each
 *        output index, then the upper one (nearest: the upper half is not read)
 *   lam  [2*(OI+OJ+OK)] fp32 device: per axis the lower weight, then the upper one (NULL: nearest)
 * out = t0*(h0*(w0*x000 + w1*x001) + h1*(w0*x010 + w1*x011)) + t1*(...), each `a*x + b*y` rounded
 * as fma(a, x, rn(b*y)), every tap read.  Replaces F.interpolate of Resize.apply_transform
 * (resize.py:71-76) and, with the nearest-down map composed into `idx`, the two F.interpolate of
 * _simulate_anisotropy (anisotropy.py:353-392).
 *
 * tio_axis_resample: dst (B, C, I, J, K) from src along one axis per batch element, Anisotropy's
 * per-instance path (_simulate_anisotropy_per_instance and its helpers, anisotropy.py:132-350).
 *   axis [B] int32 device: 0, 1 or 2, or -1 for an element copied bit for bit (factor <= 1)
 *   lo, hi [B*L] int32, w [B*L] fp32 device, L >= max(I, J, K): for element b and output index o
 *        along its axis, the source indices and weight; nearest (`linear` = 0) reads lo only
 *        (hi, w may be NULL); linear is lo*(1 - w) + hi*w in four rounded fp32 ops
 */
int tio_interpolate(const void* src, void* dst, int dtype, int volumes, int I, int J, int K, int OI,
                    int OJ, int OK, const int32_t* idx, const float* lam, int linear, void* stream);
int tio_axis_resample(const void* src, void* dst, int dtype, int B, int C, int I, int J, int K,
                      const int32_t* axis, const int32_t* lo, const int32_t* hi, const float* w, int L,
                      int linear, void* stream);

/*
 * The adjoints of tio_interpolate and tio_axis_resample for fp32 gradients, one launch each:
 * grad_in is fully written (no memset), each voxel gathered from grad_out in an order fixed by the
 * tables, with no atomics, so the result is deterministic.  Every term the forward reads is kept,
 * zero weights included, so a NaN / Inf in grad_out spreads as in the reference's backward.
 *
 * tio_interpolate_backward: grad_in (volumes, I, J, K) from grad_out (volumes, OI, OJ, OK), the
 * transpose of tio_interpolate with the same tables inverted per axis (tables.py,
 * interpolate_adjoint_tables).  Replaces ATen's upsample_trilinear3d_backward (align_corners=True)
 * and upsample_nearest3d_backward, the backward of Resize's F.interpolate and of the two
 * F.interpolate of _simulate_anisotropy.
 *   ptr  [(I+1)+(J+1)+(K+1)] int32 device: per axis (I, then J, then K) the CSR row starts of each
 *        input index, as offsets into ent / wt
 *   ent  int32 device: output index of each entry; entries of an input index in ascending output
 *   wt   fp32 device: weight of each entry (nearest: 1)
 * grad_in = sum over the three windows of ((w_i*w_j)*w_k)*g, I then J then K, each ascending.
 * volumes*I*J*ceil(K/128) must be below 2^31.
 *
 * tio_axis_resample_backward: grad_in (B, C, I, J, K) from grad_out of the same shape, the transpose
 * of tio_axis_resample with the same axis and w.  Replaces the backward of the gathers and the
 * four elementwise ops of _simulate_anisotropy_per_instance (torch.gather's scatter_add).
 *   axis [B] int32 device: as tio_axis_resample (-1: grad_in = grad_out for the element)
 *   ptr  [B*(L+1)] int32 device: for element b and input plane p along its axis, the row start of p
 *        in the element's entries
 *   ent  [B*2L] int32 device: 2*o for output o with lo[o] = p, 2*o + 1 for hi[o] = p, ascending o
 *   w    [B*L] fp32 device: the forward's weights (NULL when `linear` = 0)
 * plane p gets the sum of (1 - w[o])*g_o (lo entries, 1 - w rounded as in the forward) and w[o]*g_o
 * (hi entries); nearest (`linear` = 0) the sum of g_o; planes no output reads get 0.
 */
int tio_interpolate_backward(const float* grad_out, float* grad_in, int volumes, int I, int J, int K,
                             int OI, int OJ, int OK, const int32_t* ptr, const int32_t* ent,
                             const float* wt, void* stream);
int tio_axis_resample_backward(const float* grad_out, float* grad_in, int B, int C, int I, int J, int K,
                               const int32_t* axis, const int32_t* ptr, const int32_t* ent,
                               const float* w, int L, int linear, void* stream);

/*
 * Clamp, Mask and Swap (intensity/clamp.py, mask.py, swap.py of the reference), one launch each.
 * Image dtypes are tio_dtype codes, TIO_F16 / TIO_BF16 / TIO_F64 included.
 *
 * tio_clamp: dst = torch.clamp(src, min = *lo, max = *hi) over `count` elements.  Replaces
 * `img_batch.data.clamp(min=out_min, max=out_max)` (clamp.py:53-56).
 *   lo, hi     host pointers to one value of `dst_dtype` (the bound as torch converts it to the
 *              result dtype), or NULL for no bound; at least one is given
 *   dst_dtype  `dtype`, or TIO_F32 for an integer image clamped to a float bound (torch's promotion)
 * A NaN element stays NaN; with both bounds and either of them NaN every output is that NaN
 * (ATen's clamp_out).  In place (src == dst) when dst_dtype == dtype.
 *
 * tio_mask: torch.where(mask.expand_as(x), x, outside) over x = (B, C, vox).  Replaces
 * Mask.apply_transform (mask.py:61-97).
 *   mask        (mask_channels, vox) device, any label dtype (bool as TIO_U8); mask_channels is 1
 *               (every image channel) or C; the same mask applies to every batch element
 *   keys        n_keys < 0: a voxel is inside when it is nonzero (`.bool()`); n_keys >= 0: inside
 *               when it equals one of the ascending device keys (int64, fp32 for fp32 masks; as
 *               tio_label_lut's), so n_keys = 0 puts every voxel outside
 *   outside     host pointer to one value of `dst_dtype`
 *   dst_dtype   == dtype: in place (src NULL or == dst), only the outside voxels are written and
 *               the image is not read; TIO_F32 for an integer image (promotion by a float
 *               outside value): dst = inside ? float(src) : outside, src != dst
 *
 * tio_swap_patches: Swap's patch exchanges (swap.py:195-364), in place in `data` (B, C, I, J, K) of
 * `elem_size`-byte elements (1, 2, 4 or 8; the bytes are moved verbatim).
 *   swaps         host int32 [lists][steps][8]: ai, aj, ak, bi, bj, bk, kind, 0.  kind 0: the two
 *                 patches do not overlap (checked); 1: they may overlap, the region at b ends up
 *                 with the old patch at a and the rest of the region at a with the old patch at b;
 *                 2: no-op.  Every patch must lie inside the volume (checked before any launch).
 *   lists         1 (one list for every element) or B (element b runs list b)
 *   swaps_device  device int32 buffer of the same size; the list is copied there on `stream`
 *   stage         device scratch of B * 2 * C * pi * pj * pk elements, or NULL when no step has
 *                 kind 1
 * The steps run in order; each element's list runs on one thread-block cluster (up to 8 CTAs)
 * with a cluster barrier between steps, all elements in one launch.
 */
int tio_clamp(const void* src, void* dst, int dtype, int dst_dtype, int64_t count, const void* lo,
              const void* hi, void* stream);
int tio_mask(const void* mask, int mask_dtype, int mask_channels, const void* keys, int n_keys,
             const void* src, int dtype, void* dst, int dst_dtype, int B, int C, int64_t vox,
             const void* outside, void* stream);
int tio_swap_patches(void* data, int elem_size, int B, int C, int I, int J, int K, int pi, int pj,
                     int pk, const int32_t* swaps, int lists, int steps, int32_t* swaps_device,
                     void* stage, void* stream);

/*
 * KeepLargestComponent (label/keep_largest.py:63-125 of the reference: per element and label a
 * compare pass, a host copy, SimpleITK's ConnectedComponent + RelabelComponent, a copy back and an
 * index_put).  Here every selected label of every element is labelled in one union-find on the
 * device.  `src` / `data` is B contiguous (I, J, K) volumes of a label dtype, I*J*K < 2^32, B <= 65535.
 *
 * Which voxels take part (`mode`), with `keys` [n_keys] on the device:
 *   0  explicit labels: the value equals a key (keys as tio_label_lut's: ascending, int64, fp32 for
 *      fp32 maps; an 8-bit map holds at most 256); slot = the key's index
 *   1  labels=None on U8 / I8 / I16 maps: long(v) != background (when has_background); slot = the
 *      value (256 or 65536 slots per element)
 *   2  labels=None on I32 / I64 / F32 maps: long(v) != background, and for fp32 v finite and
 *      integral (has_background = 0 when no fp32 value equals the background label); slot = the
 *      index of v in `keys`, the ascending distinct values of the roots (tio_component_roots; int64,
 *      fp32 for fp32 maps), not needed by tio_components
 * Two neighbouring voxels that take part are connected when their values compare equal; 26
 * neighbours when `fully_connected`, else 6.
 *
 * tio_components: parent [B * I*J*K] uint32 = for a voxel that takes part, the smallest C-order
 * index (i*J + j)*K + k within its element of the voxels of its component (the root), else
 * 0xFFFFFFFF; count [B * I*J*K] uint32 = at a root, the size of its component (0 elsewhere);
 * flags [B] uint32 = per element bit 0: some voxel takes part, bit 1: a NaN, bit 2: a +-Inf.
 *
 * tio_component_roots: values (at least B*vox elements of `dtype`) = the value of every root, in no
 * particular order; *n_values (device) = how many.
 *
 * tio_keep_largest: in place, every voxel that takes part and is not in its (element, slot)'s
 * largest component (ties: the smallest root) becomes *fill (host pointer to one value of
 * `dtype`: what `t[mask] = background_label` stores); no other voxel is written.  parent / count
 * from tio_components on the same data; winner: device scratch of B * slots uint64 (slots =
 * n_keys, or 256 / 65536 for mode 1).
 */
int tio_components(const void* src, int dtype, int B, int I, int J, int K, int mode, const void* keys,
                   int n_keys, int64_t background, int has_background, int fully_connected,
                   uint32_t* parent, uint32_t* count, uint32_t* flags, void* stream);
int tio_component_roots(const void* src, int dtype, int B, int64_t vox, const uint32_t* parent,
                        void* values, uint32_t* n_values, void* stream);
int tio_keep_largest(void* data, int dtype, int B, int64_t vox, int mode, const void* keys,
                     int n_keys, int64_t background, int has_background, const uint32_t* parent,
                     const uint32_t* count, uint64_t* winner, const void* fill, void* stream);

/*
 * Spike (intensity/spike.py:124-223 of the reference: fftn of data.float(), fftshift, peak =
 * |spectrum|.amax() per (b, c), spectrum[idx] += peak * intensity per spike, ifftshift, ifftn, .real,
 * .to(dtype), torch.where for per-instance gating).  A spike at the fftshift index p of an axis of n
 * points is frequency f = (p - n / 2) mod n, and its inverse FFT is a plane wave, so
 *   out[b, c, i, j, k] = x + A[b, c] * sum_s cos(2 pi (u_s i / I + v_s j / J + w_s k / K)),
 *   A[b, c] = peak[b, c] * intensity[b] / (I J K),
 * with x = float(data) and peak = sum(x) when no voxel of the row is negative.  `data` / `src` is a
 * contiguous (B, C, I, J, K) batch of any tio_dtype; B * C <= 65535.  `intensity` is device fp32 [B]:
 * an element with intensity 0 is not active, and no call reads or writes its voxels.
 *
 * tio_spike_stats: per row r = b * C + c, sum[r] (device fp64) = sum of float(x) and flags[r]
 * (device uint32) = bit 0: some voxel < 0, bit 1: some voxel is NaN or +-Inf; both 0 for an inactive
 * row.  workspace: device scratch of tio_spike_stats_workspace_bytes(B * C) bytes.  The sum is
 * added in a fixed order: the same input gives the same bits.
 *
 * tio_spectrum_peak: peak[r] (device fp32) = max |fftn(float(x))| of every active row whose flags
 * are exactly 1 (signed and finite), 0 for the others; the rows are chosen on the device.
 * Forward half-spectrum FFT (bins 0..K/2 on the last axis hold every magnitude of a real input):
 * a K pass from the input, an in-place J pass and an I pass that only reduces, over a complex64
 * workspace of [rows][I][J][K/2 + 1]; rows are processed in chunks of workspace_bytes /
 * (I * J * (K/2 + 1) * 8), at least one.  Every axis is at most 4096 points.
 *
 * tio_spike: in place, each voxel of an active row gets x + A cos(...) cast back as the reference's
 * .to(dtype); a row with flags bit 1 becomes all NaN (the reference's FFT spreads the value).
 *   spikes  device int32 [B][S][4]: u, v, w (frequencies, 0 <= f < axis length), 1; an element's
 *           list is followed by (0, 0, 0, 0) padding up to the longest list
 *   sum, flags, peak  from tio_spike_stats / tio_spectrum_peak; A uses peak when flags bit 0 is set
 *   tables  device scratch of B * S * (I + J + K) * 8 bytes: the per-axis phase tables
 *           exp(2 pi i (f n mod L) / L), kept in shared memory when one element's fit in 96 KiB
 */
size_t tio_spike_stats_workspace_bytes(int rows);
int tio_spike_stats(const void* src, int dtype, int B, int C, int64_t vox, const float* intensity,
                    double* sum, uint32_t* flags, void* workspace, size_t workspace_bytes,
                    void* stream);
int tio_spectrum_peak(const void* src, int dtype, int B, int C, int I, int J, int K,
                      const float* intensity, const uint32_t* flags, float* peak, void* workspace,
                      size_t workspace_bytes, void* stream);
int tio_spike(void* data, int dtype, int B, int C, int I, int J, int K, const int32_t* spikes, int S,
              const float* intensity, const double* sum, const uint32_t* flags, const float* peak,
              void* tables, size_t tables_bytes, void* stream);

/*
 * Ghosting (intensity/ghosting.py:149-277 of the reference: fftn of data.float(), fftshift, times a
 * real mask that varies along one axis, ifftshift, ifftn, .real, .to(dtype), torch.where for
 * per-instance gating).  The FFTs over the other two axes cancel, so each line along the ghosted
 * axis (n points) becomes
 *   out = Re(ifft_n(H fft_n(x))) = ifft_n(Hs fft_n(x)),   Hs(f) = (H(f) + H(-f mod n)) / 2,
 * with x = float(data) and H = ifftshift(line_mask) (ghosting.py:190-197, 251-271).  In place on a
 * contiguous (B, C, I, J, K) batch of any tio_dtype; B * C <= 65535.
 *   table   device fp32 [B][n_max]: element b's H in unshifted order in its first n entries
 *   axis    device int32 [B]: element b's ghosted axis (0 = I, 1 = J, 2 = K)
 *   active  device uint8 [B]: 0 = not active, no voxel of the element is read or written
 *   axes    bit a set for each axis some active element ghosts (1..7): one launch per set bit;
 *           each of these axes is at most 4096 points and at most n_max
 *   flags   device scratch of B * C uint32
 * A row with a NaN or +-Inf voxel becomes all NaN (the reference's FFT spreads the value).
 */
int tio_ghosting(void* data, int dtype, int B, int C, int I, int J, int K, const float* table, int n_max,
                 const int32_t* axis, const uint8_t* active, int axes, uint32_t* flags, void* stream);

/*
 * Motion (intensity/motion.py:140-561 of the reference: fftn of data.float(); for each of N rigid
 * transforms, affine_grid + grid_sample (trilinear, zeros padding, align_corners=True), fftn, and
 * the first-axis k-space rows [s size, (s + 1) size) copied in (the last segment ends at I, with
 * size = I // (N + 1)); ifftn, .real, .to(dtype), torch.where for per-instance gating).  The FFTs
 * over J and K cancel, so each line along I becomes
 *   out = ifft_I(sum_s Hs_s fft_I(x_s)),   Hs_s(f) = (P_s(f) + P_s(-f mod I)) / 2,
 * with x_0 = float(data), x_s its resampled copies and P_s the indicator of segment s's rows.  Out
 * of place on contiguous (B, C, I, J, K) batches of any tio_dtype (in and out must not overlap);
 * I <= 4096, 2 <= segments <= I, B * C <= 65535.
 *   segments  N + 1
 *   theta     device fp32 [B][N][12]: segment s's affine_grid matrix (3 x 4, row major) of element b
 *             at [b][s - 1]; output voxel (i, j, k) samples theta (lin_K[k], lin_J[j], lin_I[i], 1)
 *             in the (K, J, I) frame, lin_n = linspace(-1, 1, n)
 *   active    device uint8 [B]: 0 = gated out, the element is copied bit for bit
 *   flags     device scratch of B * C uint32
 * A row with a NaN or +-Inf voxel becomes all NaN (the reference's FFT spreads the value).
 */
int tio_motion(const void* in, void* out, int dtype, int B, int C, int I, int J, int K, int segments,
               const float* theta, const uint8_t* active, uint32_t* flags, void* stream);

/*
 * PatchAggregator (data/aggregator.py of the reference), one launch per key and batch.
 *
 * tio_aggregate_patches adds the first `n` patches of a batch `patches` (B, C, pi, pj, pk) into the
 * buffer `out` (C, I, J, K), in table order, as the reference's add_batch -> _add_patch does one
 * patch at a time (aggregator.py:75-100, 143-237):
 *   mode 0 crop     out[box] = patch[src box]; where boxes overlap, the last one wins
 *   mode 1 average  out[box] += patch, counts[box] += 1, both in the buffer's dtype
 *   mode 2 hann     out[box] += patch * window, counts[box] += window, window = (w_i w_j) w_k in fp32
 *                   (fp64 for an fp64 buffer), rounded once to the buffer's dtype
 * Integer adds wrap; fp16 / bf16 are computed in fp32 and rounded after each add, as ATen's CPU
 * ops do.  Voxels no box covers are not written.  No atomics: the result does not depend on
 * scheduling.
 *   dtype          tio_dtype code of patches, out and counts; bool moves as TIO_U8 in crop mode;
 *                  hann needs TIO_F32, TIO_F16, TIO_BF16 or TIO_F64
 *   counts         (1, I, J, K) device, one channel for every channel of `out` (the reference
 *                  keeps C equal channels); NULL in crop mode
 *   boxes          HOST int32 [n][10]: dst lo i, j, k, dst hi i, j, k (exclusive), src lo i, j, k,
 *                  patch row in 0..B-1; every box non-empty, inside the buffer and inside its patch
 *                  (checked before any launch); source extent = destination extent
 *   boxes_device   the same table in device memory (the kernel reads it there)
 *   window         device fp32 [pi + pj + pk]: torch.hann_window(n + 2, periodic=False)[1:-1] of
 *                  each patch axis in turn (aggregator.py:239-245); NULL unless mode is hann
 *
 * tio_aggregate_finish writes out / counts.clamp(min=1) (aggregator.py:117-120) into `dst`, the
 * single-channel count broadcast over the C channels of `out` (C, vox).  `dst` has the buffer's
 * dtype, or fp32 for an integer buffer (true division of integers).
 */
int tio_aggregate_patches(const void* patches, void* out, void* counts, int dtype, int mode, int C, int I,
                          int J, int K, int B, int pi, int pj, int pk, int n, const int32_t* boxes,
                          const int32_t* boxes_device, const float* window, void* stream);
int tio_aggregate_finish(const void* out, const void* counts, void* dst, int dtype, int C, int64_t vox,
                         void* stream);

/*
 * PCA (intensity/pca.py of the reference: per element, A = (voxels x channels) float(x) minus its
 * channel means, torch.pca_lowrank(A, q), A @ V, whitening, normalising and the values_range map).
 * `src` is a contiguous (B, C, vox) batch of any tio_dtype, read as `data.float()`; B <= 65535.  The
 * three passes below are the only reads of the volume; the C x q algebra between them runs on the
 * host.  Both reductions add fixed-order block partials (no float atomics): the same input gives the
 * same bits.
 *
 * tio_pca_workspace_bytes: device scratch that tio_pca_mean and tio_pca_gram_apply need for this
 * shape (the larger of the two); one workspace serves both passes of a stream in turn.
 *
 * tio_pca_mean: mean[b * C + c] (device fp64) = the mean of float(x) over the element's voxels.
 *
 * tio_pca_gram_apply: out[b][c][k] (device fp64) = sum_v d[v][c] (sum_c' d[v][c'] w[b][c'][k]), that
 * is G W with G = A^T A, for d = float(x) - mean in fp64; w is device fp64 [B][C][q], 1 <= q <= 6144.
 *
 * tio_pca_project: out[b][k][v] (device fp32) = sum_c (float(x) - (float)mean) * coef[b][c][k] +
 * offset, in fp32, clamped to [0, 1] when `clip` (NaN stays NaN); coef is device fp32 [B][C][q].
 */
size_t tio_pca_workspace_bytes(int B, int C, int q, int64_t vox);
int tio_pca_mean(const void* src, int dtype, int B, int C, int64_t vox, double* mean, void* workspace,
                 size_t workspace_bytes, void* stream);
int tio_pca_gram_apply(const void* src, int dtype, int B, int C, int64_t vox, int q, const double* mean,
                       const double* w, double* out, void* workspace, size_t workspace_bytes, void* stream);
int tio_pca_project(const void* src, int dtype, int B, int C, int64_t vox, int q, const double* mean,
                    const float* coef, float offset, int clip, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TIO_B200_H */
