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
int tio_resample(const void* src, void* dst, int dtype,
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
 *   R         table half-width (max radius over the whole table)
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
 * noise.py:166-178).  Writes stream elements [offset, offset+n) to z[0..n).
 * Requires offset % 16 == 0, n % 16 == 0, n >= 16 (ragged tails and tiny draws
 * stay on the host), and offset + n <= 2^31 words.
 *   table      device copy of the jump-ahead table built once by
 *              tio_mt19937_build_table (host, ~2 s; depends only on MT19937, so
 *              callers cache it; tio_mt19937_table_bytes() gives its size)
 *   workspace  device scratch of tio_randn_mt19937_workspace_bytes(offset, n)
 * The uniforms are bit-identical to torch.s; normals agree to <= 4e-6 absolute
 * (CUDA libm vs the host.s log/sin/cos).
 */
size_t tio_mt19937_table_bytes(void);
int tio_mt19937_build_table(void* host_blob, size_t bytes);
size_t tio_randn_mt19937_workspace_bytes(uint64_t offset, uint64_t n);
int tio_randn_mt19937(uint64_t seed, uint64_t offset, uint64_t n, float* z,
                      const void* table, void* workspace, size_t workspace_bytes,
                      void* stream);

/*
 * Data-derived parameters of Standardize / Normalize, computed where the batch lives
 * (the reference reads batch element 0 on the host: standardize.py:52-79, normalize.py:121-139,
 * 332-366, _statistics.py:11-45).
 *   tio_moments    out3 (device doubles) = {sum, sum of squares, count} of the `n` values at `src`
 *                  for which mask[t] != 0 (mask NULL = all); fp64 accumulation, one pass
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
 *   scratch: B*C*I*J*K floats, required when axes_mask has bit 1 or 2 (J/K)
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

#ifdef __cplusplus
}
#endif
#endif /* TIO_B200_H */
