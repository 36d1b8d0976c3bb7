/*
 * b200raster.h -- C ABI of libb200raster.so, the H100 (sm_90a) differentiable
 * mesh rasterizer that drops in behind Jittor/jrender's rasterizer Functions.
 *
 * Every entry point replaces one `jt.code(...)` op of the reference (paths are
 * relative to the reference checkout):
 *
 *   b200r_softras_forward   <- jrender/renderer/dr/softras/cuda/soft_rasterize.py:3-521
 *                              (forward_soft_rasterize: memsets + K1 + K2), called from
 *                              jrender/renderer/dr/softras/soft_rasterize.py:75-82; also
 *                              serves the bin_size>0 call site (:91-99,
 *                              soft_rasterize_coarse_to_fine.py:7-879) -- binning is
 *                              internal here and exact, so one entry point covers both.
 *   b200r_softras_backward  <- jrender/renderer/dr/softras/cuda/soft_rasterize.py:966-1416
 *                              (backward_soft_rasterize, top-K), called from
 *                              jrender/renderer/dr/softras/soft_rasterize.py:125-132.
 *   b200r_nmr_forward       <- jrender/renderer/dr/n3mr/cuda/rasterize.py:5-217 and :219-339
 *                              (forward_face_index_map + forward_texture_sampling),
 *                              called from jrender/renderer/dr/n3mr/n3mr.py:125-133.
 *   b200r_nmr_backward      <- jrender/renderer/dr/n3mr/cuda/rasterize.py:342-648, :650-727,
 *                              :729-822 (backward_pixel_map, backward_textures,
 *                              backward_depth_map), called from n3mr.py:29-67.
 *   b200r_vol_composite_forward / _backward  <- jrender_vol/integrator/integrator.py:18-39 (about 15 elementwise ops and
 *                              their autograd)
 *   b200r_vol_resample      <- jrender_vol/integrator/sample.py:28-57 and jrender_vol/rayMarching/rayMarching.py:65-71
 *                              (mids, sample_pdf, argsort of the concat)
 *   (the other entry points name their reference code in their own comments below)
 *
 * Conventions
 *   - All tensor pointers are DEVICE pointers owned by the caller (contiguous, fp32 /
 *     int32).  No allocation and no host synchronisation happens inside; all work is
 *     enqueued on `stream` (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   - Scalar parameters are runtime arguments (the reference bakes them into JIT source).
 *   - Return 0 on success; a negative B200R_E* code for argument errors; a positive
 *     cudaError_t for CUDA failures.  b200r_last_error() returns a thread-local message.
 *   - There is no CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef B200RASTER_H
#define B200RASTER_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200R_API __attribute__((visibility("default")))
#else
#define B200R_API
#endif

#define B200R_EINVAL (-1)      /* bad argument (NULL pointer, size, enum out of range) */
#define B200R_EWORKSPACE (-2)  /* workspace too small */
#define B200R_EUNSUPPORTED (-3)

/* enum values = the reference's maps, jrender/renderer/dr/softras/soft_rasterize.py:39-42 */
enum { B200R_DIST_HARD = 0, B200R_DIST_BARYCENTRIC = 1, B200R_DIST_EUCLIDEAN = 2 };
enum { B200R_RGB_HARD = 0, B200R_RGB_SOFTMAX = 1, B200R_RGB_NONE = 2 };
enum { B200R_ALPHA_HARD = 0, B200R_ALPHA_SUM = 1, B200R_ALPHA_PROD = 2 };
enum { B200R_TEX_SURFACE = 0, B200R_TEX_VERTEX = 1 };

#define B200R_MAX_FACES_PER_PIXEL 64 /* kMaxPointsPerPixel, cuda/soft_rasterize.py:16 */

B200R_API const char* b200r_version(void);
B200R_API const char* b200r_last_error(void);

/* Device memory of one forward / backward pair, in two caller-allocated blocks:
 *   state      b200r_softras_state_bytes(batch, num_faces): written by the forward, handed to the backward -- the per-face
 *              records (what the reference keeps in `faces_info`, soft_rasterize.py:62,101) and the backward's gradient
 *              accumulator.  208 bytes per (batch, face).
 *   workspace  b200r_softras_workspace_bytes(batch, num_faces, image_size): transient scratch of the forward only (binning
 *              lists in a pool of 512-id chunks budgeted at 8 list entries per face -- bins that find the pool exhausted
 *              are flagged and their blocks filter the whole face list, so nothing is ever dropped -- and the block
 *              queue); free to be released or reused once the forward has been enqueued.  ~12 MB for 4 x 1024^2 images of
 *              39 200 faces. */
B200R_API size_t b200r_softras_workspace_bytes(int batch_size, int num_faces, int image_size);
B200R_API size_t b200r_softras_state_bytes(int batch_size, int num_faces);

/* SoftRas forward.
 *   face_vertices  [B, nf, 3, 3]  NDC x,y (+y up) and camera-space z per vertex
 *   textures       [B, nf, T, 3]  T = R*R texels (surface) or 3 (vertex)
 *   soft_colors    [B, 4, H, W]   out, planar RGBA, row 0 = top (y = +1)
 *   aggrs_info     [B, 2, H, W]   out: softmax -> (sum, max); hard rgb -> (depth_min, face_index_min)
 *   faces_id_buffer[B, K, H, W]   out, int32, the <=K nearest-z face ids per pixel in the
 *                                 reference's slot order, -1 TERMINATED: slots [0, n) hold ids, slot n (if n < K) is
 *                                 -1, and the slots behind it are left untouched (the reference memsets all of them
 *                                 to -1, soft_rasterize.py:470; the backward only ever reads up to the first -1,
 *                                 :1236-1237, and so does b200r_softras_backward).  Nothing to initialise on the caller's
 *                                 side.
 *   faces_info     [B, nf, 27]    out, optional (may be NULL): the reference's K1 output
 *   dist_eps_logit = ln(1/dist_eps - 1) computed by the host as soft_rasterize.py:25
 * Background colour is always 0, as in the reference (the op memsets soft_colors). */
B200R_API int b200r_softras_forward(const float* face_vertices, const float* textures,
                          float* soft_colors, float* aggrs_info, int32_t* faces_id_buffer,
                          float* faces_info, void* state, size_t state_bytes,
                          void* workspace, size_t workspace_bytes,
                          int batch_size, int num_faces, int texture_size, int image_size,
                          int max_faces_per_pixel, float near, float far, float eps,
                          float sigma_val, float gamma_val, float dist_eps_logit,
                          int dist_func, int rgb_func, int alpha_func, int texture_type,
                          int double_side, void* stream);

/* SoftRas top-K backward.  grad_face_vertices [B,nf,3,3] and grad_textures [B,nf,T,3]
 * are overwritten (zeroed inside, then accumulated). */
B200R_API int b200r_softras_backward(const float* face_vertices, const float* textures,
                           const float* soft_colors, const float* aggrs_info,
                           const int32_t* faces_id_buffer, void* state,
                           size_t state_bytes, const float* grad_soft_colors,
                           float* grad_face_vertices, float* grad_textures,
                           int batch_size, int num_faces, int texture_size, int image_size,
                           int max_faces_per_pixel, float near, float far, float eps,
                           float sigma_val, float gamma_val, float dist_eps_logit,
                           int dist_func, int rgb_func, int alpha_func, int texture_type,
                           int double_side, void* stream);

/* Anti-aliased flavours (SURVEY.md section 8f rank 2): replace SoftRasterizer.execute's "render at 2 x image_size, then
 * 2x2 mean-pool" (jrender/renderer/dr/softras/rasterizer.py:45,54-55) without the extra passes.  image_size is the
 * SUPERSAMPLED size (even).  forward_aa additionally writes pooled_colors [B,4,image_size/2,image_size/2], the 2x2 means of
 * soft_colors, from the forward kernel's output staging (soft_colors is still written: the backward reads it);
 * backward_aa takes grad_pooled_colors [B,4,image_size/2,image_size/2] and forms avg_pool2d's backward (grad / 4 at each
 * of the four source pixels) while loading, instead of materialising a 4x larger gradient tensor. */
B200R_API int b200r_softras_forward_aa(const float* face_vertices, const float* textures, float* soft_colors,
                           float* pooled_colors, float* aggrs_info, int32_t* faces_id_buffer, float* faces_info,
                           void* state, size_t state_bytes, void* workspace, size_t workspace_bytes,
                           int batch_size, int num_faces, int texture_size, int image_size,
                           int max_faces_per_pixel, float near, float far, float eps,
                           float sigma_val, float gamma_val, float dist_eps_logit,
                           int dist_func, int rgb_func, int alpha_func, int texture_type,
                           int double_side, void* stream);
B200R_API int b200r_softras_backward_aa(const float* face_vertices, const float* textures,
                           const float* soft_colors, const float* aggrs_info,
                           const int32_t* faces_id_buffer, void* state,
                           size_t state_bytes, const float* grad_pooled_colors,
                           float* grad_face_vertices, float* grad_textures,
                           int batch_size, int num_faces, int texture_size, int image_size,
                           int max_faces_per_pixel, float near, float far, float eps,
                           float sigma_val, float gamma_val, float dist_eps_logit,
                           int dist_func, int rgb_func, int alpha_func, int texture_type,
                           int double_side, void* stream);

/* ---- NMR (dr_type='n3mr') hard rasterizer -------------------------------------------------
 * Maps keep the reference kernels' orientation [B, yi, xi] with yi UP (row 0 = bottom); the
 * vertical flip to image orientation belongs to the caller (n3mr.py:239-247).
 *   faces               [B, nf, 3, 3]
 *   textures            [B, nf, ts, ts, ts, 3]           (return_rgb)
 *   face_index_map      [B, H, W] int32, -1 = background
 *   weight_map          [B, H, W, 3]      depth_map [B, H, W] (far where uncovered)
 *   rgb_map             [B, H, W, 3]      already mixed with background_rgb (host float[3], may be NULL = black)
 *   alpha_map           [B, H, W]         (face_index >= 0)
 *   sampling_index_map  [B, H, W, 8] int32, sampling_weight_map [B, H, W, 8]
 *   face_inv_map        [B, H, W, 9]      (return_depth)
 * Equal-depth ties are won by the lowest face id (the reference's winner is race-dependent). */
B200R_API size_t b200r_nmr_workspace_bytes(int batch_size, int num_faces, int image_size);
B200R_API int b200r_nmr_forward(const float* faces, const float* textures, int32_t* face_index_map,
                                float* weight_map, float* depth_map, float* rgb_map, float* alpha_map,
                                int32_t* sampling_index_map, float* sampling_weight_map, float* face_inv_map,
                                void* workspace, size_t workspace_bytes, int batch_size, int num_faces,
                                int texture_size, int image_size, float near, float far, float eps,
                                const float* background_rgb, int return_rgb, int return_alpha,
                                int return_depth, void* stream);
/* grad_faces [B,nf,3,3] and grad_textures [B,nf,ts,ts,ts,3] are overwritten.  Sub-ops follow
 * n3mr.py:29-67: pixel-map gradient (x,y) -> texture gradient -> depth gradient accumulated in place.
 * `scratch` (b200r_nmr_backward_scratch_bytes) holds the packed row-/column-major pixel records the
 * pixel-map gradient scans; it is only needed when return_rgb or return_alpha. */
B200R_API size_t b200r_nmr_backward_scratch_bytes(int batch_size, int image_size);
B200R_API int b200r_nmr_backward(const float* faces, const int32_t* face_index_map, const float* weight_map,
                                 const float* depth_map, const float* rgb_map, const float* alpha_map,
                                 const int32_t* sampling_index_map, const float* sampling_weight_map,
                                 const float* face_inv_map, const float* grad_rgb_map,
                                 const float* grad_alpha_map, const float* grad_depth_map, float* grad_faces,
                                 float* grad_textures, void* scratch, size_t scratch_bytes,
                                 int batch_size, int num_faces, int texture_size,
                                 int image_size, float eps, int return_rgb, int return_alpha,
                                 int return_depth, void* stream);

/* ---- fused pre-raster geometry stage (SURVEY.md section 8f rank 1) ------------------------------
 * World-space vertices -> camera space -> projection -> per-face gather in ONE launch.  Replaces
 * the tensor-op chain of jrender/renderer/transform/look_at.py:24-38 (or look.py:23-53),
 * transform/perspective.py:11-16 / orthogonal.py:12-15 and structures/utils/faces_vertices.py:14-19,
 * called from transform/transform.py:52-58 and structures/mesh.py (face_vertices property).
 *   vertices       [vertices_batch, nv, 3]   world space; vertices_batch = B, or 1 = shared mesh
 *   faces          [faces_batch, nf, 3] int32; faces_batch = B or 1; an index outside [0, nv) makes
 *                  that corner NaN (the reference reads out of bounds)
 *   eye            [eye_batch, 3] device; eye_batch = B or 1
 *   face_vertices  [B, nf, 3, 3]   out: x, y projected (perspective: X/Z/width; orthogonal: X*scale), z = camera Z
 *   at_or_direction, up: HOST float[3] (look_at: the `at` point; look: the viewing direction)
 *   width_or_scale: tan(viewing_angle) (perspective.py:11-12) or viewing_scale (orthogonal)
 * The backward overwrites grad_vertices [vertices_batch, nv, 3] with the sum over every (batch, face,
 * corner) that references the vertex (float atomics).  No gradient for eye / at / up. */
enum { B200R_CAM_LOOK_AT = 0, B200R_CAM_LOOK_RIGHT = 1, B200R_CAM_LOOK_LEFT = 2 };
enum { B200R_PROJ_PERSPECTIVE = 0, B200R_PROJ_ORTHOGONAL = 1 };
B200R_API int b200r_project_faces_forward(const float* vertices, const int32_t* faces, const float* eye,
                                          float* face_vertices,
                                          const float* at_or_direction, const float* up, float width_or_scale,
                                          int camera_mode, int projection, int batch_size, int num_vertices,
                                          int num_faces, int vertices_batch, int faces_batch, int eye_batch, void* stream);
B200R_API int b200r_project_faces_backward(const float* vertices, const int32_t* faces, const float* eye,
                                           const float* grad_face_vertices, float* grad_vertices,
                                           const float* at_or_direction, const float* up, float width_or_scale,
                                           int camera_mode, int projection, int batch_size, int num_vertices,
                                           int num_faces, int vertices_batch, int faces_batch, int eye_batch, void* stream);

/* ---- fused mesh regularisers of the fitting loop (SURVEY.md section 8f rank 4) ---------------------
 * Each call writes loss [B] AND d(loss_b)/d(vertices) [B, nv, 3] (both overwritten) in one launch.
 *   b200r_flatten_loss   <- jrender/loss/flatten_loss.py:38-79; v0s..v3s [E] int32 = the edge table the
 *                           reference builds at :14-36 (edge v0-v1 shared by the faces with apexes v2, v3)
 *   b200r_laplacian_loss <- jrender/loss/laplacian_loss.py:29-36 with the row-normalised Laplacian of :11-27
 *                           stored as a padded neighbour table: (L x)_i = diag[i] x_i + sum_k w[i,k] x[nbr[i,k]],
 *                           neighbours / neighbour_weights [nv, max_degree] (weight 0 = padding), diag [nv] */
B200R_API int b200r_flatten_loss(const float* vertices, const int32_t* v0s, const int32_t* v1s, const int32_t* v2s,
                                 const int32_t* v3s, float* loss, float* grad_vertices, int batch_size,
                                 int num_vertices, int num_edges, float eps, void* stream);
B200R_API int b200r_laplacian_loss(const float* vertices, const int32_t* neighbours, const float* neighbour_weights,
                                   const float* diag, float* loss, float* grad_vertices, int batch_size,
                                   int num_vertices, int max_degree, void* stream);

/* ---- texture baking (SURVEY.md section 8f rank 3) -------------------------------------------------------------
 * Replaces _load_textures_for_softras / load_textures_cuda_kernel (jrender/io/utils/load_textures.py:3-101):
 * image [H, W, 3] f32 (already flipped vertically by the caller, _load_obj_for_softras.py:136), faces_uv [nf, 3, 2],
 * is_update [nf] int32, textures [nf, R*R, 3] updated in place where is_update != 0.  Device pointers. */
B200R_API int b200r_bake_textures_softras(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                          int nf, int texture_res, int image_height, int image_width, void* stream);
/* The adjoint of b200r_bake_textures_softras: overwrites grad_image [H, W, 3] with the gradient of the baked textures
 * grad_textures [nf, R*R, 3] (faces with is_update == 0 contribute nothing), scattered with the forward's bilinear weights
 * into the pixels it read (out-of-image taps clamped to the last element, as there).  Nothing flows to faces_uv.
 * Accumulates with float atomics, so the summation order may vary between runs.  Device pointers. */
B200R_API int b200r_bake_textures_softras_backward(const float* grad_textures, const float* faces_uv, const int32_t* is_update,
                                                   float* grad_image, int nf, int texture_res, int image_height,
                                                   int image_width, void* stream);
/* Replaces _load_textures_for_n3mr / load_textures_cuda_kernel (jrender/io/utils/load_textures.py:103-246), the bake of
 * the NMR rasterizer's [nf, ts, ts, ts, 3] textures: texel (a, b, c) samples the image at the barycentric point
 * (a, b, c) / (ts - 1) normalised to sum 1, through the face's wrapped UVs.  texture_wrapping: 0 REPEAT, 1 MIRRORED_REPEAT,
 * 2 CLAMP_TO_EDGE, 3 CLAMP_TO_BORDER (writes zeros, like the reference); use_bilinear: bilinear (1) or nearest (0) fetch.
 * texture_size >= 2 (the reference divides by texture_size - 1).  faces_uv is read-only here (the reference wraps it in
 * place from every thread of the face, a race).  textures updated in place where is_update != 0. */
B200R_API int b200r_bake_textures_n3mr(const float* image, const float* faces_uv, const int32_t* is_update, float* textures,
                                       int nf, int texture_size, int image_height, int image_width, int texture_wrapping,
                                       int use_bilinear, void* stream);

/* ---- texture-atlas export (the inverse of the bake) ------------------------------------------------------------
 * Replaces create_texture_image_cuda_kernel (jrender/io/utils/create_texture_image.py:3-104), called from
 * create_texture_image, jrender/io/save_obj.py:7-29: paints every face's texels into its texture_res_out^2 tile of
 * image [H, W, 3] f32 (W = tile_width * texture_res_out; face fn owns tile (fn % tile_width, fn / tile_width); rows top
 * down, the caller flips), through the face's tile triangle tile_vertices [nf, 3, 2] in pixel units.  Every pixel is
 * written: those of tiles past the last face are set to 1.  texture_res_out must be 2 or >= 4 (at 3 the tile triangle
 * is degenerate).  Device pointers.
 *   softras: textures [nf, R*R, 3], R = texture_res >= 1; each pixel copies one texel (the texel index is clamped to
 *            the face's own texels, where the reference reads unchecked).
 *   n3mr:    textures [nf, ts, ts, ts, 3], ts = texture_size >= 2; each pixel samples the face's volume trilinearly at
 *            its barycentric weights times (ts - 1), as the NMR forward sampler does (no reference counterpart). */
B200R_API int b200r_texture_atlas_softras(const float* tile_vertices, const float* textures, float* image, int nf,
                                          int texture_res, int texture_res_out, int tile_width, int image_height,
                                          int image_width, void* stream);
B200R_API int b200r_texture_atlas_n3mr(const float* tile_vertices, const float* textures, float* image, int nf,
                                       int texture_size, int texture_res_out, int tile_width, int image_height,
                                       int image_width, void* stream);

/* ---- mesh voxelization -----------------------------------------------------------------------------------------
 * Replaces jrender/renderer/utils/voxelization.py:1-57 and its four kernels (renderer/utils/cuda/voxelization.py).
 * voxels [B, vs, vs, vs] int32 is indexed [b, c0, c1, c2] in the faces' coordinate order; 1 <= vs <= 1024.
 *   surface: faces [B, nf, 3, 3] f32 in voxel units (already scaled).  Zeroes voxels, then sets the surface voxels of
 *            all three axes (voxelize_sub1: integer columns (y, x), the four voxels around each accepted column) and the
 *            voxel of every face corner (voxelize_sub2).  Bit-equal to the reference's all-columns loop in unfused
 *            float32; a non-finite depth writes nothing.
 *   fill:    in place: voxels becomes 1 - visible, visible = empty (== 0) voxels 6-connected through empty voxels to
 *            the grid boundary (voxelize_sub3/4 and the host loop).  No host synchronisation; workspace of
 *            b200r_voxelize_workspace_bytes(B, vs) bytes (0 for out-of-range arguments). */
B200R_API size_t b200r_voxelize_workspace_bytes(int batch_size, int voxel_size);
B200R_API int b200r_voxelize_surface(const float* faces, int32_t* voxels, int batch_size, int num_faces, int voxel_size,
                                     void* stream);
B200R_API int b200r_voxelize_fill(int32_t* voxels, void* workspace, size_t workspace_bytes, int batch_size, int voxel_size,
                                  void* stream);

/* ---- fused surface-mode lighting of the pre-raster stage (SURVEY.md section 8f rank 1) -------------------------
 * Replaces Lighting.execute with light_mode='surface', no normal map, no SSS, one directional light:
 *   jrender/renderer/lighting/lighting.py:186-204, ambient_lighting.py:4-9, directional_lighting.py:54-135
 *   (diffuse branch, and the Cook-Torrance branch when with_specular and eye / metallic / roughness are given),
 *   surface normals of jrender/structures/mesh.py:213-229.
 * vertices [vertices_batch, nv, 3] world space, faces [faces_batch, nf, 3] int32, textures / out_textures
 * [B, nf, T, 3] (T = texture_res^2, or ts^3 for n3mr), metallic / roughness [B, nf, Tm] or NULL, eye [eye_batch, 3]
 * (eye_batch 0: none).  Batches of 1 broadcast.  ambient_color, directional_color, direction: HOST pointers to 3 floats
 * (direction already normalised).  backward overwrites grad_textures [B, nf, T, 3], grad_vertices
 * [vertices_batch, nv, 3], and grad_metallic / grad_roughness [B, nf, Tm] (each NULL: not needed).  A material gradient
 * is the gradient of the face's mean material value spread evenly over its Tm texels; it is 0 where the Cook-Torrance
 * branch is off (with_specular 0 or no eye).  Material gradients need metallic, roughness and Tm > 0 (else B200R_EINVAL). */
B200R_API int b200r_surface_lighting_forward(const float* vertices, const int32_t* faces, const float* textures, const float* metallic,
                                             const float* roughness, const float* eye, float* out_textures, int B, int vertices_batch,
                                             int faces_batch, int eye_batch, int nv, int nf, int T, int Tm, float ambient_intensity,
                                             const float* ambient_color, float directional_intensity, const float* directional_color,
                                             const float* direction, int with_specular, void* stream);
B200R_API int b200r_surface_lighting_backward(const float* vertices, const int32_t* faces, const float* textures, const float* metallic,
                                              const float* roughness, const float* eye, const float* grad_out, float* grad_textures,
                                              float* grad_vertices, float* grad_metallic, float* grad_roughness, int B,
                                              int vertices_batch, int faces_batch, int eye_batch, int nv, int nf, int T, int Tm,
                                              float ambient_intensity, const float* ambient_color, float directional_intensity,
                                              const float* directional_color, const float* direction, int with_specular, void* stream);

/* ---- normal-mapped surface lighting ---------------------------------------------------------------------------------
 * Lighting.execute's normal-map branch (jrender/renderer/lighting/lighting.py:186-204 with mesh.normal_textures, and the
 * 4-D branch of directional_lighting.py:63-135): one normal per texel, N = normalize(n_t . TBN) (structures/mesh.py:276-284,
 * surface_ResNormals), the face centroid as position, and per-texel metallic / roughness (not averaged).  One thread per
 * texel forward.  Same light parameters and batch rules as b200r_surface_lighting_*; in addition
 *   textures / out_textures [B, nf, T, 3], normal_textures [normal_batch, normal_faces, normal_texels, 3] (tangent space),
 *   tbn [tbn_batch, tbn_faces, 3, 3] (rows T, B, N), metallic / roughness [B, nf, T] or NULL.
 * normal_batch and tbn_batch are 1 or B; normal_faces, normal_texels and tbn_faces must equal nf and T (else B200R_EINVAL).
 * backward overwrites each of grad_textures [B, nf, T, 3], grad_normal_textures [normal_batch, nf, T, 3] (summed over the
 * batch when normal_batch is 1), grad_vertices [vertices_batch, nv, 3] (through the centroid only) and the per-texel
 * grad_metallic / grad_roughness [B, nf, T] that is not NULL.  No gradient reaches the TBN.  Material gradients need
 * metallic and roughness (else B200R_EINVAL); they are 0 where the Cook-Torrance branch is off. */
B200R_API int b200r_normal_mapped_lighting_forward(const float* vertices, const int32_t* faces, const float* textures,
                                                   const float* normal_textures, const float* tbn, const float* metallic,
                                                   const float* roughness, const float* eye, float* out_textures, int B,
                                                   int vertices_batch, int faces_batch, int eye_batch, int normal_batch,
                                                   int normal_faces, int normal_texels, int tbn_batch, int tbn_faces, int nv, int nf,
                                                   int T, float ambient_intensity, const float* ambient_color,
                                                   float directional_intensity, const float* directional_color,
                                                   const float* direction, int with_specular, void* stream);
B200R_API int b200r_normal_mapped_lighting_backward(const float* vertices, const int32_t* faces, const float* textures,
                                                    const float* normal_textures, const float* tbn, const float* metallic,
                                                    const float* roughness, const float* eye, const float* grad_out,
                                                    float* grad_textures, float* grad_normal_textures, float* grad_vertices,
                                                    float* grad_metallic, float* grad_roughness, int B, int vertices_batch,
                                                    int faces_batch, int eye_batch, int normal_batch, int normal_faces,
                                                    int normal_texels, int tbn_batch, int tbn_faces, int nv, int nf, int T,
                                                    float ambient_intensity, const float* ambient_color,
                                                    float directional_intensity, const float* directional_color,
                                                    const float* direction, int with_specular, void* stream);

/* ---- normal and depth G-buffers (Lighting(Gbuffer='normal' | 'depth')) ----------------------------------------------
 * jrender/renderer/lighting/lighting.py:180-204 with directional_lighting.py:136-144: the textures become ones and the
 * light terms are replaced, out = clamp(1 * value + 1 * (specular * 0), 0, 1), value = N * 0.5 + 0.5 (mode 0, normal) or
 * z / M in all three channels (mode 1, depth), z the camera depth of the face centroid and M the max of z over every
 * (batch, face), NaN if any z is.  specular is the Cook-Torrance term of b200r_surface_lighting_* (0 without that
 * branch): multiplied by 0, it only matters where it is not finite.
 * b200r_gbuffer_lighting_*: the flat branch.  Same vertices / faces / metallic / roughness / eye / batch / T / Tm rules
 * and light parameters as b200r_surface_lighting_* (no ambient: it does not reach the result), out_textures [B, nf, T, 3]
 * (T = texture_res^2, or ts^3 for n3mr).  Depth also needs camera_eye [camera_eye_batch, 3] (1 or B), the camera
 * (camera_mode B200R_CAM_*, camera_at_or_direction and camera_up: HOST pointers to 3 floats, as b200r_project_faces_*),
 * a device workspace of b200r_gbuffer_workspace_floats(B, nf) floats (else B200R_EWORKSPACE) and a device float
 * depth_max; normal mode ignores all four.  Forward: one launch (normal) or two (depth); the depth workspace then holds
 * each face's z, which the backward takes as face_depth together with depth_max.  Backward: grad_vertices
 * [vertices_batch, nv, 3] and grad_metallic / grad_roughness [B, nf, Tm] (each NULL: not needed); two launches for depth
 * (a workspace of its own, same size), one for normal.  The max's gradient goes in full to every face whose z equals
 * M.  Material gradients are 0, or NaN where a partial of the specular term is not finite.  No host synchronisation.
 * b200r_normal_mapped_gbuffer_*: the normal-map branch, mode normal only, N = normalize(n_t . TBN) per texel;
 * normal_textures [normal_batch, nf, T, 3], tbn [tbn_batch, nf, 3, 3], metallic / roughness [B, nf, T] per texel,
 * backward writes grad_normal_textures (summed over the batch when normal_batch is 1), grad_vertices (through the
 * specular term only) and the per-texel material gradients, each NULL: not needed. */
B200R_API size_t b200r_gbuffer_workspace_floats(int batch_size, int num_faces);
B200R_API int b200r_gbuffer_lighting_forward(const float* vertices, const int32_t* faces, const float* metallic,
                                             const float* roughness, const float* eye, const float* camera_eye,
                                             float* out_textures, float* workspace, size_t workspace_floats, float* depth_max,
                                             int mode, int B, int vertices_batch, int faces_batch, int eye_batch,
                                             int camera_eye_batch, int nv, int nf, int T, int Tm, float directional_intensity,
                                             const float* directional_color, const float* direction, int with_specular,
                                             const float* camera_at_or_direction, const float* camera_up, int camera_mode,
                                             void* stream);
B200R_API int b200r_gbuffer_lighting_backward(const float* vertices, const int32_t* faces, const float* metallic,
                                              const float* roughness, const float* eye, const float* camera_eye,
                                              const float* grad_out, const float* face_depth, const float* depth_max,
                                              float* workspace, size_t workspace_floats, float* grad_vertices,
                                              float* grad_metallic, float* grad_roughness, int mode, int B, int vertices_batch,
                                              int faces_batch, int eye_batch, int camera_eye_batch, int nv, int nf, int T,
                                              int Tm, float directional_intensity, const float* directional_color,
                                              const float* direction, int with_specular, const float* camera_at_or_direction,
                                              const float* camera_up, int camera_mode, void* stream);
B200R_API int b200r_normal_mapped_gbuffer_forward(const float* vertices, const int32_t* faces, const float* normal_textures,
                                                  const float* tbn, const float* metallic, const float* roughness,
                                                  const float* eye, float* out_textures, int B, int vertices_batch,
                                                  int faces_batch, int eye_batch, int normal_batch, int tbn_batch, int nv,
                                                  int nf, int T, float directional_intensity, const float* directional_color,
                                                  const float* direction, int with_specular, void* stream);
B200R_API int b200r_normal_mapped_gbuffer_backward(const float* vertices, const int32_t* faces, const float* normal_textures,
                                                   const float* tbn, const float* metallic, const float* roughness,
                                                   const float* eye, const float* grad_out, float* grad_normal_textures,
                                                   float* grad_vertices, float* grad_metallic, float* grad_roughness, int B,
                                                   int vertices_batch, int faces_batch, int eye_batch, int normal_batch,
                                                   int tbn_batch, int nv, int nf, int T, float directional_intensity,
                                                   const float* directional_color, const float* direction, int with_specular,
                                                   void* stream);

/* ---- NeRF volume rendering (jrender_vol) -------------------------------------------------------------------------
 * One warp per ray; no atomics, no host synchronisation, no workspace.  Every ray holds at most B200R_VOL_MAX_SAMPLES
 * samples (S for compositing, S + Ni for resampling); beyond that the calls return B200R_EUNSUPPORTED.  num_rays 0 is a
 * no-op.  Device pointers, float32, contiguous.
 *
 * b200r_vol_composite_forward replaces integrator() (jrender_vol/integrator/integrator.py:5-39):
 *   raw [N, S, C] (C >= 4; channels 0-2 colour logits, 3 density, the rest ignored), z_vals [N, S], rays_d [N, 3],
 *   noise [N, S] already scaled by raw_noise_std, or NULL -> rgb_map [N, 3], disp_map [N], acc_map [N], weights [N, S],
 *   depth_map [N].  The reference's float32 expressions unfused: last interval 1e10 * |d|, alpha = 1 - exp(-relu(sigma +
 *   noise) dist), exclusive product of (1 - alpha) + 1e-10.  disp = 1 / max(1e-10, depth / acc) with jt.maximum read as
 *   std::max(1e-10, q), which does not propagate NaN: a ray with acc == 0 gets disp = 1e10, not NaN.
 * b200r_vol_composite_backward: the gradient of those five outputs (each upstream gradient may be NULL = zero) with
 *   respect to raw, written to grad_raw [N, S, C] (channels >= 4 zero).  acc_map / depth_map are the forward's (needed
 *   with grad_disp_map).  Nothing flows to z_vals, rays_d or noise; disp passes gradient only where 1e-10 < depth / acc.
 * b200r_vol_resample replaces sample_pdf() (jrender_vol/integrator/sample.py:28-57) and the fine stage of render_rays
 *   (jrender_vol/rayMarching/rayMarching.py:65-71): weights + 1e-5, cdf, searchsorted(right=True), denom < 1e-5 -> 1.
 *   u [N, Ni] uniform draws, or NULL for det (u = linspace(0, 1, Ni)).  Two shapes of call:
 *     fine stage:  z_vals [N, S] (num_bins = S >= 2), weights [N, S] the coarse weights; bins are the mids of z_vals and
 *                  the pdf uses weights[:, 1:S-1].  Writes z_samples [N, Ni] and z_vals_fine [N, S + Ni], the ascending
 *                  sort of the concatenation (NaN last).  bins must be NULL.
 *     sample_pdf:  bins [N, num_bins] (>= 1), weights [N, num_bins - 1]; z_vals and z_vals_fine NULL; writes z_samples. */
#define B200R_VOL_MAX_SAMPLES 1024
B200R_API int b200r_vol_composite_forward(const float* raw, const float* z_vals, const float* rays_d, const float* noise,
                                          float* rgb_map, float* disp_map, float* acc_map, float* weights, float* depth_map,
                                          int num_rays, int num_samples, int raw_channels, int white_bkgd, void* stream);
B200R_API int b200r_vol_composite_backward(const float* raw, const float* z_vals, const float* rays_d, const float* noise,
                                           const float* acc_map, const float* depth_map, const float* grad_rgb_map,
                                           const float* grad_disp_map, const float* grad_acc_map, const float* grad_weights,
                                           const float* grad_depth_map, float* grad_raw, int num_rays, int num_samples,
                                           int raw_channels, int white_bkgd, void* stream);
B200R_API int b200r_vol_resample(const float* z_vals, const float* bins, const float* weights, const float* u,
                                 float* z_samples, float* z_vals_fine, int num_rays, int num_bins, int num_importance,
                                 void* stream);

/* ---- texture-space subsurface scattering ---------------------------------------------------------------------------
 * Replaces the map stages of SSS (jrender/renderer/lighting/lighting.py:108-150): computeStretchMap
 * (renderer/utils/ToStretchMap.py:5-13) and the gaussian_blur / _blur_for_SSS ops (renderer/utils/gaussian_blur.py:4-204).
 * Maps are float32 device planes [H, W], row 0 = the top row of the SoftRas image they were rasterized into; [3, H, W]
 * inputs are planar (the first three planes of a SoftRas soft_colors [4, H, W] can be passed as they are).  Gradients: the
 * _backward entry points below.
 *   b200r_sss_stretch: world_map [3, H, W] (world coordinates, before the reference's `* 7`) -> stretch_u, stretch_v
 *       [H, W]: 1 / |7 (w(y, x) - w(y, x + 1))| and 1 / |7 (w(y, x) - w(y + 1, x))| with the last column / row replicated,
 *       each clamped to [0, 1].  One launch.
 *   b200r_sss_blur_pyramid: for each level i < num_levels, stretch_u <- blur_x(stretch_u, mod = stretch_u),
 *       irr <- blur_x(irr, mod = stretch_u), stretch_v <- blur_y(stretch_v, mod = stretch_v), irr <- blur_y(irr, mod =
 *       stretch_v), final_c += weights[c * num_levels + i] * irr_c; then final = final * irradiance_map + specular_map,
 *       written to out_map [H, W, 3] with the rows flipped.  The blurs are the reference kernels' 7-tap modulated blurs
 *       with taps [num_levels][7] and tap_widths [num_levels] (GaussWidth); taps, tap_widths and weights [3][num_levels]
 *       are HOST arrays.  irradiance_map and specular_map [3, H, W]; stretch_u / stretch_v are read only.  The maps must be
 *       square (the reference's y kernel clamps rows against the width); 1 <= num_levels <= 8.  2 * num_levels launches.
 *       workspace: b200r_sss_workspace_bytes(H, W) bytes (13 maps; 0 for non-positive sizes). */
B200R_API size_t b200r_sss_workspace_bytes(int height, int width);
B200R_API int b200r_sss_stretch(const float* world_map, float* stretch_u, float* stretch_v, int height, int width, void* stream);
B200R_API int b200r_sss_blur_pyramid(const float* stretch_u, const float* stretch_v, const float* irradiance_map,
                                     const float* specular_map, float* out_map, void* workspace, size_t workspace_bytes,
                                     const float* taps, const float* tap_widths, const float* weights, int num_levels,
                                     int height, int width, void* stream);
/* Gradients (Lighting.sss_grad):
 *   b200r_sss_stretch_backward: overwrites grad_world_map [3, H, W] with the gradient of world_map through
 *       b200r_sss_stretch, given grad_stretch_u / grad_stretch_v [H, W].  Where a clamp is active (including every
 *       face's inside, where the difference is 0) the gradient is 0.  No atomics; one launch.
 *   b200r_sss_blur_pyramid_backward: given the forward's inputs stretch_u, stretch_v, irradiance_map [3, H, W] and
 *       grad_out [H, W, 3] (rows flipped, as out_map), overwrites grad_irradiance_map and grad_specular_map [3, H, W], and,
 *       when both are non-NULL, grad_stretch_u / grad_stretch_v [H, W] (both NULL: the stretch maps' gradients and their
 *       modulation terms are not computed).  The gradients are taken at the forward's decisions (tap indices, clamps,
 *       the <= 1e-6 replacements and the centre test).  Same taps, tap_widths, weights, num_levels and square-map rule
 *       as the forward, and width <= 8192.  workspace: b200r_sss_backward_workspace_bytes(H, W, num_levels) bytes
 *       ((8 num_levels + 10) maps; 0 for out-of-range arguments), else B200R_EWORKSPACE.  The forward's 2 * num_levels
 *       launches again, then 2 * num_levels backward launches; y-pass gradients are summed with float atomics, so the
 *       order of the sums may vary between runs. */
B200R_API size_t b200r_sss_backward_workspace_bytes(int height, int width, int num_levels);
B200R_API int b200r_sss_stretch_backward(const float* world_map, const float* grad_stretch_u, const float* grad_stretch_v,
                                         float* grad_world_map, int height, int width, void* stream);
B200R_API int b200r_sss_blur_pyramid_backward(const float* stretch_u, const float* stretch_v, const float* irradiance_map,
                                              const float* grad_out, float* grad_irradiance_map, float* grad_specular_map,
                                              float* grad_stretch_u, float* grad_stretch_v, void* workspace,
                                              size_t workspace_bytes, const float* taps, const float* tap_widths,
                                              const float* weights, int num_levels, int height, int width, void* stream);

/* ---- screen-space image passes (render2) --------------------------------------------------------------------------
 * Replace SSAO_cuda, SSDO_cuda and FXAA_cuda (jrender/render2/utils/cuda/{SSAO,SSDO,FXAA}_cuda.py).  Images are square,
 * image_size x image_size pixels, HWC, row 0 at the top; 1 <= image_size and 3 * image_size^2 <= INT_MAX.  One launch
 * each; no gradients.
 *   b200r_ssao: depth [is, is] (view-space z), face_ind [is, is] int32 (-1 = background), normals [is, is, 3] (view
 *       space) -> occlusion [is, is]: for each covered pixel, the share of sample_num points drawn in a half ball of radius
 *       sample_range_r around the pixel's view-space point (x, y = NDC * width * z) whose projection lands on a pixel in
 *       front of it; 0 on the background.  Pixel i draws from curand XORWOW curand_init(1, i, 0), x, y, z per sample,
 *       as the reference does, so the results are the reference's bit for bit.  sample_num >= 0 (0 gives NaN).
 *   b200r_ssdo: the same samples; color [is, is, 3] -> image [is, is, 3]: the ambient share (samples whose pixel is no
 *       more than 0.01 in front of them) times the colour, plus one bounce of indirect light from the other samples'
 *       pixels; the background passes the colour through.
 *   b200r_fxaa: texture [is, is, 3] -> image [is, is, 3], the reference's FXAA: its edge search never moves (see
 *       DESIGN.md), so a pixel is either kept or resampled bilinearly at the sub-pixel offset across its edge.  Reads only
 *       inside the image; the taps the reference reads past the last row count as 0, as they have weight 0 there.
 * The three launches are profiled under B200R_K_SSS, the id of the image passes. */
B200R_API int b200r_ssao(const float* depth, const int32_t* face_ind, const float* normals, float* occlusion,
                         int image_size, int sample_num, float sample_range_r, float width, void* stream);
B200R_API int b200r_ssdo(const float* color, const float* depth, const int32_t* face_ind, const float* normals,
                         float* image, int image_size, int sample_num, float sample_range_r, float width, void* stream);
B200R_API int b200r_fxaa(const float* texture, float* image, int image_size, void* stream);

/* Launch counter: number of kernels this library has launched in this process
 * (bench.py reports the delta over the timed region as "gpu_launches"). */
B200R_API unsigned long long b200r_launch_count(void);

/* Tuning knobs (process-wide):
 *   "softras_exact_tail"     1 = the reference's double-precision sigmoid / alpha-product tails bit for bit;
 *                            0 (default) = the same expressions in fp32 for the default euclidean+softmax
 *                            mode (<= 1 ulp on D; all index / depth outputs are identical either way)
 *   "softras_list_pool_chunks" >= 0 caps the binning-list chunk pool (exercises the pool-exhausted path in tests);
 *                            -1 (default) = the size b200r_softras_workspace_bytes accounts for; results are
 *                            identical for every setting */
B200R_API int b200r_set_option(const char* name, int value);

/* Per-kernel device timing (CUDA events recorded on the launch stream around every kernel
 * this library launches; each launch is counted under exactly one id).  Off by default.  bench.py
 * uses it for the roofline of the dominant kernel; b200r_profile_read synchronises the outstanding
 * events.  Ids are 0 .. B200R_K_COUNT - 1. */
enum { B200R_K_FACE_SETUP = 0, B200R_K_COARSE_BIN = 1, B200R_K_SOFTRAS_FWD = 2, B200R_K_SOFTRAS_BWD = 3,
       B200R_K_TILE_ORDER = 4, B200R_K_NMR_SETUP = 5, B200R_K_NMR_FWD = 6, B200R_K_NMR_BWD_PIXEL = 7,
       B200R_K_NMR_BWD_MAPS = 8, B200R_K_SOFTRAS_BWD_FINALIZE = 9, B200R_K_NMR_PACK = 10,
       B200R_K_PROJECT_FWD = 11, B200R_K_PROJECT_BWD = 12, B200R_K_FLATTEN_LOSS = 13, B200R_K_LAPLACIAN_LOSS = 14,
       B200R_K_LIGHTING = 15, B200R_K_BAKE = 16, B200R_K_ATLAS = 17, B200R_K_VOXEL_SURFACE = 18,
       B200R_K_VOXEL_FILL = 19, B200R_K_CHUNK_RECTS = 20, B200R_K_DEBUG = 21, B200R_K_VOL_COMPOSITE_FWD = 22,
       B200R_K_VOL_COMPOSITE_BWD = 23, B200R_K_VOL_RESAMPLE = 24, B200R_K_SSS = 25, B200R_K_COUNT };
B200R_API void b200r_profile_enable(int on);
B200R_API void b200r_profile_reset(void);
B200R_API int b200r_profile_read(int kernel, double* total_ms, long long* launches);

/* Test hook: checks the exact-arithmetic helpers (csrc/exact_math.cuh) against the plain
 * IEEE expressions they replace on n (a[i], b[i]) pairs; mismatch7[0..5] count bit
 * differences (must all be 0), mismatch7[6] counts pairs that took the reciprocal fast path. */
B200R_API int b200r_debug_exact_math(const float* a, const float* b, int n, int* mismatch7, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RASTER_H */
