/*
 * genre_b200.h — C ABI of libgenre_b200.so (sm_90a).
 *
 * This is the drop-in boundary for the GenRe/ShapeHD geometric-projection hot path.  Every entry
 * point takes plain device pointers, sizes, element strides and a cudaStream_t (passed as void*);
 * there are no torch types.  The caller (the Python mirror of the reference's toolbox packages, or
 * any other host) owns every buffer, including scratch ("workspace"): the library never allocates
 * device memory and never synchronises the device.  All launches go to the given stream and are
 * CUDA-graph capturable.
 *
 * Each function states the reference interface it replaces (paths relative to the reference root).
 * Reference convention: cffi functions on THCudaTensor*, returning int 1, failing through
 * THError("aborting") (toolbox/cam_bp/cam_bp/src/back_projection.c:9-57).  Here: return 0 on success,
 * a positive cudaError_t if a launch failed, or a negative GENRE_B200_E* code for an argument error;
 * genre_b200_last_error() gives the message (thread-local).  The Python mirror turns non-zero into
 * RuntimeError, which is what THError became on the Python side.
 *
 * All tensors are fp32 unless stated otherwise.  "strides" are in ELEMENTS, not bytes, and may be 0
 * (broadcast) where noted.
 */
#ifndef GENRE_B200_H
#define GENRE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GENRE_B200_OK 0
#define GENRE_B200_EINVAL (-1)      /* bad shape / null pointer / unsupported size        */
#define GENRE_B200_EWORKSPACE (-2)  /* workspace too small (see *_workspace_bytes)         */
#define GENRE_B200_EALIGN (-3)      /* a dense buffer is not 16-byte aligned               */

/* flags for the projection entry points */
#define GENRE_B200_FLAG_SHIFT_TDF 1u /* fuse Camera_back_projection_layer.shift_tdf: 1 - R*tdf */
#define GENRE_B200_FLAG_OVERLAP 2u  /* cam_bp_forward, experimental: project and splat overlapped in ONE kernel (interleaved block
                                      order, per-map completion counters).  Slower than back to back on the GPU it was
                                      written for and not measured on the H100, so off by default */

const char *genre_b200_last_error(void);
/* library/ABI version: major*1000 + minor */
int genre_b200_version(void);

/* ---------------------------------------------------------------------------------------------
 * Camera back-projection, depth -> voxel TDF.
 * Replaces back_projection_forward (toolbox/cam_bp/cam_bp/src/back_projection.h:1,
 * back_projection.c:9-17, back_projection_kernel.cu:199-306,760-838) together with the dense
 * initialisation the Python caller performs (functions/cam_back_projection.py:22-24) and, when
 * GENRE_B200_FLAG_SHIFT_TDF is set, modules/camera_backprojection_module.py:26-28.
 *
 *   depth   [N, C, H, W]  any strides (sN,sC,sH,sW); ray depth, pixels with depth < 0 are skipped
 *   fl      [N, C]        strides (fN, fC)     focal length in pixels
 *   camdist [N, C]        strides (dN, dC)     camera distance from the origin along -x
 *   tdf     [N, C, R, R, R] dense, 16-byte aligned, written completely (no pre-initialisation needed)
 *             without SHIFT: mean point-to-centre distance on hit voxels, 1/R elsewhere
 *             with    SHIFT: 1 - R*mean on hit voxels, 1 - R*(1/R) elsewhere
 *   cnt     [N, C, R, R, R] dense or NULL; if given, the per-voxel point count as fp32 (what the
 *             reference keeps on ctx for backward, cam_back_projection.py:28)
 *   workspace: genre_b200_voxelize_workspace_bytes(N*C, H*W, R) bytes, 16-byte aligned
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_voxelize_workspace_bytes(int64_t n_maps, int64_t pixels_per_map, int res);

int genre_b200_cam_bp_forward(const float *depth, int64_t N, int64_t C, int64_t H, int64_t W,
                              int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                              const float *fl, int64_t fN, int64_t fC,
                              const float *camdist, int64_t dN, int64_t dC,
                              float *tdf, float *cnt, int res, unsigned flags,
                              void *workspace, size_t workspace_bytes, void *stream);

/* Replaces back_projection_backward (back_projection.h:2, back_projection_kernel.cu:365-471,897-963)
 * with the intended cam_dist indexing (the reference reads cam_dist with cnt's strides at :401).
 *   cnt, grad_tdf [N,C,R,R,R] dense;  grad_depth [N,C,H,W] dense (fully written);
 *   grad_fl, grad_camdist [N,C] dense (fully written). */
int genre_b200_cam_bp_backward(const float *depth, int64_t N, int64_t C, int64_t H, int64_t W,
                               int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                               const float *fl, int64_t fN, int64_t fC,
                               const float *camdist, int64_t dN, int64_t dC,
                               const float *cnt, const float *grad_tdf, int res,
                               float *grad_depth, float *grad_fl, float *grad_camdist, void *stream);

/* Replaces get_surface_mask (back_projection.h:3, back_projection_kernel.cu:309-358,840-891).
 *   cnt  [N,C,R,R,R] dense (from genre_b200_cam_bp_forward);  mask [N,C,R,R,R] dense, fully written:
 *   1 everywhere except empty voxels that lie behind the observed depth surface. */
int genre_b200_surface_mask(const float *depth, int64_t N, int64_t C, int64_t H, int64_t W,
                            int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                            const float *fl, int64_t fN, int64_t fC,
                            const float *camdist, int64_t dN, int64_t dC,
                            const float *cnt, float *mask, int res, void *stream);

/* Posed multi-view back-projection: V depth maps per grid, each from its own camera, fused into one TDF grid.
 *   depth   [N, V, H, W]  any strides (sN,sV,sH,sW); ray depth from the view's eye, pixels with depth < 0 skipped
 *   fl[n*fN + v*fV], rot + n*rN + v*rV (9 floats), eye + n*eN + v*eV (3 floats): view (n, v)'s camera in the frame
 *           of genre_b200_render_views_forward (rot row-major, its columns the camera's axes in the grid frame: x
 *           forward, image w towards -y, image h towards -z; eye the camera's centre).  Strides in elements; 0 over n
 *           shares one camera set across the batch.
 *   tdf, cnt [N, 1, R, R, R] as genre_b200_cam_bp_forward (cnt may be NULL); flags: GENRE_B200_FLAG_SHIFT_TDF only.
 *   workspace genre_b200_voxelize_workspace_bytes(N, V*H*W, R) bytes.
 * Pixel (h, w) of view v is unprojected into the camera frame exactly as genre_b200_cam_bp_forward does (z = d cos,
 * cy = (imw * -z) / fl, cz = (imh * -z) / fl), then moved into the grid frame in fp32, every operation rounded to
 * nearest in this order:  g_i = fma(rot[i][2], cz, fma(rot[i][1], cy, rot[i][0] * z)) + eye_i.  The voxel index,
 * centre distance and quantisation are genre_b200_cam_bp_forward's, and the point lies on
 * genre_b200_render_views_forward's ray of that pixel at t = d.  All V views of grid n are splatted into grid n: a
 * voxel's value is the mean distance over every point any view put in it, and the integer sums make the output
 * bitwise reproducible and independent of the order of the views.  rot = I and eye = (-cam_dist, 0, 0) reproduce
 * genre_b200_cam_bp_forward bit for bit.  Limits: 1 <= N, V <= 65535, V*H*W < 2^20 (the splat's 20-bit count),
 * every input pointer 4-byte aligned (else GENRE_B200_EALIGN); arguments are checked before any launch.
 * Two kernel launches. */
int genre_b200_cam_bp_views_forward(const float *depth, int64_t N, int64_t V, int64_t H, int64_t W,
                                    int64_t sN, int64_t sV, int64_t sH, int64_t sW,
                                    const float *fl, int64_t fN, int64_t fV,
                                    const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                    float *tdf, float *cnt, int res, unsigned flags,
                                    void *workspace, size_t workspace_bytes, void *stream);
/* The depth gradient of the above: grad_depth [N, V, H, W] dense, fully written, from cnt and grad_tdf [N, 1, R, R, R]
 * dense.  The formula is genre_b200_cam_bp_backward's with the ray direction (-fl, imw, imh) / len rotated by rot in
 * the forward's fma order; at the identity pose it equals that backward's grad_depth bit for bit.  fl, rot and eye are
 * not differentiated.  One kernel launch. */
int genre_b200_cam_bp_views_backward(const float *depth, int64_t N, int64_t V, int64_t H, int64_t W,
                                     int64_t sN, int64_t sV, int64_t sH, int64_t sW,
                                     const float *fl, int64_t fN, int64_t fV,
                                     const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                     const float *cnt, const float *grad_tdf, int res, float *grad_depth, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Spherical back-projection, spherical depth map -> voxel TDF + count.
 * Replaces spherical_back_proj_forward / _backward (back_projection.h:4-5,
 * back_projection_kernel.cu:474-757; functions/sperical_to_tdf.py:13-47).
 *   sph  [N, C, H, W]    any strides; radius along the ray, < 0 skipped
 *   grid [N, C, H, W, 3] any strides (gN may be 0: one direction table shared by the batch)
 *   tdf, cnt [N,C,R,R,R] dense, fully written: mean distance / count on hit voxels, 0 elsewhere
 * ------------------------------------------------------------------------------------------- */
int genre_b200_sph_bp_forward(const float *sph, int64_t N, int64_t C, int64_t H, int64_t W,
                              int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                              const float *grid, int64_t gN, int64_t gC, int64_t gH, int64_t gW, int64_t gD,
                              float *tdf, float *cnt, int res,
                              void *workspace, size_t workspace_bytes, void *stream);

int genre_b200_sph_bp_backward(const float *sph, int64_t N, int64_t C, int64_t H, int64_t W,
                               int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                               const float *grid, int64_t gN, int64_t gC, int64_t gH, int64_t gW, int64_t gD,
                               const float *cnt, const float *grad_tdf, int res,
                               float *grad_sph, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Stop probability along rays.  Replaces calc_prob_forward / calc_prob_backward
 * (toolbox/calc_prob/calc_prob/src/calc_prob.h:1-2, calc_prob_kernel.cu:112-266).
 *   prob_in, stop_prob, grad_in...: [n_rays, Z] dense (the reference's [N,C,X,Y,Z] flattened)
 *   forward : stop[z] = p[z] * prod_{k<z} (1 - p[k])        (p must lie in (0,1), as the reference)
 *   backward: grad_prob from stop_prob_weighted = stop * grad_stop (calc_prob.py:27)
 * ------------------------------------------------------------------------------------------- */
int genre_b200_calc_prob_forward(const float *prob_in, float *stop_prob, int64_t n_rays, int64_t Z, void *stream);
int genre_b200_calc_prob_backward(const float *prob_in, const float *stop_prob_weighted, float *grad_prob,
                                  int64_t n_rays, int64_t Z, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Fused spherical renderer: voxel occupancy -> spherical depth map.
 * Replaces render_spherical.forward (toolbox/spherical_proj.py:62-72): trilinear grid_sample
 * (align_corners=True semantics of torch 0.4.1, zero padding) of vox.permute(0,1,4,3,2) along
 * rays dir[h,w]*2*(1 - k/(Z-1)), clamp to [1e-5, 1-1e-5], stop-probability scan, expected depth
 * sum_k s_k*k/(Z-1) + prod_k(1 - p_k), without materialising any [N,1,S,S,Z] tensor.
 *   vox  [N, R, R, R] dense (C must be 1 as in the reference)
 *   dirs [S, S, 3]    dense fp64 unit directions (the numpy table of spherical_proj.py:43-51 BEFORE its
 *                     float cast; sample positions are formed in fp64 and rounded once, like :52-57)
 *   depth_weight [Z]  the module's registered buffer linspace(0,1,Z) (spherical_proj.py:58)
 *   out  [N, S, S]    dense
 * ------------------------------------------------------------------------------------------- */
int genre_b200_render_spherical_forward(const float *vox, int64_t N, int res,
                                        const double *dirs, int sph_res, int z_res,
                                        const float *depth_weight, float *out, void *stream);
/* gradient of the above w.r.t. vox; grad_vox [N,R,R,R] must be zeroed by the caller (accumulated with
 * atomics, like grid_sampler_3d_backward); z_res <= 256 */
int genre_b200_render_spherical_backward(const float *vox, int64_t N, int res,
                                         const double *dirs, int sph_res, int z_res,
                                         const float *depth_weight,
                                         const float *grad_out, float *grad_vox, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Camera-view renderer of voxel grids and the differentiable ray-consistency loss (no reference
 * counterpart: the reference's util/util_reproj.py attempt is not called by any model).
 *
 * The camera is cam_bp's: at (-cam_dist, 0, 0) looking along +x, focal length fl in pixels.  Pixel
 * (h, w) of an H x W map casts the ray o + t u, u = (fl, -imw, -imh) / |(fl, imw, imh)|,
 * imh = h - (H-1)/2, imw = w - (W-1)/2, so the point genre_b200_cam_bp_forward places from pixel
 * (h, w) at ray depth d lies on this ray at t = d.  Z samples t_k = cam_dist - sqrt(3)/2 +
 * k sqrt(3)/(Z-1) (t_0 only for Z = 1) cover the unit cube for every ray.  Voxel (i, j, l) of vox[n]
 * sits at cam_bp's voxel centre ((i+0.5)/R - 0.5, (j+0.5)/R - 0.5, (l+0.5)/R - 0.5): a point g is
 * sampled trilinearly at voxel coordinate f = (g + 0.5) R - 0.5 with zero padding (not
 * render_spherical's align_corners mapping: this op inverts cam_bp).  Then, as render_spherical,
 *   p_k = clamp(raw_k, 1e-5, 1 - 1e-5),  T_k = prod_{j<k} (1 - p_j),  s_k = p_k T_k,
 * and a ray's value is the expected cost  sum_k s_k c_k + T_Z c_esc.
 *
 * Arithmetic of the sample coordinate: fp64, every operation rounded to nearest, in the order
 *   nrm = sqrt((fl*fl + imw*imw) + imh*imh);  u = (fl/nrm, -imw/nrm, -imh/nrm)
 *   t = (cam_dist - sqrt(3)/2) + k * (sqrt(3)/(Z-1));  g = (t*ux - cam_dist, t*uy, t*uz)
 *   f = (g + 0.5) * R - 0.5
 * (fl, cam_dist widened exactly from fp32; sqrt(3) the nearest double), then f and t are each
 * rounded once to fp32.  Everything after the coordinate is fp32.
 *
 *   vox  [N, R, R, R] dense (C = 1), 2 <= R <= 1024;  fl, camdist [N] with strides fN, dN (0: shared)
 *   1 <= H, W <= 16384;  1 <= z_res <= 4096;  every pointer 4-byte aligned (else GENRE_B200_EALIGN)
 *   outputs and upstream gradients [N, H, W] dense; grad_vox [N,R,R,R] dense, zeroed by the caller
 *   (accumulated with fp32 atomics: not bitwise repeatable, and a contribution or sum below 2^-126
 *   is flushed to zero).  The forwards are bitwise repeatable and
 *   each ray's value does not depend on the batch.  No allocation, no synchronisation.
 * The gradient w.r.t. p_k is T_k c_k - (sum_{j>k} s_j c_j + T_Z c_esc) / (1 - p_k), zero where the
 * clamp is active (and at NaN samples, which render as p = 1e-5), scattered through the tap weights.
 * ------------------------------------------------------------------------------------------- */
/* depth = sum_k s_k t_k + T_Z bg,  silhou = 1 - T_Z */
int genre_b200_render_camera_forward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                     const float *fl, int64_t fN, const float *camdist, int64_t dN, float bg,
                                     float *depth, float *silhou, void *stream);
int genre_b200_render_camera_backward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                      const float *fl, int64_t fN, const float *camdist, int64_t dN, float bg,
                                      const float *grad_depth, const float *grad_silhou, float *grad_vox,
                                      void *stream);
/* Differentiable ray consistency (Tulsiani et al., CVPR 2017) against an observed ray-depth map
 * obs [N, H, W] with any strides (oN, oH, oW): per ray the expected cost with
 *   obs > 0 (foreground):  c_k = |t_k - obs|, c_esc = miss_cost
 *   obs <= 0 (background): c_k = miss_cost,   c_esc = 0     (GenRe's get_abs_depth writes 0 there)
 * loss [N, H, W]; the backward takes the per-ray upstream gradient grad_loss [N, H, W]. */
int genre_b200_ray_consistency_forward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                       const float *fl, int64_t fN, const float *camdist, int64_t dN,
                                       const float *obs, int64_t oN, int64_t oH, int64_t oW, float miss_cost,
                                       float *loss, void *stream);
int genre_b200_ray_consistency_backward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                        const float *fl, int64_t fN, const float *camdist, int64_t dN,
                                        const float *obs, int64_t oN, int64_t oH, int64_t oW, float miss_cost,
                                        const float *grad_loss, float *grad_vox, void *stream);
/* Posed views: the same ops from V cameras per grid, rays over [N, V, H, W], all V views of grid n
 * reading vox[n] (the backward's atomics sum the views' gradients into grad_vox[n]).  View (n, v) has
 *   fl[n*fN + v*fV]                 focal length in pixels
 *   rot + n*rN + v*rV  (9 floats)   3x3 rotation, row-major, its columns the camera's axes in the grid
 *                                   frame (x forward; image w grows towards -y, image h towards -z)
 *   eye + n*eN + v*eV  (3 floats)   the camera's centre in the grid frame, |eye| > sqrt(3)/2
 * (strides in elements; 0 over n shares one camera set across the batch).  Pixel (h, w) keeps the
 * camera-frame direction u above; the ray's arithmetic is, in fp64 with every operation rounded:
 *   u'_i = (rot[i][0]*ux + rot[i][1]*uy) + rot[i][2]*uz;   d = sqrt((ex*ex + ey*ey) + ez*ez)
 *   t = (d - sqrt(3)/2) + k * (sqrt(3)/(Z-1));   g = (t*u'x + ex, t*u'y + ey, t*u'z + ez)
 * then f = (g + 0.5) * R - 0.5, and f and t rounded once to fp32 as above.  rot = I and
 * eye = (-cam_dist, 0, 0) give the fixed camera's outputs bit for bit.  Outputs and upstream gradients
 * [N, V, H, W] dense; obs [N, V, H, W] with any strides (oN, oV, oH, oW).  1 <= V, N V H W <= 2^34. */
int genre_b200_render_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res,
                                    const float *fl, int64_t fN, int64_t fV, const float *rot, int64_t rN, int64_t rV,
                                    const float *eye, int64_t eN, int64_t eV, float bg, float *depth, float *silhou,
                                    void *stream);
int genre_b200_render_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res,
                                     const float *fl, int64_t fN, int64_t fV, const float *rot, int64_t rN, int64_t rV,
                                     const float *eye, int64_t eN, int64_t eV, float bg, const float *grad_depth,
                                     const float *grad_silhou, float *grad_vox, void *stream);
int genre_b200_ray_consistency_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                             int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                             int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                             const float *obs, int64_t oN, int64_t oV, int64_t oH, int64_t oW,
                                             float miss_cost, float *loss, void *stream);
int genre_b200_ray_consistency_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                              int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                              int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                              const float *obs, int64_t oN, int64_t oV, int64_t oH, int64_t oW,
                                              float miss_cost, const float *grad_loss, float *grad_vox, void *stream);
/* Pose gradients of the posed views: the backwards above plus d(sum of upstream gradient x output)/d rot and d/d eye
 * per view, written (not accumulated) to grad_rot [N, V, 9] (row-major, the ambient gradient of the 9 entries) and
 * grad_eye [N, V, 3], dense, per (n, v) even where rot / eye are shared over n (stride 0).  The derivative is the
 * discrete op's along its own samples, which move with |eye|; the fp32 roundings of f and t count as the identity and
 * the trilinear interpolant is differentiated in the cell make_taps selects.  Not differentiated: fl, obs.
 *   grad_vox   nullable: NULL skips the voxel atomics (pose-only fitting); else accumulated exactly as the
 *              backwards above.
 *   workspace  genre_b200_render_views_pose_workspace_bytes(N, V, H, W) bytes, 8-byte aligned, caller-owned: one
 *              CTA's fp64 partial sums per 8 rays of a view, summed per view in a fixed order, so grad_rot and
 *              grad_eye are bitwise repeatable.  Two kernel launches.
 * Null or misaligned pose outputs: GENRE_B200_EINVAL / GENRE_B200_EALIGN; a short workspace: GENRE_B200_EWORKSPACE. */
size_t genre_b200_render_views_pose_workspace_bytes(int64_t N, int64_t V, int64_t H, int64_t W);
int genre_b200_render_views_backward_pose(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                          int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                          int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, float bg,
                                          const float *grad_depth, const float *grad_silhou, float *grad_vox,
                                          float *grad_rot, float *grad_eye, void *workspace, size_t workspace_bytes,
                                          void *stream);
int genre_b200_ray_consistency_views_backward_pose(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                   int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                   const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                   int64_t eN, int64_t eV, const float *obs, int64_t oN, int64_t oV,
                                                   int64_t oH, int64_t oW, float miss_cost, const float *grad_loss,
                                                   float *grad_vox, float *grad_rot, float *grad_eye, void *workspace,
                                                   size_t workspace_bytes, void *stream);
/* Surface normals of the posed views: the cameras, rays, samples, p_k, T_k and s_k above, arguments laid out as the
 * views entries, plus eps > 0 (finite; else GENRE_B200_EINVAL), in occupancy per unit length.  At sample k,
 *   g_k = R d raw / d f (the interpolant's gradient per unit length in the grid frame, in the cell the taps come from,
 *         zero padding),  rho_k = sqrt(|g_k|^2 + eps^2),  n_k = -g_k / rho_k  (outward);  a NaN raw gives n_k = 0.
 * render_normal:       normal [N, V, 3, H, W] dense = rot^T sum_k s_k n_k (summed in the grid frame, rotated once per
 *                      ray): the expected normal in the camera frame (x forward, +y towards image -w, +z towards
 *                      image -h), not renormalised; an escaping ray contributes 0.  grad_normal [N, V, 3, H, W] dense.
 * normal_consistency:  obs_normal [N, V, 3, H, W] in that camera frame, any strides (oN, oV, oC, oH, oW); a pixel
 *                      whose 3 components are all exactly 0 is background.  Elsewhere m = rot obs / |obs| (fp64,
 *                      rounded once to fp32), and stops cost c_k = 1 - n_k . m, escape miss_cost; on background every
 *                      stop costs miss_cost and escape is free.  loss and grad_loss [N, V, H, W] dense.
 * The backwards accumulate into grad_vox (as above) both the path through p_k (zero where the clamp is active) and the
 * path through n_k (at every sample with s_k != 0), one atomic per valid tap; rot, eye, fl, obs_normal and eps are not
 * differentiated.  Limits as the views entries: 2 <= R <= 1024, 1 <= z_res <= 4096, N V H W <= 2^34.  One kernel
 * launch each; the forwards are bitwise repeatable and each ray's value does not depend on the batch. */
int genre_b200_render_normal_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                           int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                           int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, float eps,
                                           float *normal, void *stream);
int genre_b200_render_normal_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                            int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                            int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, float eps,
                                            const float *grad_normal, float *grad_vox, void *stream);
int genre_b200_normal_consistency_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                                int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                                int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                                const float *obs_normal, int64_t oN, int64_t oV, int64_t oC, int64_t oH,
                                                int64_t oW, float miss_cost, float eps, float *loss, void *stream);
int genre_b200_normal_consistency_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                                 int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                                 int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                                 const float *obs_normal, int64_t oN, int64_t oV, int64_t oC,
                                                 int64_t oH, int64_t oW, float miss_cost, float eps,
                                                 const float *grad_loss, float *grad_vox, void *stream);
/* Depth and normal sketches together: ray_consistency_views and normal_consistency_views fused into one walk per ray,
 * differentiable in the grid and the poses.  The leading arguments are the views entries'; then obs_depth
 * [N, V, H, W] (any strides (odN, odV, odH, odW); <= 0 is background), obs_normal [N, V, 3, H, W] (any strides; all
 * three exactly 0 is background), the weights wd = depth_weight and wn = normal_weight (finite, >= 0, one of them > 0;
 * else GENRE_B200_EINVAL), miss_cost and eps (as normal_consistency_views).  The samples t_k, p_k, T_k, s_k are
 * ray_consistency_views' and n_k is render_normal_views', bit for bit; each stop costs
 *   c_k = fma(wn, c^n_k, wd c^d_k)   and escaping   c_esc = fma(wn, c^n_esc, wd c^d_esc),
 * c^d and c^n the two entries' costs, each with its own background rule, so a ray's loss is wd L_depth + wn L_normal.
 * loss and grad_loss [N, V, H, W] dense.  The backward accumulates into grad_vox the path through p_k and the path
 * through n_k (weighted by wn), one atomic per valid tap.  _backward_pose also writes grad_rot and grad_eye as the
 * *_views_backward_pose entries (same workspace, grad_vox nullable, two kernel launches, bitwise repeatable), with the
 * normal term's position gradient through the interpolant's in-cell second derivatives and the frame term of
 * m = rot obs / |obs|.  Not differentiated: fl, obs_depth, obs_normal, eps, the weights.  Limits as the views entries. */
int genre_b200_sketch_consistency_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                                int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                                int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                                const float *obs_depth, int64_t odN, int64_t odV, int64_t odH,
                                                int64_t odW, const float *obs_normal, int64_t onN, int64_t onV,
                                                int64_t onC, int64_t onH, int64_t onW, float depth_weight,
                                                float normal_weight, float miss_cost, float eps, float *loss,
                                                void *stream);
int genre_b200_sketch_consistency_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                                 int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                                 int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
                                                 const float *obs_depth, int64_t odN, int64_t odV, int64_t odH,
                                                 int64_t odW, const float *obs_normal, int64_t onN, int64_t onV,
                                                 int64_t onC, int64_t onH, int64_t onW, float depth_weight,
                                                 float normal_weight, float miss_cost, float eps,
                                                 const float *grad_loss, float *grad_vox, void *stream);
int genre_b200_sketch_consistency_views_backward_pose(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_depth, int64_t odN, int64_t odV, int64_t odH, int64_t odW, const float *obs_normal, int64_t onN,
    int64_t onV, int64_t onC, int64_t onH, int64_t onW, float depth_weight, float normal_weight, float miss_cost,
    float eps, const float *grad_loss, float *grad_vox, float *grad_rot, float *grad_eye, void *workspace,
    size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Chamfer nearest-neighbour distance.  Replaces nnd_forward_cuda / nnd_backward_cuda
 * (toolbox/nndistance/src/my_lib_cuda.h:1-4, nnd_cuda.cu:6-177; functions/nnd.py:8-63).
 *   xyz1 [B,N,3], xyz2 [B,M,3] dense;  dist1 [B,N], dist2 [B,M] squared distances;
 *   idx1 [B,N], idx2 [B,M] int32 argmin, lowest index on ties.
 *   backward fully writes grad_xyz1 [B,N,3], grad_xyz2 [B,M,3] (zeroing included).
 * Unlike the reference (nnd_cuda.cu:130-131 launches on the legacy default stream) the given
 * stream is honoured.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_nnd_forward(const float *xyz1, const float *xyz2, int64_t B, int64_t N, int64_t M,
                           float *dist1, float *dist2, int32_t *idx1, int32_t *idx2, void *stream);
int genre_b200_nnd_backward(const float *xyz1, const float *xyz2, int64_t B, int64_t N, int64_t M,
                            const float *grad_dist1, const float *grad_dist2,
                            const int32_t *idx1, const int32_t *idx2,
                            float *grad_xyz1, float *grad_xyz2, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Stage-level entry points of the voxelisation pipeline (used by bench.py to time the dominant
 * kernel on its own, and by tests).  genre_b200_cam_bp_forward == stage_project + stage_splat.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_cam_bp_stage_project(const float *depth, int64_t N, int64_t C, int64_t H, int64_t W,
                                    int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                                    const float *fl, int64_t fN, int64_t fC,
                                    const float *camdist, int64_t dN, int64_t dC, int res,
                                    void *workspace, size_t workspace_bytes, void *stream);
int genre_b200_voxelize_stage_splat(int64_t n_maps, int64_t pixels_per_map, int res,
                                    float *tdf, float *cnt, float hit_alpha, float hit_beta, float background,
                                    void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * ConvTranspose3d(kernel K in {4, 8}, stride 2, padding K/2 - 1) forward as a wgmma implicit GEMM (TF32 operands,
 * FP32 accumulation in registers).  Replaces the cuDNN call behind nn.ConvTranspose3d in networks/networks.py:211-222
 * (Unet_3D Deconv3d_skip: the channel concatenation of :221 is walked as two K ranges, never materialised) and
 * :253-256 (deconv3d_2x of VoxelDecoder / VoxelGenerator).
 *   src0 [B*D][cg0][H][W][16 B], src1 [...] or NULL   channel-blocked activations; a channel group is 16 bytes per
 *           position: 4 fp32 read as TF32 (f16 = 0) or 8 fp16 (f16 = 1; same 10-bit mantissa, half the operand bytes:
 *           the kernels are bound by shared-memory operand bandwidth, so this path is ~2x faster)
 *   wpack   weights packed per (parity, z-tap, 8-channel chunk) stage: see genre_shapehd_b200/ops_conv.py
 *   scale, shift [npad]   y = act(acc * scale + shift): bias and folded eval-mode BatchNorm3d
 *   slope   LeakyReLU slope (1 = none);   out [B*2D][cgo][2H][2W][4], or NULL with operand outputs (below)
 * Supported: W in {16,32}, H % 16 == 0, cg0 + cg1 even, 4*cgo <= npad, npad in {32,64}.
 *
 * Operand outputs.  genre_b200_convt3d_s2_forward, genre_b200_convt3d_s2_merged_forward, genre_b200_conv3d_k8s2_s4d_forward
 * and genre_b200_conv3d_k4s2_forward write either `out` or, instead, up to two destinations dst0, dst1 (dst1 may be NULL) of
 * the fp16 operand the NEXT layers read, so that no layout pass runs between them.  Exactly one of out and dst0 is non-NULL
 * (anything else is GENRE_B200_EINVAL); without dst0 the layout and cpad arguments are ignored.  Operand outputs need fp16
 * operands: f16 = 2: parts = 2, hi = fp16(a) | lo' = fp16((a - hi) * 2^11) (the fp32-accurate mode; bit-identical to
 * genre_b200_blocked_split2_f16 of the fp32 output); f16 = 1: parts = 1, fp16(a).  With the output extent Do, Ho, Wo:
 *   layout 1 (plain)   dst [B*Do][parts][cpad/8][Ho][Wo][8 fp16]
 *   layout 2 (parity)  dst [B*Do/2][parts][8 s][cpad/8][Ho/2][Wo/2][8 fp16], s = ((z&1)*2 + (y&1))*2 + (x&1): the parity
 *                      sub-volumes of a following conv3d_k4s2 (= genre_b200_ncdhw_to_blocked mode 2 with group 16)
 * Channels from 4*cgo up to cpad (a multiple of 8, >= 4*cgo) are written as zeros on every call.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_convt3d_s2_forward(const void *src0, int cg0, const void *src1, int cg1,
                                  int64_t B, int64_t D, int64_t H, int64_t W,
                                  const void *wpack, int ksize, int npad, int f16,
                                  const float *scale, const float *shift, float slope,
                                  float *out, int cgo,
                                  void *dst0, int layout0, int cpad0, void *dst1, int layout1, int cpad1,
                                  void *stream);

/* Stride-1 convolution with `taps` (3 or 5) taps per dimension on channel-blocked activations, same wgmma kernel:
 *   out[b,z,y,x,n] = act(scale[n] * sum_{t,c} in[b, z+base-tz, y+base-ty, x+base-tx, c] * W[t][c][n] + shift[n])
 * Replaces the cuDNN call behind nn.Conv3d of Unet_3D.enc1 (networks/networks.py:151,197: Conv3d(2->20, k=8, s=2, p=3))
 * after a space-to-depth of the input (k=8/s=2 over C channels == 5 taps/s=1 over 8C channels).
 *   wpack [taps][C/8][taps*taps][2][npad/8][8][4];  out [B*D][cgo][H][W][4];  W in {16,32,64}, H % 16 == 0, npad = 32
 *   (npad = 64 with 3 taps: Conv3d(1 -> 64, k4, s2, p1) over the 2x space-to-depth input, VoxelDiscriminator main.0;
 *    npad = 96 with 5 taps: Conv3d(20 -> 80, k8, s2, p3) = the input gradient of Unet_3D.dec5) */
int genre_b200_conv3d_taps_forward(const void *src0, int cg0, const void *src1, int cg1,
                                   int64_t B, int64_t D, int64_t H, int64_t W,
                                   const void *wpack, int taps, int base, int npad, int f16,
                                   const float *scale, const float *shift, float slope,
                                   float *out, int cgo, void *stream);

/* Conv3d(kernel 4, stride 2, padding 1) forward on the same wgmma kernel.  Replaces the cuDNN call behind conv3d_half
 * (VoxelDiscriminator, networks/networks.py:247-250) and Unet_3D.enc2..enc5 (:152-155).  The input arrives as its 8 parity
 * sub-volumes in one channel-blocked tensor src [B*D'][8*cgs][H'][W'][16 B] (D' = D/2 ...; group index = s*cgs + c,
 * s = (pz*2+py)*2+px); sub-volume s is a K range with 2 taps per dimension (kernel index 3 - 2t - p).
 *   wpack [2][kblocks*8*cgs/2][4][2][npad/8][8][g];  out [B*D'][cgo][H'][W'][4];  W' in {16,32}, H' % 16 == 0, cgs even,
 *   npad in {32,64,96,128}.  kblocks: 1, or 3 when src holds the lo|hi|hi blocks of genre_b200_blocked_split3. */
int genre_b200_conv3d_k4s2_forward(const void *src, int cgs, int kblocks, int64_t B, int64_t D, int64_t H, int64_t W,
                                   const void *wpack, int npad, int f16,
                                   const float *scale, const float *shift, float slope,
                                   float *out, int cgo,
                                   void *dst0, int layout0, int cpad0, void *dst1, int layout1, int cpad1,
                                   void *stream);

/* The k 4 / s 2 / p 1 convolutions of the SMALL volumes (coarse side <= 8^3: Unet_3D.enc4, enc5, dec2, dec3,
 * networks/networks.py:157-165; the 4^3 / 8^3 stages of VoxelDecoder / VoxelGenerator / VoxelDiscriminator :40-57,:79-97,:247-256)
 * as a wgmma implicit GEMM over the flattened, zero-separated volume (csrc/convflat.cu).  Replaces the cuDNN calls behind
 * those nn.Conv3d / nn.ConvTranspose3d modules in eval mode.
 *   genre_b200_convflat_positions: positions per channel-group array of the operand of a coarse (B, D, H, W) volume
 *       (*lead = index of position 0);
 *   genre_b200_convflat_pack: NCDHW fp32 -> operand [parts][cgs][P][8 fp16] (parts 2 = fp16 hi | lo' = (a - hi) * 2^11), groups
 *       [cg_off, ...); subvol = 1: src is [B, C, 2D, 2H, 2W] and becomes 8 parity sub-volume blocks of C/8 groups (C % 8 == 0);
 *       src NULL: zero `zero_groups` groups (padding to an even group count);
 *   genre_b200_convflat_forward: out[B, Cout, Do, Ho, Wo] (NCDHW fp32) = lrelu(scale * conv + shift); transposed 1:
 *       ConvTranspose3d, output 2x the coarse volume; 0: Conv3d of the 2x volume given as sub-volume blocks (cgs % 16 == 0),
 *       output the coarse volume.  wpack [classes 8|1][ceil(Cout/npad)][cgs/2][8 taps][2][parts*npad/8][8][8] fp16, npad 64 | 80,
 *       op 1 (fp16 operands) | 2 (hi/lo split, fp32-accurate). */
int64_t genre_b200_convflat_positions(int64_t B, int D, int H, int W, int *lead);
int genre_b200_convflat_pack(const float *src, int C, int64_t B, int D, int H, int W, int subvol, void *operand, int cg_off,
                             int cgs, int parts, int zero_groups, void *stream);
int genre_b200_convflat_forward(const void *operand, int cgs, int64_t B, int D, int H, int W, int transposed,
                                const void *wpack, int npad, int op, const float *scale, const float *shift, float slope,
                                float *out, int Cout, void *stream);

/* The two degenerate convolutions at the bottom of the U-Net as weight-streaming FP32 products (csrc/skinny_gemm.cu):
 * Conv3d whose kernel covers its whole input (Unet_3D.enc6, networks/networks.py:157: W is [N = Cout][K = Cin*k^3], w_is_nk = 1)
 * and ConvTranspose3d on a 1^3 input (Unet_3D.dec1 :162, VoxelDecoder / VoxelGenerator main.0 :40,:79: W is [K = Cin][N = Cout*k^3],
 * w_is_nk = 0, chan_div = k^3).  Replaces the cuDNN / cuBLAS calls behind those modules in eval mode.
 *   out[M][N] = lrelu(scale[n / chan_div] * (x[M][K] @ W) + shift[n / chan_div]); fp32 throughout (FP32 FMAs, fixed summation order);
 *   the contiguous extent of W a multiple of 4; workspace = genre_b200_skinny_gemm_workspace_bytes(M, N, K, w_is_nk). */
size_t genre_b200_skinny_gemm_workspace_bytes(int64_t M, int64_t N, int64_t K, int w_is_nk);
int genre_b200_skinny_gemm(const float *x, const float *W, int64_t M, int64_t N, int64_t K, int w_is_nk, int chan_div,
                           const float *scale, const float *shift, float slope, float *out, void *workspace,
                           size_t workspace_bytes, void *stream);

/* ConvTranspose3d(Cin -> 1, kernel 4, stride 2, padding 1) on 64-wide volumes as a wgmma GEMM over the 64 kernel taps
 * (P[position, tap] = sum_c x[c, position] W[c, tap]) followed by a shared-memory col2im (csrc/convt_c1_col2im.cu).  Replaces the
 * cuDNN call behind the last layer of each decoder (Unet_3D.dec6 networks/networks.py:167-168, VoxelDecoder :57, VoxelGenerator :98).
 *   src0 [B*D][parts*cg0][H][64][8 fp16], src1 likewise (cg1 groups) or NULL; parts 1 (op 1: fp16) | 2 (op 2: hi | lo' split,
 *   fp32-accurate); cg0 + cg1 even; H % 8 == 0; W == 64; wpack [(cg0+cg1)/2][2][parts*8][8][8] fp16 with row n = t*8 + r = tap 2t + r
 *   per dimension; bias: one float on the device; out [B][2D][2H][128] fp32, fully overwritten (a strided memset node + one kernel). */
int genre_b200_convt_c1_col2im_forward(const void *src0, int cg0, const void *src1, int cg1, int64_t B, int64_t D, int64_t H,
                                       int64_t W, const void *wpack, int op, const float *bias, float *out, void *stream);

/* ConvTranspose3d(Cin -> 1, kernel 4, stride 2, padding 1) forward on channel-blocked fp32 inputs (FP32 pipe: with one
 * output channel there is no GEMM for the tensor cores).  Replaces the cuDNN call behind the last layer of each decoder:
 * Unet_3D.dec6 (networks/networks.py:167-168, two sources = the skip concatenation), VoxelDecoder main.17 (:57),
 * VoxelGenerator (:98).   weight [Cin][64] = the module's [Cin,1,4,4,4];  out [B][2D][2H][2W] (NCDHW, C = 1). */
int genre_b200_convt_c1_forward(const float *src0, int cg0, const float *src1, int cg1,
                                int64_t B, int64_t D, int64_t H, int64_t W,
                                const float *weight, float bias, int act_sigmoid, float *out, void *stream);

/* ConvTranspose3d(k 8, s 2, p 3), Cout <= 20, with the four (y,x) output parity classes merged along N (one N = 80 MMA
 * instead of four N = 20 MMAs): Unet_3D.dec5 = ConvT(80 -> 20) (networks/networks.py:166), 53.7 of the refiner's 78 GFLOP.
 * Operands as genre_b200_convt3d_s2_forward except scale, shift [20] and wpack, npad = 80 columns n = (py*2+px)*20 + co, in
 * one of two layouts, chosen by `paired`:
 *   paired = 1, valid only with fp16 operands (f16 = 1, 2) and W in {16, 32}: PAIRED classes, 4x4 taps (coarse position j
 *     computes outputs 2j - 1 and 2j per dimension, which read the same inputs): [2 z-parity][4][Cin chunk][16][2][npad/8][8][8]
 *     (ops_conv.pack_convt_paired_weights);
 *   paired = 0: the 5x5 UNION of the classes' taps, zero weights where a class does not use a tap:
 *     [2 z-parity][4][Cin chunk][25][2][npad/8][8][g] (ops_conv.pack_convt_merged_weights).
 * Any other `paired`, or paired = 1 outside its domain, is GENRE_B200_EINVAL.  The two forms give bit-identical results; the
 * paired one issues 28 % fewer MMAs at 32^2. */
int genre_b200_convt3d_s2_merged_forward(const void *src0, int cg0, const void *src1, int cg1,
                                         int64_t B, int64_t D, int64_t H, int64_t W,
                                         const void *wpack, int ksize, int npad, int f16, int paired,
                                         const float *scale, const float *shift, float slope,
                                         float *out, int cgo,
                                         void *dst0, int layout0, int cpad0, void *dst1, int layout1, int cpad1,
                                         void *stream);

/* Conv3d(k 8, s 2, p 3), Cout <= 20, as a 3-tap stride-1 convolution over the 4x space-to-depth input whose N = 160
 * columns are the 8 output classes of the 2x finer output grid: Unet_3D.enc1 = Conv3d(2 -> 20) on 128^3
 * (networks/networks.py:151).  src [B*D][cg][H][W][16 B] with D,H,W = input extent / 4 (genre_b200_ncdhw_to_blocked
 * mode 3); wpack [3][chunk][9][2][20][8][g]; scale, shift [20]; out [B*2D][cgo][2H][2W][4] fp32.  W,H % 16 == 0. */
int genre_b200_conv3d_k8s2_s4d_forward(const void *src, int cg, int64_t B, int64_t D, int64_t H, int64_t W,
                                       const void *wpack, int npad, int f16,
                                       const float *scale, const float *shift, float slope,
                                       float *out, int cgo,
                                       void *dst0, int layout0, int cpad0, void *dst1, int layout1, int cpad1,
                                       void *stream);

/* ConvTranspose3d(Cin -> 1, k 4, s 2, p 1) on the tensor cores: 3 union taps per dimension, the 8 output classes as
 * N columns, bias [1] (device) and optional sigmoid in the epilogue, NCDHW fp32 output [B][2D][2H][2W].  Same layers
 * as genre_b200_convt_c1_forward (the FP32-pipe variant); wpack [3][chunk][9][2][2][8][g].  W in {16,32,64}. */
int genre_b200_convt_c1_tc_forward(const void *src0, int cg0, const void *src1, int cg1,
                                   int64_t B, int64_t D, int64_t H, int64_t W,
                                   const void *wpack, int f16, const float *bias, int act_sigmoid,
                                   float *out, void *stream);

/* Backward of ConvTranspose3d(Cin -> 1, k 4, s 2, p 1) (Unet_3D.dec6 networks/networks.py:167-168 and the decoders' last
 * layers): cuDNN answers the weight gradient of this 1-channel layer with a grouped direct kernel that takes 40.7 ms of
 * a 60 ms Unet_3D training step at B=4 (profiles/r01_train_unet_launches.csv).
 *   wgrad: x [B][Cin][D][H][W], gy [B][1][2D][2H][2W] -> dW [Cin][1][4][4][4]; deterministic (fixed-order reduction of
 *          per-CTA partials in `workspace`, genre_b200_convt_c1_wgrad_workspace_bytes(Cin) bytes); Cin <= 64, H % 8 == 0.
 *   dgrad: gy, weight -> dx [B][Cin][D][H][W]; Cin <= 192, H % 8 == 0. */
size_t genre_b200_convt_c1_wgrad_workspace_bytes(int cin);
int genre_b200_convt_c1_wgrad(const float *x, const float *gy, int64_t B, int64_t Cin, int64_t D, int64_t H, int64_t W,
                              float *dW, void *workspace, size_t workspace_bytes, void *stream);
int genre_b200_convt_c1_dgrad(const float *gy, const float *weight, int64_t B, int64_t Cin, int64_t D, int64_t H, int64_t W,
                              float *dx, void *stream);

/* Weight gradient of Conv3d(Cin <= 2 -> Cout <= 20, k 8, s 2, p 3) = Unet_3D.enc1 (networks/networks.py:151): the
 * cuDNN kernel for it (wgrad2d_grouped_direct_kernel) is 40.7 ms of a 60 ms Unet_3D training step at B=4.
 * x [B][Cin][D][H][W], gy [B][Cout][D/2][H/2][W/2] -> dW [Cout][Cin][8][8][8]; deterministic; H % 16 == 0, W <= 128. */
size_t genre_b200_conv_k8s2_wgrad_workspace_bytes(void);
int genre_b200_conv_k8s2_wgrad(const float *x, const float *gy, int64_t B, int64_t Cin, int64_t Cout,
                               int64_t D, int64_t H, int64_t W, float *dW,
                               void *workspace, size_t workspace_bytes, void *stream);

/* BatchNorm3d with BATCH statistics (training) fused with its ReLU / LeakyReLU, forward and backward, NCDHW fp32:
 * nn.BatchNorm3d + nn.LeakyReLU of Conv3d_block / Deconv3d_skip (networks/networks.py:193-222) and the BatchNorm3d + ReLU of
 * the decoders' stacks (:40-57) while training (cuDNN: 5.3 ms of a 22 ms Unet_3D step for ~0.3 ms worth of HBM traffic).
 * x, y, dy, dx [B][C][S] contiguous and 16-byte aligned, S = D*H*W a multiple of 4; gamma / beta / running_* [C] or NULL;
 * slope: 1 = no activation, 0 = ReLU; two-pass variance, fixed-order reductions (bitwise reproducible).
 * OPT-IN (GENRE_B200_BN_TRAIN=1): written after round 1's GPU budget was spent, not yet run on a GPU. */
size_t genre_b200_bn_workspace_bytes(int64_t C);
int genre_b200_bn_act_train_forward(const float *x, int64_t B, int64_t C, int64_t S,
                                    const float *gamma, const float *beta, float *running_mean, float *running_var,
                                    float eps, float momentum, float slope,
                                    float *y, float *save_mean, float *save_invstd,
                                    void *workspace, size_t workspace_bytes, void *stream);
int genre_b200_bn_act_train_backward(const float *x, const float *dy, int64_t B, int64_t C, int64_t S,
                                     const float *gamma, const float *beta, const float *save_mean, const float *save_invstd,
                                     float slope, float *dx, float *dgamma, float *dbeta,
                                     void *workspace, size_t workspace_bytes, void *stream);

/* Layout boundary of the convolution kernels: contiguous NCDHW fp32 (what networks/networks.py's modules exchange,
 * e.g. Unet_3D.forward networks.py:170-190) <-> channel-blocked [B*D][C/g][H][W][g] (16 bytes per unit).
 *   mode 0: plain;  mode 1: space-to-depth, channel = ((c*2+pz)*2+py)*2+px (Conv3d k8 s2, Unet_3D.enc1; with cpad > 8C the
 *           channel axis is zero-padded to cpad channels: Conv3d(1 -> 64, k4 s2), VoxelDiscriminator's first layer);
 *   mode 2: the 8 parity sub-volumes one after the other, each padded to cpad channels (Conv3d k4 s2);
 *   mode 3: 4x space-to-depth, channel = ((c*4+rz)*4+ry)*4+rx (Conv3d k8 s2 as a 3-tap convolution, Unet_3D.enc1).
 *   group 4: fp32 units, group 8: fp16 units (cast on the way).  One pass, 16-byte stores. */
int genre_b200_ncdhw_to_blocked(const float *src, int64_t B, int64_t C, int64_t D, int64_t H, int64_t W,
                                int mode, int group, int cpad, void *dst, void *stream);

/* blocked fp32 [B*D][cg][H][W][4] -> contiguous NCDHW [B,C,D,H,W], 4*(cg-1) < C <= 4*cg (channel padding dropped) */
int genre_b200_blocked_to_ncdhw(const float *src, int cg, int64_t B, int64_t C, int64_t D, int64_t H, int64_t W,
                                float *dst, void *stream);

/* ---- fused GenRe glue (SURVEY 8f-1; opt-in, inference only; genre_shapehd_b200/fused.py) --------------------------
 * The frozen callers wrap the ops in ~19 dense elementwise passes over 128^3 volumes (depth_pred_with_sph_inpaint.py:
 * 120-126, genre_full_model.py:120-143).  These three entry points fold them into the kernels. */

/* render_spherical over clamp(vox * pre_scale, pre_lo, pre_hi) applied as each voxel is fetched
 * (`render_spherical(torch.clamp(proj * 50, 1e-5, 1 - 1e-5))`, depth_pred_with_sph_inpaint.py:124). */
int genre_b200_render_spherical_forward_pre(const float *vox, int64_t N, int res, const double *dirs,
                                            int sph_res, int z_res, const float *depth_weight,
                                            float pre_scale, float pre_lo, float pre_hi, float *out, void *stream);

/* The spherical renderer with EMPTY-SPACE SKIPPING (forward): same contract and results (within ~1e-6) as
 * genre_b200_render_spherical_forward / _forward_pre (use_pre != 0 renders clamp(vox * pre_scale, pre_lo, pre_hi)).
 * A pre-pass marks the 8^3 bricks that hold a voxel > 1e-5 (dilated by one voxel); along each ray, 32-sample chunks that
 * only touch unmarked bricks (every sample clamps to p = 1e-5, spherical_proj.py:66) are advanced in closed form instead
 * of 32 x 8 gathers.  GenRe's input is a thin shell: ~80 % of the chunks.  workspace: caller-owned,
 * genre_b200_render_spherical_workspace_bytes(N, res) bytes (zeroed by the call).  Falls back to the plain kernels when
 * res % 4 != 0 or z_res > 1024. */
size_t genre_b200_render_spherical_workspace_bytes(int64_t N, int res);
int genre_b200_render_spherical_forward_skip(const float *vox, int64_t N, int res, const double *dirs, int sph_res,
                                             int z_res, const float *depth_weight, int use_pre, float pre_scale,
                                             float pre_lo, float pre_hi, float *out, void *workspace,
                                             size_t workspace_bytes, void *stream);

/* Net.backproject_spherical (genre_full_model.py:134-143) in one call: radius = in_bias + in_scale * sph (the
 * `1 - crop_sph`; the crop is expressed through the strides), out = 1 - R * mean distance on hit voxels and 0
 * elsewhere (= (-tdf + 1/R) * R * clamp(cnt,0,1)), maps written out_map_stride floats apart (a channel of the
 * refiner's [B,2,R,R,R] input).  Workspace as genre_b200_sph_bp_forward. */
int genre_b200_sph_bp_forward_fused(const float *sph, int64_t N, int64_t C, int64_t H, int64_t W,
                                    int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                                    const float *grid, int64_t gN, int64_t gC, int64_t gH, int64_t gW, int64_t gD,
                                    float in_scale, float in_bias, float *out, int64_t out_map_stride, int res,
                                    void *workspace, size_t workspace_bytes, void *stream);

/* dst[m][:] = clamp(src[m][:] * scale, lo, hi), dst maps dst_map_stride floats apart
 * (`torch.clamp(proj_depth / 50, 1e-5, 1 - 1e-5)` + torch.cat, genre_full_model.py:126-127). */
int genre_b200_scale_clamp_strided(const float *src, int64_t maps, int64_t n, float scale, float lo, float hi,
                                   float *dst, int64_t dst_map_stride, void *stream);

/* blocked fp32 [BD][cg4][H][W][4] -> blocked fp16 [BD][(cg4+1)/2][H][W][8], channel padding zero-filled: turns the
 * fp32 output of one tensor-core layer into the fp16 operand of the next without going through NCDHW */
int genre_b200_blocked_f32_to_f16(const float *src, int cg4, int64_t BD, int64_t H, int64_t W, void *dst, void *stream);

/* blocked fp32 [BD][cg4][H][W][4] -> fp16 [BD][2 parts][(cg4+1)/2][H][W][8]: part 0 = hi = fp16(a), part 1 = lo' =
 * fp16((a - hi) * 2^11).  The activation operand of the conv kernels' op = 2 ("f16x2") mode: the fp32-accurate replacement of
 * the reference's fp32 cuDNN convolutions (networks/networks.py:197-218) at 2 tensor-core MMAs per K step
 * (A_hi x [W_hi | W_lo'] and A_lo' x W_hi; weights packed [W_hi | W_lo'] along N by ops_conv._pack).  In that mode every
 * conv entry point above takes per-part channel-group counts and `f16` = 2. */
int genre_b200_blocked_split2_f16(const float *src, int cg4, int64_t BD, int64_t H, int64_t W, void *dst, void *stream);

/* blocked fp32 [BD][cg][H][W][4] -> [BD][3*cg][H][W][4] = (lo | hi | hi): hi = value rounded to TF32, lo = value - hi.
 * With weights packed as (W_hi | W_lo | W_hi) along K, the TF32 tensor-core kernels above compute
 * A_lo*W_hi + A_hi*W_lo + A_hi*W_hi = the fp32 product to ~2^-21 relative (small terms first: the tensor core's
 * fp32 accumulator truncates, ~2^-26 of the partial sum per MMA step) ("3xTF32"): the mode the 3D nets run in when
 * torch.backends.cudnn.allow_tf32 is off, so that occupancies match the fp32 reference within 1e-4. */
int genre_b200_blocked_split3(const float *src, int cg, int64_t BD, int64_t H, int64_t W, float *dst, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Ground-truth surface voxels (SURVEY 8f-3).  Replaces the per-sample CPU code of Model.preprocess
 * (models/genre_full_model.py:86-96, scipy.ndimage.binary_erosion inside DataLoader workers):
 *     val  = flip(transpose(voxel, (0,2,1)), 2)                      (transpose_flip != 0; :89-90)
 *     out  = clip(val - binary_erosion(val != 0, ones((3,3,3)), iterations), 0, 1)   (:91-93, border value 0)
 *   vox, out [N, R, R, R] dense fp32, distinct buffers; R a multiple of 32, at most 256; 1 <= iterations <= 15
 *   workspace: genre_b200_voxel_surface_workspace_bytes(N, R) bytes (one bit per voxel), caller-owned
 * Bit-exact against scipy (tests/test_gpu_toolbox.py).
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_voxel_surface_workspace_bytes(int64_t N, int res);
int genre_b200_voxel_surface(const float *vox, int64_t N, int res, int iterations, int transpose_flip, float *out,
                             void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Batched marching cubes (SURVEY 8f-3).  Replaces skimage.measure.marching_cubes_lewiner(df, th, spacing=...) in
 * Visualizer._save_iso_obj (visualize/visualizer.py:160) and util_sph.py:47, for a batch resident on the device.
 *   vol     [N, D, H, W] dense fp32; 2 <= D, H, W <= 512, 1 <= N <= 65535.  A point is inside iff v > level (NaN: outside).
 *   vertices: one per grid edge with ends on different sides; point p owns its edges to p+e0, p+e1, p+e2.  For the edge from p
 *             (value v0) to q (value v1) along axis a: t = fl(fl(level - v0) / fl(v1 - v0)),
 *             x_a = fl(fl(fl(p_a + t) * spacing_a) - shift_a), x_b = fl(fl(p_b * spacing_b) - shift_b) for the other axes
 *             (one rounding per step, no FMA).  Axis 0 is the first array axis (skimage's convention).
 *             Non-finite voxels follow the same formula: a crossing edge with a finite low end p and an infinite high end
 *             has t = +-0, so its vertex is p; with a NaN end, or an infinite low end, t and x_a are NaN.
 *             Order: sample, point index (i*H + j)*W + k, axis.
 *   faces:    per-cell segment linking with the asymptotic decider on ambiguous faces (inside corners a, d on a diagonal
 *             are joined iff fl(a'*d') > fl(b'*c'), x' = fl(x - level)); loops fanned as (v0, v_i, v_{i+1}).  Interior
 *             ambiguities (Lewiner's tunnel cases) are not resolved; the triangles are not skimage's.  Counter-clockwise
 *             seen from the <= level side.  Order: sample, cell index, loop (by smallest local edge id 4a + 2*ob + oc),
 *             fan position.  int32 indices into the sample's own vertex block.
 *             The full rules are in csrc/isosurface.cu; oracle_iso/isosurface_oracle.c restates them bit for bit.
 * Output sizes depend on the data, so there are two calls and the caller allocates between them:
 *   count: counts [N, 2] int64 (vertices, faces) on the device; per-tile offsets stay in the workspace.
 *   emit:  vert_off, face_off [N+1] int64 on the device, the exclusive prefix sums of counts[:, 0] and counts[:, 1];
 *          verts [sum V, 3] fp32, faces [sum F, 3] int32.  Same vol, level and workspace as the count call, untouched in between.
 *   workspace: genre_b200_isosurface_workspace_bytes(N, D, H, W) bytes (0: unsupported shape), 16-byte aligned, caller-owned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_isosurface_workspace_bytes(int64_t N, int D, int H, int W);
int genre_b200_isosurface_count(const float *vol, int64_t N, int D, int H, int W, float level, int64_t *counts,
                                void *workspace, size_t workspace_bytes, void *stream);
int genre_b200_isosurface_emit(const float *vol, int64_t N, int D, int H, int W, float level, float sx, float sy, float sz,
                               float shx, float shy, float shz, const int64_t *vert_off, const int64_t *face_off, float *verts,
                               int32_t *faces, void *workspace, size_t workspace_bytes, void *stream);
/* backward: grad_vol [N, D, H, W] fp32 (fully written, no memset needed) = the gradient of the emitted vertex coordinates with
 * respect to vol, given grad_verts [sum V, 3] fp32.  Same vol, N, D, H, W, level and workspace as the count and emit calls,
 * the workspace untouched since emit; the spacing and vert_off of the emit call.  Only x_a of the vertex on the edge from p
 * (value v0) to q = p + e_a (value v1) depends on vol; with g = grad_verts[v][a] (the other two components are ignored),
 * in fp64 from the fp32 operands, one rounding per operation, in this order:
 *     d = v1 - v0,  k = (g * s_a) / (d * d),  c0 = k * (level - v1) to p,  c1 = k * (v0 - level) to q.
 * An edge with a non-finite end contributes 0.  Grid point p sums in fp64, from 0, its own crossing edges a = 0, 1, 2 (c0),
 * then the edges arriving from p - e_a, a = 0, 1, 2 (c1), and rounds once to fp32; a point on no crossing edge gets 0.
 * A gather without atomics: deterministic, bit-equal to the numpy restatement in tests/surface_grad_ref.py. */
int genre_b200_isosurface_backward(const float *vol, int64_t N, int D, int H, int W, float level, float sx, float sy, float sz,
                                   const int64_t *vert_off, const float *grad_verts, float *grad_vol, void *workspace,
                                   size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * First-hit ray casting of batched triangle meshes (SURVEY 8f-4).  Replaces trimesh's
 * mesh.ray.intersects_id(origins, dirs, multiple_hits=False) in util_sph.render_model (util/util_sph.py:7-18), one mesh per
 * sample, for a batch resident on the device.
 *   meshes  the packed output of genre_b200_isosurface_*: verts [V, 3] fp32 (finite), faces [F, 3] int32 indexing the sample's
 *           own vertex block, vert_off / face_off [N+1] int64 on the device (exclusive prefix sums; V, F the totals).
 *   rays    origins, dirs [N|1, R, 3] fp32; ray_batch_stride = 3*R (per-sample rays) or 0 (one table shared by the batch).
 *           A ray with a non-finite component or a zero direction misses.
 *   hit     a face is DEGENERATE iff fl(fl(v1 - v0) x fl(v2 - v0)) is the zero vector; degenerate faces never hit.  Otherwise
 *           the two-sided watertight test of Woop, Benthin and Wald (2013) in fp32, one rounding per step, as spelled out in
 *           csrc/raycast.cu: kz = argmax |d| (lowest axis on ties), shear by d_kx/d_kz, d_ky/d_kz, 1/d_kz, edge functions
 *           U, V, W, det = (U+V)+W, T = (U*Az + V*Bz) + W*Cz, t = T/det; a hit iff the edge functions do not have mixed
 *           signs, det != 0 and 0 < t < inf.
 *   result  t [N, R] fp32 and face [N, R] int32 (local to the sample): the hit with the smallest t, ties to the smallest face
 *           index; +inf and -1 on a miss.  Equal, bit for bit, to a loop over all of the sample's faces for every G
 *           (the argument is in csrc/raycast.cu); oracle_ray/raycast_oracle.c is that loop.
 * Three calls; the caller owns every buffer, the library never synchronises:
 *   count:     refs [N] int64 on the device, the number of (cell, face) references of each sample's uniform G^3 grid.
 *   build:     ref_off [N+1] int64 on the device, the exclusive prefix sums of refs; ref_ids [sum refs] int32.
 *   first_hit: writes t and face.  Same meshes, G and workspace in all three calls, untouched in between.
 *   G in [1, 256], N in [1, 65535]; workspace: genre_b200_raycast_workspace_bytes(N, G) bytes (0: unsupported), 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_raycast_workspace_bytes(int64_t N, int G);
int genre_b200_raycast_count(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                             const int64_t *face_off, int64_t N, int G, int64_t *refs, void *workspace,
                             size_t workspace_bytes, void *stream);
int genre_b200_raycast_build(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                             const int64_t *face_off, int64_t N, int G, const int64_t *ref_off, int32_t *ref_ids,
                             void *workspace, size_t workspace_bytes, void *stream);
int genre_b200_raycast_first_hit(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                                 const int64_t *face_off, int64_t N, int G, const int64_t *ref_off, const int32_t *ref_ids,
                                 const float *origins, const float *dirs, int64_t R, int64_t ray_batch_stride, float *t,
                                 int32_t *face, void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Voxel-grid utilities.  Replace the per-sample CPU toolkit util/util_voxel.py for a batch resident on the device.
 * Common rules: vol [N, D, H, W] dense fp32, every dimension in [2, 512], 1 <= N <= 65535; the caller owns every buffer and
 * workspace; the library allocates nothing and never synchronises; argument errors are reported before any launch.
 *
 * fill (replaces _fill / fill, util_voxel.py:167-238): a voxel is occupied iff v > threshold (NaN: empty; the reference
 *   casts its input to uint8, so threshold = 0.5 is its semantics on {0, 1} grids).  out [N, D, H, W] uint8 is 1 for occupied
 *   voxels and for empty voxels not connected, through empty voxels, to the outside (a virtual empty shell around the grid);
 *   connectivity 6 (faces) or 26 (faces, edges, corners: the reference's six_way=False).  Union-find labelling of the empty
 *   voxels (csrc/voxel_tools.cu): a fixed number of passes whatever the shape.  The result is a set membership, so it does not
 *   depend on the order the unions happen in: it is deterministic.
 *   workspace: genre_b200_voxel_fill_workspace_bytes(N, D, H, W) bytes (0: unsupported shape), 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_voxel_fill_workspace_bytes(int64_t N, int D, int H, int W);
int genre_b200_voxel_fill(const float *vol, int64_t N, int D, int H, int W, float threshold, int connectivity, uint8_t *out,
                          void *workspace, size_t workspace_bytes, void *stream);

/* transform (replaces transform_by_matrix / transform, util_voxel.py:133-161): resampling by an affine map from output grid
 * indices to input coordinates.  params [N, 12] fp64 on the device: a row-major 3x3 matrix M and a translation t per sample.
 * For output point (i0, i1, i2), with n = (D, H, W): u_b = i_b - n_b/2, and for every axis a, in this order and one rounding
 * per step (no contraction):
 *     x_a = (((M[a][0]*u_0 + M[a][1]*u_1) + M[a][2]*u_2) + n_a/2) + t_a
 * (the reference forms inv(matrix) . (i - n/2) + n/2 - offset; M = inv(R(angles) S(scales)) and t = -offset give it).
 * The value is scipy's RegularGridInterpolator(method='linear', bounds_error=False, fill_value=0): 0 when x_a lies outside
 * [0, n_a - 1] on any axis (or is NaN); else, with c_a = min(floor(x_a), n_a - 2), y_a = x_a - c_a, the 8 corners in C order
 * (last axis fastest) each add vol[corner] * ((w_0 * w_1) * w_2) to a sum that starts at 0, w_a = 1 - y_a or y_a, all in fp64.
 * Epilogues (flags): GENRE_B200_VOXEL_CLAMP clips the fp64 value to [clamp_lo, clamp_hi] (np.clip); then either
 * GENRE_B200_VOXEL_THRESHOLD writes out [N, D, H, W] uint8 = value > threshold (compared in fp64), or out [N, D, H, W] fp32
 * gets the value rounded once to fp32.
 * ------------------------------------------------------------------------------------------- */
#define GENRE_B200_VOXEL_CLAMP 1u
#define GENRE_B200_VOXEL_THRESHOLD 2u
int genre_b200_voxel_transform(const float *vol, int64_t N, int D, int H, int W, const double *params, unsigned flags,
                               double clamp_lo, double clamp_hi, double threshold, void *out, void *stream);

/* stats: one pass over a (and b).  bounds [N, 6] int32 (or NULL): find_bound (util_voxel.py:31-52) of a > th_a, as
 * (min_0, min_1, min_2, max_0, max_1, max_2), lower bound inclusive, upper bound exclusive, all zeros for an empty sample.
 * counts [N, 3] int64 (or NULL; needs b): |A|, |B|, |A and B| with A = pool(a) > th_a, B = pool(b) > th_b, pool = downsample
 * (util_voxel.py:10-28) by `pool` on every axis (the remainder ignored), GENRE_B200_POOL_MAX (exact) or GENRE_B200_POOL_MEAN
 * (fp64 sum in C order, divided by pool^3 in fp64).  Comparisons: the fp32 voxels (the bounds, and the counts at pool = 1)
 * with the threshold rounded to fp32, as numpy and torch compare an fp32 grid with a Python float; pooled values (pool > 1)
 * in fp64 with the fp64 threshold, as the reference thresholds the fp64 output of its downsample.  The bounds are always
 * those of the full-resolution a.  1 <= pool <= min(D, H, W).  No workspace; at least one of bounds, counts.
 * ------------------------------------------------------------------------------------------- */
#define GENRE_B200_POOL_MAX 0
#define GENRE_B200_POOL_MEAN 1
int genre_b200_voxel_stats(const float *a, const float *b, int64_t N, int D, int H, int W, int pool, int pool_mode,
                           double th_a, double th_b, int32_t *bounds, int64_t *counts, void *stream);

/* downsample (replaces downsample, util_voxel.py:10-28): vol [N, R, R, R] -> out [N, d, d, d] fp32, d = R / times (the
 * remainder ignored, as the reference does), 1 <= times <= R.  use_max != 0: the block's maximum (exact; NaN propagates, as
 * np.max); else the mean: fp64 sum in C order divided by times^3 in fp64, rounded once to fp32.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_voxel_downsample(const float *vol, int64_t N, int R, int times, int use_max, float *out, void *stream);

/* translate (replaces the copy of translate, util_voxel.py:87-90): bounds [N, 6] int32 as stats writes them, offsets [N, 3]
 * int32, both on the device.  out[p] = vol[p - off] when p - off lies inside the box [min, max) (and the grid), else 0: the
 * box's contents move by off and everything outside the box is dropped, as in the reference.  Choosing the offset and
 * checking that the moved box stays inside the grid (the reference's assert) is the caller's.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_voxel_translate(const float *vol, int64_t N, int D, int H, int W, const int32_t *bounds, const int32_t *offsets,
                               float *out, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Area-weighted uniform surface sampling of batched triangle meshes: n points per sample, the step from a marching-cubes mesh
 * to a Chamfer / F-score evaluation (the reference's nndistance op) without leaving the device.
 *   meshes  the packed output of genre_b200_isosurface_*: verts [V, 3] fp32, faces [F, 3] int32 indexing the sample's own
 *           vertex block, vert_off / face_off [N+1] int64 on the device.  F (the total) < 2^31, 1 <= N <= 65535.
 *   weight  per face, fp64 from the fp32 vertices a, b, c, one rounding per operation, no contraction: e1 = b - a, e2 = c - a,
 *           n = (e1y*e2z - e1z*e2y, e1z*e2x - e1x*e2z, e1x*e2y - e1y*e2x), s = sqrt((nx*nx + ny*ny) + nz*nz), a non-finite s
 *           counting as 0.  smax_b = the sample's largest s; w = floor(ldexp(s / smax_b, 32)) as uint64 (all 0 when
 *           smax_b = 0).  P = the inclusive prefix sums of w per sample (exact in uint64), T_b = the last one (0 without faces).
 *   point i of sample b: r_j = splitmix64(seed_b + (3i + j + 1) * 0x9E3779B97F4A7C15), j = 0, 1, 2, in wrapping uint64
 *           arithmetic (splitmix64's output function, spelled out in csrc/surface_sample.cu); the face is the smallest f with
 *           P_f > mulhi64(r_0, T_b); U = r_1 >> 40, V = r_2 >> 40, replaced by 2^24 - U, 2^24 - V when U + V > 2^24;
 *           u = U * 2^-24, v = V * 2^-24; per axis p = fl(fl(a + fl(u * fl(b - a))) + fl(v * fl(c - a))), no FMA.
 *   seeds   [N] uint64 on the device.  n in [1, 2^30].
 *   output  points [N, n, 3] fp32, face [N, n] int32 local to the sample; a sample with T_b = 0 gets NaN points and face -1.
 *           A point depends only on (seed_b, i) and its own mesh: deterministic and batch-equivariant.
 *           tests/surface_sample_ref.py restates the whole contract in numpy, bit for bit.
 *   workspace: genre_b200_surface_sample_workspace_bytes(N, F) bytes (0: unsupported), 16-byte aligned, caller-owned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_surface_sample_workspace_bytes(int64_t N, int64_t F);
int genre_b200_surface_sample(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                              const int64_t *face_off, int64_t N, const uint64_t *seeds, int64_t n, float *points,
                              int32_t *face, void *workspace, size_t workspace_bytes, void *stream);
/* backward: grad_verts [V, 3] fp32 (fully written: the call clears it first) = the gradient of the points with respect to the
 * vertices, the drawn faces and barycentric draws held fixed (no gradient through the area weights).  faces, vert_off,
 * face_off, seeds, N and n as in the forward call; face [N, n] the forward's output (trusted); grad_points [N, n, 3] fp32.
 * Point i of sample b redraws (u, v) from (seed_b, i) as above and adds fl32(w * g) for w = 1 - u - v, u, v (exact in fp32)
 * to its face's three vertices by fp32 atomicAdd: the order is unspecified, so the result is not bitwise reproducible.
 * Points with face -1 contribute nothing.  No workspace. */
int genre_b200_surface_sample_backward(const int32_t *faces, int64_t F, const int64_t *vert_off, const int64_t *face_off,
                                       int64_t N, const uint64_t *seeds, int64_t n, const int32_t *face,
                                       const float *grad_points, int64_t V, float *grad_verts, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Earth mover's distance between B pairs of equal-size point sets: an auction (Bertsekas) with eps-scaling and Jacobi
 * bidding, one CTA per pair, everything but p in shared memory.  The assignment is a bijection whose mean cost is within the
 * final eps_eff of the optimum (eps-complementary slackness): opt <= emd <= opt + eps_eff, up to the fp64 rounding of the sum.
 *   inputs  p, q [B, n, 3] fp32, dense; 1 <= n <= 4096, 1 <= B <= 65535, eps finite and > 0.  Persons are p's points,
 *           objects q's.
 *   cost    c_ij = sqrt((dx*dx + dy*dy) + dz*dz) in fp32, d = p_i - q_j, one rounding per operation, no FMA, sqrt correctly
 *           rounded.  Everything after it is fp64, one rounding per operation, no FMA.
 *   refusal a pair with a coordinate that is NaN or of magnitude above 2^62 (where an fp32 squared distance could overflow)
 *           never enters the auction: match -1 for all its points, emd NaN, rounds = phases = 0.
 *   eps     lo_a / hi_a = the smallest / largest fp32 coordinate a over both sets, e_a = (double)hi_a - (double)lo_a,
 *           D = sqrt((e0*e0 + e1*e1) + e2*e2); eps_eff = max(eps, D * 2^-32) (below that a bid could fail to raise an
 *           fp64 price, and the auction would never end).  Phase k = 0, 1, ... runs at eps_0 = max(D * 0.25, eps_eff),
 *           eps_{k+1} = max(eps_k * 0.25, eps_eff); the phase run at eps_eff is the last.  Prices start at 0 and carry
 *           over; every phase starts with no person assigned.
 *   round   (Jacobi) every unassigned person i bids at once, against the prices at the round's start:
 *             v_ij = (-(double)c_ij) - price_j;  v1 = max_j v_ij, j1 = the lowest j attaining it;  v2 = max over j != j1
 *             (n = 1: v2 = v1);  bid_i = (price_j1 + (v1 - v2)) + eps_k.
 *           Every object with bids goes to its highest bid, the lowest i among equal bids; its price becomes that bid and its
 *           previous owner, if any, is unassigned.  The phase ends after the first round that leaves nobody unassigned.
 *   cap     2^22 rounds per pair over all phases: a pair whose 2^22-th round still leaves a person unassigned gets the
 *           refusal's output (with its counts).  Far above what point sets of <= 4096 points need; it is a safety net.
 *   output  match [B, n] int32, match[b, i] = the object of person i: a permutation of 0..n-1.  emd [B] fp64 = S / n with
 *           S the fp64 sum of the matched costs (double)c_{i, match[i]}, zero-padded to N2 = the smallest power of two
 *           >= n and summed by halving: a_i += a_{i + h} for h = N2/2, N2/4, ..., 1 (S = c_0 when n = 1).
 *           The result depends only on the pair: deterministic, independent of scheduling and of the rest of the batch.
 *           tests/emd_ref.py restates the whole contract in numpy, bit for bit.
 *   workspace: genre_b200_emd_workspace_bytes(B, n) bytes (0: unsupported), 16-byte aligned, caller-owned.  Its first 8 B bytes
 *           receive int32 [B, 2]: the rounds and the phases each pair ran (a debug counter).
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_emd_workspace_bytes(int64_t B, int64_t n);
int genre_b200_emd_forward(const float *p, const float *q, int64_t B, int64_t n, double eps, int32_t *match, double *emd,
                           void *workspace, size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Exact Euclidean distance transform of N cubic grids (separable lower envelopes, Felzenszwalb & Huttenlocher 2012):
 *   vox     [N, R, R, R] fp32, dense; 1 <= R <= 256, 1 <= N <= 65535, level not NaN.
 *   out_sq  [N, R, R, R] fp32, dense, must not alias vox: for every voxel, the squared Euclidean distance in voxel units
 *           to the nearest voxel of the same grid with value >= level (a NaN voxel never is one; level may be +-inf).
 *           Every value is an integer, at most 3 (R-1)^2
 *           < 2^24, so it is exact; a grid with no such voxel is +inf everywhere.  Parabola intersections are compared by
 *           int64 cross-multiplication: the result is exact and independent of scheduling and of the rest of the batch.
 *   Three kernels (one per axis), all in place on out_sq; no workspace.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_distance_transform(const float *vox, int64_t N, int res, float level, float *out_sq, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Scores of K candidate cameras per grid against observed camera-frame points (no backward: a search, not a loss).
 *   field   [N, R, R, R] fp32, dense: a distance to the grid's surface in grid units, finite (the caller clamps it to tau);
 *           1 <= R <= 256, 1 <= N <= 65535.
 *   points  [N, P, 3] fp32, dense: points in the camera frame (x forward, +y towards image -w, +z towards image -h);
 *           1 <= P <= 4096.  counts [N] int32: rows 0 .. counts[n]-1 of sample n are its points.  A count outside
 *           [1, P] is not dereferenced: that sample's scores are NaN (callers check the counts on the host first).
 *   rot     element (n, k) at rot + n rN + k rK, a dense row-major 3x3 whose columns are the camera's axes in the grid
 *           frame; eye at eye + n eN + k eK, 3 floats: the camera's centre.  rN = eN = 0 shares the candidates across the
 *           batch.  The convention of genre_b200_render_views_*.  1 <= K <= 2^30, strides >= 0, tau > 0 finite.
 *   score   [N, K] fp32: score[n, k] = (sum_p c_p) / counts[n], with, in fp32, one rounding per operation:
 *             x_i = fma(rot[i][2], p_z, fma(rot[i][1], p_y, rot[i][0] * p_x)) + eye_i
 *             f_i = (x_i + 0.5) * R - 0.5
 *             c_p = v * v, v = the trilinear interpolation of field at f (render.cuh's make_taps_at /
 *                   sample_trilinear<false>), if 0 <= f_i <= R - 1 on all three axes; else c_p = tau * tau.
 *           The sum starts at 0 and adds c_0, c_1, ... in point order on one thread, so a candidate's score is bitwise
 *           repeatable and does not depend on K, on the other candidates or on the launch tiling.
 *   Every buffer 4-byte aligned (else GENRE_B200_EALIGN); arguments are checked before the launch.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_pose_score(const float *field, int64_t N, int res, const float *points, int64_t P, const int32_t *counts,
                          const float *rot, int64_t rN, int64_t rK, const float *eye, int64_t eN, int64_t eK, int64_t K,
                          float tau, float *score, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Conservative voxelisation of batched triangle meshes, the inverse of genre_b200_isosurface_*: ground-truth meshes become
 * grids for voxel_iou / voxel_fill and training targets without a CPU tool.
 *   meshes  the packed format of genre_b200_isosurface_*: verts [V, 3] fp32, faces [F, 3] int32 indexing the sample's own
 *           vertex block (trusted: in [0, V_n)), vert_off / face_off [N+1] int64 on the device.  F (the total) < 2^31,
 *           1 <= N <= 65535, every dimension of the D x H x W grid in [1, 512].
 *   frame   voxel (i0, i1, i2) is the closed cube [i_a/n_a - 0.5, (i_a+1)/n_a - 0.5] per axis, (n0, n1, n2) = (D, H, W), axis 0
 *           = vertex coordinate 0 = the first array axis (as genre_b200_isosurface_*).  Grid units, fp64 from the fp32 vertex:
 *           g_a = fl(fl(p_a + 0.5) * n_a); the voxel is then the box [i_a, i_a + 1].
 *   rule    a voxel is set iff the closed triangle and the closed cube intersect (touching counts: a face on a grid plane sets
 *           both layers, which makes voxel_fill sound on the result of a closed mesh).  Separating-axis test in grid units,
 *           fp64, one rounding per operation, no contraction, separation only by a strict inequality:
 *             box axes  i_a in [max(ceil(min_k g_ka) - 1, 0), min(floor(max_k g_ka), n_a - 1)];
 *             v_ka = g_ka - (i_a + 0.5); f0 = g1 - g0, f1 = g2 - g1, f2 = g0 - g2, e = g2 - g0;
 *             normal    m = (f0_1*e_2 - f0_2*e_1, f0_2*e_0 - f0_0*e_2, f0_0*e_1 - f0_1*e_0);
 *                       separated iff |(m0*v00 + m1*v01) + m2*v02| > 0.5 * ((|m0| + |m1|) + |m2|);
 *             edges     for each f_j and box axis a, the two non-zero components (A on s, B on t, s < t) of e_a x f_j:
 *                       a = 0: (-f_j2, f_j1) on (1, 2); a = 1: (f_j2, -f_j0) on (0, 2); a = 2: (-f_j1, f_j0) on (0, 1);
 *                       p_k = A*v_ks + B*v_kt, separated iff min_k p_k > 0.5*(|A| + |B|) or max_k p_k < -0.5*(|A| + |B|).
 *           A face with a non-finite vertex coordinate, or whose fp64 normal (b - a) x (c - a) from the fp32 vertices (the
 *           order of genre_b200_surface_sample's weight) is exactly 0, sets nothing.  Faces outside the grid are clipped.
 *   output  out [N, D, H, W] fp32, 1.0 for a set voxel and 0.0 elsewhere, written once and dense.  Deterministic and
 *           batch-equivariant; nothing is copied to the host (graph-capturable).  tests/mesh_voxelize_ref.py restates the
 *           contract in numpy, bit for bit.
 *   workspace: genre_b200_mesh_voxelize_workspace_bytes(N, F, D, H, W) bytes (0: unsupported), 16-byte aligned, caller-owned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_mesh_voxelize_workspace_bytes(int64_t N, int64_t F, int D, int H, int W);
int genre_b200_mesh_voxelize(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                             const int64_t *face_off, int64_t N, int D, int H, int W, float *out, void *workspace,
                             size_t workspace_bytes, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Generalized winding numbers of batched triangle meshes (Jacobson, Kavan & Sorkine-Hornung 2013), the exact sum over every
 * face: w(q) = sum_f Omega_f(q) / 4 pi, the signed solid angles of the faces seen from q.  1 inside and 0 outside a closed,
 * consistently oriented mesh; across holes and self-intersections it changes smoothly, so |w| > 0.5 is the intended solid.
 *   meshes  the packed format of genre_b200_isosurface_* / genre_b200_mesh_voxelize: verts [V, 3] fp32, faces [F, 3] int32
 *           indexing the sample's own vertex block (trusted: in [0, V_n)), vert_off / face_off [N+1] int64 on the device.
 *           F (the total) < 2^31, 1 <= N <= 65535.
 *   queries points mode (points != NULL): points [N|1, P, 3] fp32, sample n's table at points + n pN, pN = 3P or 0 (one
 *           table shared by the batch), 0 <= P < 2^31, D = H = W = 0; out [N, P].
 *           grid mode (points == NULL): P = pN = 0, every dimension of the D x H x W grid in [1, 512]; the query of voxel
 *           (i0, i1, i2) is its centre in genre_b200_mesh_voxelize's frame, c_a = fl(fl(i_a + 0.5) / n_a) - 0.5 in fp32
 *           ((n0, n1, n2) = (D, H, W), axis 0 = vertex coordinate 0); out [N, D, H, W].  Points mode fed these fp32 centres
 *           gives the same bits.
 *   skip    a face with a non-finite vertex coordinate, or whose fp64 normal (b - a) x (c - a) from the fp32 vertices is
 *           exactly 0 (genre_b200_mesh_voxelize's rule), contributes 0.
 *   term    for a kept face (v0, v1, v2) and query q, in fp32, one rounding per operation, fma only where written:
 *             n_x = fma(e1y, e2z, -(e1z*e2y)), n_y = fma(e1z, e2x, -(e1x*e2z)), n_z = fma(e1x, e2y, -(e1y*e2x)),
 *                   e1 = v1 - v0, e2 = v2 - v0;
 *             a = v0 - q, b = v1 - q, c = v2 - q;
 *             det = fma(a_z, n_z, fma(a_y, n_y, a_x*n_x))          (= a . (b x c) in exact arithmetic);
 *             la = sqrt(fma(a_z, a_z, fma(a_y, a_y, a_x*a_x))), lb, lc likewise (sqrt correctly rounded);
 *             ab = fma(a_z, b_z, fma(a_y, b_y, a_x*b_x)), bc = (b, c), ca = (c, a) likewise;
 *             den = fma(ca, lb, fma(bc, la, fma(ab, lc, (la*lb)*lc)));
 *             term = 0 if det == 0 (q on the face's plane, an edge or a vertex), else atan2f(det, den) = Omega_f / 2.
 *   sum     S = the fp64 sum of the terms, from 0, in face order on one thread; w = fl32(S * 0.15915494309189535) (the fp64
 *           value nearest 1 / 2 pi).  A sample without faces gives 0.  So w is bitwise repeatable and does not depend on
 *           the batch, on P, on the other samples or on the launch tiling.  tests/winding_ref.py restates the contract in
 *           fp64 with a per-query bound on this fp32 order's error.
 *   One launch (none when the query count is 0), no workspace, no host synchronisation: graph-capturable.  fp32 and int32
 *   buffers 4-byte aligned, offsets 8-byte aligned (else GENRE_B200_EALIGN); arguments are checked before the launch.
 * ------------------------------------------------------------------------------------------- */
int genre_b200_winding_number(const float *verts, int64_t V, const int32_t *faces, int64_t F, const int64_t *vert_off,
                              const int64_t *face_off, int64_t N, const float *points, int64_t P, int64_t pN, int D, int H,
                              int W, float *out, void *stream);

/* ---------------------------------------------------------------------------------------------
 * Input preprocessing: the test-time silhouette crop (util_img.get_bbox + util_img.crop of every preprocess_wrapper) and
 * MarrnetBaseModel.preprocess (models/marrnetbase.py:71-126), batched.  fp64 in the reference's operation order, one
 * rounding per operation, no FMA (fp32 only where stated); outputs rounded once to fp32, as convert_to_float32 does.
 *   sources  packed: data (bytes) and desc [B, 4] int64 on the device, (byte offset, H, W, C) per sample, dtype 0 uint8 or
 *            1 uint16, read as x / 255.0 or x / 65535.0; dense (desc NULL): [B, H, W, C] dtype 2 float32 or 3 float64.
 *            C in {1, 3, 4}: masks, depth and silhou read channel 0, rgb and normal channels 0..2.  Descriptors are trusted.
 *   crop     bbox = min / max row and column of mask > th (fp64); no such pixel: valid[b] = 0 and the sample's crops NaN.
 *            Window as util_img.crop with pad_zero=False: y1, x1, y2, x2 = (min col, min row, max col, max row),
 *            l = max(x2 - x1, y2 - y1) * out / (out - 2 pad), x1' = rint((x1 + x2) / 2 - l / 2), x2' = rint(... + l / 2),
 *            likewise y; the window reads clamped image rows and columns (edge padding).  cv2 INTER_LINEAR of the
 *            window (rows and columns scaled separately) to out x out: s = (d + 0.5) (n / out) - 0.5, taps floor(s) and
 *            floor(s) + 1 clamped into the window, weights (1 - f, f), horizontal pass then vertical.  The photo's three
 *            channels -> rgb [B, out, out, 3] fp64, the mask's channel 0 -> silhou [B, out, out] fp64 (or NULL).
 *   preprocess  kind 0 rgb, 1 depth, 2 silhou, 3 normal -> out [B, 3 or 1, S, S] fp32, S = im_size.  Square sources only.
 *            cv2 INTER_CUBIC n -> S: fx = (float)((d + 0.5) (1 / (S / n)) - 0.5), i = floor(fx), fx -= i, the four
 *            A = -0.75 coefficients in fp32 (c3 = 1 - c0 - c1 - c2), taps i-1 .. i+2 clamped, fp64 sums in tap order,
 *            horizontal then vertical.  depth / normal: clamp to the source's min and max (none if it holds a NaN), *
 *            scale_25d; silhou: clamp, 1 if > 0.999 else 0, * scale_25d; rgb: (x - mean_c) / std_c (ImageNet), and in
 *            train mode first the jitter steps order[b][k] (0 brightness, 1 contrast, 2 saturation) with alpha[b][k]:
 *            x = a x + (1 - a) * {0, m, gray(x)}, gray = (0.299 r + 0.587 g) + 0.114 b, then x_c += noise[b][c].  m = the mean
 *            of gray at the contrast step, summed in a fixed order (csrc/preprocess.cu).  order int32, alpha and noise fp64,
 *            [B, 3] each on the device.  Results depend only on the sample's own inputs.
 *            tests/preprocess_ref.py restates the whole contract in numpy, bit for bit.
 *   workspace: the _workspace_bytes query's bytes (0: unsupported), 16-byte aligned, caller-owned.
 * ------------------------------------------------------------------------------------------- */
size_t genre_b200_crop_to_render_workspace_bytes(int64_t B);
int genre_b200_crop_to_render(const void *img, const int64_t *img_desc, int img_dtype, const void *mask,
                              const int64_t *mask_desc, int mask_dtype, int64_t B, int out_size, double pad, double th,
                              double *rgb, double *silhou, uint8_t *valid, void *workspace, size_t workspace_bytes,
                              void *stream);
size_t genre_b200_preprocess_workspace_bytes(int kind, int train, int64_t B, int im_size);
int genre_b200_preprocess(int kind, int train, const void *src, const int64_t *desc, int dtype, int64_t B, int64_t H,
                          int64_t W, int64_t C, int im_size, double scale_25d, const int32_t *order, const double *alpha,
                          const double *noise, float *out, void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* GENRE_B200_H */
