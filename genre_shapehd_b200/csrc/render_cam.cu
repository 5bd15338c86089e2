// render_cam.cu — camera-view renderer of voxel occupancy grids and the differentiable ray-consistency loss, forward +
// backward.
//
// The camera is cam_bp's (cam_bp.cu cam_unproject): at o = (-cam_dist, 0, 0), looking along +x, focal length fl in
// pixels, so pixel (h, w) casts the ray o + t u with u = (fl, -imw, -imh) / |(fl, imw, imh)|, imh = h - (H-1)/2,
// imw = w - (W-1)/2, and t is cam_bp's ray depth.  Samples t_k = cam_dist - sqrt(3)/2 + k sqrt(3)/(Z-1) cover the unit
// cube for every ray.  Voxel (i, j, l) of vox[n] sits at cam_bp's voxel centre ((i+0.5)/R - 0.5, ...), so the trilinear
// coordinate of a point g is f = (g + 0.5) R - 0.5 (zero padding).  The stop-probability model is render_spherical's:
//     p_k = clamp(raw_k, 1e-5, 1 - 1e-5),   T_k = prod_{j<k} (1 - p_j),   s_k = p_k T_k,
// and a ray's value is an expected cost  V = sum_k s_k c_k + T_Z c_esc:
//     render           c_k = t_k, c_esc = bg (depth);  silhou = 1 - T_Z
//     ray consistency  obs > 0: c_k = |t_k - obs|, c_esc = miss;   obs <= 0: c_k = miss, c_esc = 0
// d V / d p_k = T_k c_k - (sum_{j>k} s_j c_j + T_Z c_esc) / (1 - p_k), zero where the clamp is active, scattered through
// the tap weights.  The backward of the renderer is the same walk with the cost g_depth t_k + g_silhou, escape g_depth bg
// (d silhou / d p_k is the expected cost of c_k = 1, c_esc = 0).
//
// Layout (as render_sph.cu): one warp per ray, lanes take 32 consecutive samples, the transmittance crosses lanes with a
// shuffle product-scan and crosses 32-sample chunks through a register carry; only [N,H,W] maps are written.  The
// backward walks each ray twice: forward, keeping each chunk's carry in shared memory (one float per chunk), then
// backward over the chunks, recomputing the samples, so the suffix sum is a running sum of the chunks already walked and
// T_k is the forward's value bit for bit.
//
// Sample coordinates (the arithmetic is part of the op's definition; tests/render_cam_ref.py restates it): in fp64, each
// operation rounded to nearest in this order (explicit intrinsics: never contracted),
//     nrm = sqrt((fl*fl + imw*imw) + imh*imh);  u = (fl / nrm, -imw / nrm, -imh / nrm)
//     t   = (cam_dist - sqrt(3)/2) + k * (sqrt(3) / (Z - 1))          (k * 0 for Z = 1)
//     g   = (t*ux - cam_dist, t*uy, t*uz);   f = (g + 0.5) * R - 0.5
// then f and t are each rounded once to fp32.  fl and cam_dist are the fp32 inputs widened exactly.  Everything after is
// fp32.
//
// Posed views (the *_views entry points): rays over [N, V, H, W], all V views of grid n reading vox[n] (the backward's
// atomics sum the views' gradients into it).  View (n, v) has a rotation rot (3x3 row-major, its columns the camera's
// axes in the grid frame), an eye e and fl; pixel (h, w) keeps the camera-frame u above, and the ray is, in the same
// fp64 arithmetic,
//     u'_i = (rot[i][0]*ux + rot[i][1]*uy) + rot[i][2]*uz;   d = sqrt((ex*ex + ey*ey) + ez*ez)
//     t    = (d - sqrt(3)/2) + k * (sqrt(3) / (Z - 1));      g = (t*u'x + ex, t*u'y + ey, t*u'z + ez)
// With rot = I and e = (-cam_dist, 0, 0) every value equals the fixed camera's bit for bit (products by 1 are exact,
// products by 0 add a signed zero, and the square root of a widened fp32 square is exact).  The fixed camera is the
// POSED = false instantiation of the same templates, with exactly the arithmetic above it.  It is not replaced by the
// posed instantiation at rot = I, which is slower on the fixed camera's calls: in kernel time, +1.0-1.9% for the render
// forward and +1.1-2.3% for the consistency forward, whose posed instance needs 48 registers instead of 40 (5 resident
// 256-thread CTAs per SM instead of 6); whole calls through such a routing lost 1-4% (DESIGN.md §4.2).
//
// Pose gradients (the *_views_backward_pose entry points; tests/render_pose_ref.py restates them): the derivative of
// this discrete op along its own samples, which move with |e|, with two simplifications that are part of the
// definition: the fp32 roundings of f_k and t_k count as the identity, and the trilinear interpolant is differentiated
// piecewise (on a voxel face, the one-sided derivative of the cell make_taps_at selects).  With w_k = dV/dp_k (the
// backward's dp: 0 where the clamp is active or raw is NaN), grad_k = R d raw / d f at f_k and c'_k = d c_k / d t_k
// (render g_depth; consistency scale sign(t_k - obs), 0 at equality and on background rays):
//     dV/du'_i = sum_k w_k t_k grad_k,i;   dV/dt(shift) = sum_k (w_k grad_k . u' + s_k c'_k)
//     dV/de_i  = sum_k w_k grad_k,i + (e_i / d) dV/dt(shift)
//     grad_rot[i][j] = sum over the view's rays of dV/du'_i u_j (the ambient gradient of the 9 entries);  grad_eye = sum dV/de
// Not differentiated: fl, obs; no double backward.
#include <initializer_list>

#include "render.cuh"

namespace gb {

constexpr int RC_THREADS = 256;  // 8 rays per CTA
constexpr int RC_WARPS = RC_THREADS / 32;
constexpr int RC_MAX_Z = 4096;
constexpr int RC_MAX_CHUNKS = RC_MAX_Z / 32;
constexpr int RC_MAX_RES = 1024;
constexpr int RC_MAX_HW = 16384;
constexpr double RC_SQRT3 = 1.7320508075688772;       // the double nearest sqrt(3)
constexpr double RC_HALF_SQRT3 = 0.8660254037844386;  // RC_SQRT3 / 2 (exact)

enum { RC_RENDER = 0, RC_CONSISTENCY = 1 };

struct CamRay {
  double ux, uy, uz;  // direction (grid frame)
  double ex, ey, ez;  // eye (the fixed camera uses ex = -cam_dist only)
  double t0, dt;      // first sample's depth, spacing
};

// pixel (h, w)'s camera-frame direction and the sample spacing
__device__ __forceinline__ CamRay cam_dir(float fl, int h, int w, int H, int W, int Z) {
  const double f = (double)fl;
  const double imh = (double)h - 0.5 * (double)(H - 1), imw = (double)w - 0.5 * (double)(W - 1);  // exact
  const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(f, f), __dmul_rn(imw, imw)), __dmul_rn(imh, imh)));
  CamRay r;
  r.ux = __ddiv_rn(f, nrm);
  r.uy = __ddiv_rn(-imw, nrm);
  r.uz = __ddiv_rn(-imh, nrm);
  r.dt = Z > 1 ? __ddiv_rn(RC_SQRT3, (double)(Z - 1)) : 0.0;
  return r;
}

// the fixed camera at (-cam_dist, 0, 0) looking along +x
__device__ __forceinline__ CamRay cam_ray(float fl, float cam_dist, int h, int w, int H, int W, int Z) {
  CamRay r = cam_dir(fl, h, w, H, W, Z);
  r.ex = -(double)cam_dist;
  r.t0 = __dadd_rn((double)cam_dist, -RC_HALF_SQRT3);
  return r;
}

// a posed view: rot [9] row-major, eye [3]
__device__ __forceinline__ CamRay cam_ray_posed(float fl, const float *__restrict__ rot, const float *__restrict__ eye,
                                                int h, int w, int H, int W, int Z) {
  const CamRay c = cam_dir(fl, h, w, H, W, Z);
  double m[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) m[i] = (double)__ldg(rot + i);
  CamRay r;
  r.ux = __dadd_rn(__dadd_rn(__dmul_rn(m[0], c.ux), __dmul_rn(m[1], c.uy)), __dmul_rn(m[2], c.uz));
  r.uy = __dadd_rn(__dadd_rn(__dmul_rn(m[3], c.ux), __dmul_rn(m[4], c.uy)), __dmul_rn(m[5], c.uz));
  r.uz = __dadd_rn(__dadd_rn(__dmul_rn(m[6], c.ux), __dmul_rn(m[7], c.uy)), __dmul_rn(m[8], c.uz));
  r.ex = (double)__ldg(eye);
  r.ey = (double)__ldg(eye + 1);
  r.ez = (double)__ldg(eye + 2);
  const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(r.ex, r.ex), __dmul_rn(r.ey, r.ey)), __dmul_rn(r.ez, r.ez)));
  r.t0 = __dadd_rn(d, -RC_HALF_SQRT3);
  r.dt = c.dt;
  return r;
}

// sample k of the ray: taps at its fp32 voxel coordinate (also stored in f when given), and its fp32 ray depth
template <bool POSED>
__device__ __forceinline__ float cam_sample(const CamRay &r, int k, int R, Taps &taps, float *f = nullptr) {
  const double Rd = (double)R;
  const double t = __dadd_rn(r.t0, __dmul_rn((double)k, r.dt));
  const double gx = __dadd_rn(__dmul_rn(t, r.ux), r.ex);
  const double gy = POSED ? __dadd_rn(__dmul_rn(t, r.uy), r.ey) : __dmul_rn(t, r.uy);
  const double gz = POSED ? __dadd_rn(__dmul_rn(t, r.uz), r.ez) : __dmul_rn(t, r.uz);
  const float fx = (float)__dadd_rn(__dmul_rn(__dadd_rn(gx, 0.5), Rd), -0.5);
  const float fy = (float)__dadd_rn(__dmul_rn(__dadd_rn(gy, 0.5), Rd), -0.5);
  const float fz = (float)__dadd_rn(__dmul_rn(__dadd_rn(gz, 0.5), Rd), -0.5);
  make_taps_at(fx, fy, fz, R, taps);
  if (f) {
    f[0] = fx;
    f[1] = fy;
    f[2] = fz;
  }
  return (float)t;
}

// cost c_k = a t_k + b, escape e: the renderer's depth (a = 1, b = 0, e = bg) and its backward's weighted sum of the
// depth and silhouette gradients
struct LinearCost {
  float a, b, e;
  __device__ __forceinline__ float at(float t) const { return fmaf(a, t, b); }
  __device__ __forceinline__ float esc() const { return e; }
  __device__ __forceinline__ float slope(float) const { return a; }  // d c_k / d t_k
};

// differentiable ray consistency against an observed ray depth (<= 0: background)
struct RayCost {
  float obs, miss;
  __device__ __forceinline__ float at(float t) const { return obs > 0.0f ? fabsf(t - obs) : miss; }
  __device__ __forceinline__ float esc() const { return obs > 0.0f ? miss : 0.0f; }
  __device__ __forceinline__ float slope(float t) const {  // sign(t - obs), 0 at equality and on background rays
    return obs > 0.0f ? (t > obs ? 1.0f : (t < obs ? -1.0f : 0.0f)) : 0.0f;
  }
};

// The forward walk: returns (sum_k s_k c_k, T_Z) to every lane.  With chunk_T, chunk c's carry (T before its first
// sample) is stored there and *last_chunk is the last chunk walked; the walk stops once T underflows to 0 (every later
// term, and every later gradient, is exactly 0).
template <bool POSED, class Cost>
__device__ __forceinline__ void cam_walk(const float *__restrict__ vol, int R, const CamRay &ray, int Z, const Cost &cost,
                                         float &sum, float &trans, float *chunk_T, int *last_chunk) {
  const int lane = threadIdx.x & 31;
  float carry = 1.0f, acc = 0.0f;
  for (int c = 0; c * 32 < Z; ++c) {
    const int k = c * 32 + lane;
    float p = 0.0f, ck = 0.0f;  // lanes past the end behave like p = 0 (factor 1, no contribution)
    if (k < Z) {
      Taps t;
      ck = cost.at(cam_sample<POSED>(ray, k, R, t));
      p = fminf(fmaxf(sample_trilinear<false>(vol, t, R, VoxPre{}), RS_PMIN), RS_PMAX);
    }
    if (chunk_T) {
      if (lane == 0) chunk_T[c] = carry;
      *last_chunk = c;
    }
    float total;
    const float before = carry * warp_excl_prod32(1.0f - p, total);
    if (k < Z) acc = fmaf(p * before, ck, acc);
    carry *= total;
    if (carry == 0.0f) break;  // warp-uniform
  }
  sum = warp_sum(acc);
  trans = carry;
}

struct CamArgs {
  const float *vox;
  int R, H, W, Z;
  long long n_rays;
  const float *fl, *cd;
  long long fN, dN;
  long long V;               // posed: views per grid (rays over [N,V,H,W])
  const float *rot, *eye;    // posed: 9 and 3 contiguous floats per view, strides (rN, rV), (eN, eV); fl strides (fN, fV)
  long long fV, rN, rV, eN, eV;
  float bg;                  // render: escape depth
  const float *obs;          // consistency: observed ray depth [N,(V,)H,W], strides (oN, (oV,) oH, oW)
  long long oN, oV, oH, oW;
  float miss;
  const float *g0, *g1;      // backward: grad_depth, grad_silhou (render) or grad_loss (consistency), [N,(V,)H,W] dense
  float *out0, *out1;        // forward: depth, silhou (render) or loss (consistency), [N,(V,)H,W] dense
  float *grad_vox;           // backward: [N,R,R,R] dense, accumulated
};

struct RayIndex {
  long long n, v;
  int h, w;
};

template <bool POSED>
__device__ __forceinline__ RayIndex ray_index(const CamArgs &a, long long ray) {
  const long long hw = (long long)a.H * a.W;
  RayIndex ri;
  const long long nv = ray / hw;
  const int pix = (int)(ray - nv * hw);
  if (POSED) {
    ri.n = nv / a.V;
    ri.v = nv - ri.n * a.V;
  } else {
    ri.n = nv;
    ri.v = 0;
  }
  ri.h = pix / a.W;
  ri.w = pix - ri.h * a.W;
  return ri;
}

template <bool POSED>
__device__ __forceinline__ CamRay ray_of(const CamArgs &a, const RayIndex &ri) {
  if (!POSED) return cam_ray(a.fl[ri.n * a.fN], a.cd[ri.n * a.dN], ri.h, ri.w, a.H, a.W, a.Z);
  return cam_ray_posed(a.fl[ri.n * a.fN + ri.v * a.fV], a.rot + ri.n * a.rN + ri.v * a.rV, a.eye + ri.n * a.eN + ri.v * a.eV,
                       ri.h, ri.w, a.H, a.W, a.Z);
}

template <bool POSED>
__device__ __forceinline__ float obs_of(const CamArgs &a, const RayIndex &ri) {
  return a.obs[ri.n * a.oN + (POSED ? ri.v * a.oV : 0) + ri.h * a.oH + ri.w * a.oW];
}

template <int MODE, bool POSED>
__global__ void __launch_bounds__(RC_THREADS) render_camera_forward_kernel(const CamArgs a) {
  const long long ray = (long long)blockIdx.x * RC_WARPS + (threadIdx.x >> 5);
  if (ray >= a.n_rays) return;
  const RayIndex ri = ray_index<POSED>(a, ray);
  const float *vol = a.vox + (size_t)ri.n * a.R * a.R * a.R;
  const CamRay r = ray_of<POSED>(a, ri);
  float sum, T;
  if (MODE == RC_RENDER) {
    const LinearCost cost{1.0f, 0.0f, a.bg};
    cam_walk<POSED>(vol, a.R, r, a.Z, cost, sum, T, nullptr, nullptr);
    if ((threadIdx.x & 31) == 0) {
      a.out0[ray] = fmaf(T, cost.esc(), sum);
      a.out1[ray] = 1.0f - T;
    }
  } else {
    const RayCost cost{obs_of<POSED>(a, ri), a.miss};
    cam_walk<POSED>(vol, a.R, r, a.Z, cost, sum, T, nullptr, nullptr);
    if ((threadIdx.x & 31) == 0) a.out0[ray] = fmaf(T, cost.esc(), sum);
  }
}

// the two walks of one ray; `scale` multiplies every gradient (the consistency loss's upstream gradient)
template <bool POSED, class Cost>
__device__ __forceinline__ void cam_backward_ray(const float *__restrict__ vol, float *__restrict__ gvol, int R,
                                                 const CamRay &ray, int Z, const Cost &cost, float scale, float *chunk_T) {
  const int lane = threadIdx.x & 31;
  float sum, T_Z;
  int last = 0;
  cam_walk<POSED>(vol, R, ray, Z, cost, sum, T_Z, chunk_T, &last);
  __syncwarp();
  float suffix = T_Z * cost.esc();  // sum over the chunks already walked of s_j c_j, plus the escape term
  for (int c = last; c >= 0; --c) {
    const int k = c * 32 + lane;
    const bool live = k < Z;
    float raw = 0.0f, p = 0.0f, ck = 0.0f;
    Taps t;
    if (live) {
      ck = cost.at(cam_sample<POSED>(ray, k, R, t));
      raw = sample_trilinear<false>(vol, t, R, VoxPre{});
      p = fminf(fmaxf(raw, RS_PMIN), RS_PMAX);
    }
    float total;
    const float Tk = chunk_T[c] * warp_excl_prod32(1.0f - p, total);  // the forward's T_k, bit for bit
    float chunk_sum;
    const float Ak = suffix + warp_excl_suffix_sum32(live ? p * Tk * ck : 0.0f, chunk_sum);
    suffix += chunk_sum;
    if (live && raw >= RS_PMIN && raw <= RS_PMAX) {  // NaN and clamped samples pass no gradient
      const float dp = scale * (Tk * ck - Ak / (1.0f - p));
      if (dp != 0.0f) {
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (t.valid & (1u << i)) atomicAdd(gvol + t.base + tap_offset(i, R), dp * t.w[i]);
      }
    }
  }
}

template <int MODE, bool POSED>
__global__ void __launch_bounds__(RC_THREADS) render_camera_backward_kernel(const CamArgs a) {
  __shared__ float s_T[RC_WARPS][RC_MAX_CHUNKS];
  const int warp = threadIdx.x >> 5;
  const long long ray = (long long)blockIdx.x * RC_WARPS + warp;
  if (ray >= a.n_rays) return;
  const RayIndex ri = ray_index<POSED>(a, ray);
  const size_t vol_off = (size_t)ri.n * a.R * a.R * a.R;  // every view of grid n scatters into grad_vox[n]
  const float g0 = a.g0[ray], g1 = MODE == RC_RENDER ? a.g1[ray] : 0.0f;
  if (g0 == 0.0f && g1 == 0.0f) return;  // warp-uniform
  const CamRay r = ray_of<POSED>(a, ri);
  if (MODE == RC_RENDER)
    cam_backward_ray<POSED>(a.vox + vol_off, a.grad_vox + vol_off, a.R, r, a.Z, LinearCost{g0, g1, g0 * a.bg}, 1.0f,
                            s_T[warp]);
  else
    cam_backward_ray<POSED>(a.vox + vol_off, a.grad_vox + vol_off, a.R, r, a.Z, RayCost{obs_of<POSED>(a, ri), a.miss}, g0,
                            s_T[warp]);
}

// ---- pose gradients of the posed views (the *_views_backward_pose entry points) ----------------------------------------
// Their own kernel, so that CamArgs and the kernels above keep their argument block and code.
struct PoseOut {
  float *grad_rot, *grad_eye;  // [N, V, 9] and [N, V, 3] dense
  double *part;                // workspace: per view, RP_TERMS rows of bpv per-CTA partial sums
  long long bpv;               // CTAs per view
};
constexpr int RP_TERMS = 13;   // (dV/du') (x) u: 9;  sum_k w_k grad_k: 3;  dV/dt(shift): 1

// cam_backward_ray's two walks (the same T_k, A_k, dp and voxel atomics, none without gvol) plus the ray's pose sums,
// each lane over its own samples, with g_k = d raw / d f at f_k in voxel units (the caller scales by R):
//   acc[0..2] = sum_k w_k t_k g_k,  acc[3..5] = sum_k w_k g_k,  acc[6] = sum_k w_k g_k . u',  acc[7] = sum_k s_k c'_k
// w_k = dp (zero where the clamp is active or raw is NaN), c'_k = scale * d c_k / d t_k.
template <class Cost>
__device__ __forceinline__ void cam_backward_ray_pose(const float *__restrict__ vol, float *__restrict__ gvol, int R,
                                                      const CamRay &ray, int Z, const Cost &cost, float scale,
                                                      float *chunk_T, float (&acc)[8]) {
  const int lane = threadIdx.x & 31;
  float sum, T_Z;
  int last = 0;
  cam_walk<true>(vol, R, ray, Z, cost, sum, T_Z, chunk_T, &last);
  __syncwarp();
  const float ux = (float)ray.ux, uy = (float)ray.uy, uz = (float)ray.uz;
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.0f;
  float suffix = T_Z * cost.esc();
  for (int c = last; c >= 0; --c) {
    const int k = c * 32 + lane;
    const bool live = k < Z;
    float raw = 0.0f, p = 0.0f, ck = 0.0f, tk = 0.0f, gx = 0.0f, gy = 0.0f, gz = 0.0f;
    Taps t;
    if (live) {
      float f[3];
      tk = cam_sample<true>(ray, k, R, t, f);
      ck = cost.at(tk);
      raw = sample_trilinear_grad(vol, t, R, f[0], f[1], f[2], gx, gy, gz);
      p = fminf(fmaxf(raw, RS_PMIN), RS_PMAX);
    }
    float total;
    const float Tk = chunk_T[c] * warp_excl_prod32(1.0f - p, total);  // the forward's T_k, bit for bit
    float chunk_sum;
    const float Ak = suffix + warp_excl_suffix_sum32(live ? p * Tk * ck : 0.0f, chunk_sum);
    suffix += chunk_sum;
    if (live) acc[7] = fmaf(p * Tk, scale * cost.slope(tk), acc[7]);
    if (live && raw >= RS_PMIN && raw <= RS_PMAX) {  // NaN and clamped samples pass no gradient
      const float dp = scale * (Tk * ck - Ak / (1.0f - p));
      if (dp != 0.0f) {
        if (gvol) {
#pragma unroll
          for (int i = 0; i < 8; ++i)
            if (t.valid & (1u << i)) atomicAdd(gvol + t.base + tap_offset(i, R), dp * t.w[i]);
        }
        const float wx = dp * gx, wy = dp * gy, wz = dp * gz;
        acc[0] = fmaf(wx, tk, acc[0]);
        acc[1] = fmaf(wy, tk, acc[1]);
        acc[2] = fmaf(wz, tk, acc[2]);
        acc[3] += wx;
        acc[4] += wy;
        acc[5] += wz;
        acc[6] = fmaf(wz, uz, fmaf(wy, uy, fmaf(wx, ux, acc[6])));
      }
    }
  }
}

// One CTA per 8 rays of one view (CTAs never straddle views): each warp reduces its ray's sums, and the CTA writes the
// RP_TERMS fp64 sums of its 8 rays, in warp order, to the workspace.  No atomics on the pose terms: bitwise repeatable.
template <int MODE>
__global__ void __launch_bounds__(RC_THREADS) render_views_pose_backward_kernel(const CamArgs a, const PoseOut po) {
  __shared__ float s_T[RC_WARPS][RC_MAX_CHUNKS];
  __shared__ double s_part[RC_WARPS][RP_TERMS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long hw = (long long)a.H * a.W;
  const long long view = blockIdx.x / po.bpv, blk = blockIdx.x - view * po.bpv;
  const long long pix = blk * RC_WARPS + warp;
  double part[RP_TERMS];
#pragma unroll
  for (int i = 0; i < RP_TERMS; ++i) part[i] = 0.0;
  if (pix < hw) {
    const long long ray = view * hw + pix;
    const float g0 = a.g0[ray], g1 = MODE == RC_RENDER ? a.g1[ray] : 0.0f;
    if (g0 != 0.0f || g1 != 0.0f) {  // warp-uniform
      const RayIndex ri = ray_index<true>(a, ray);
      const size_t vol_off = (size_t)ri.n * a.R * a.R * a.R;
      float *gvol = a.grad_vox ? a.grad_vox + vol_off : nullptr;
      const CamRay r = ray_of<true>(a, ri);
      float acc[8];
      if (MODE == RC_RENDER)
        cam_backward_ray_pose(a.vox + vol_off, gvol, a.R, r, a.Z, LinearCost{g0, g1, g0 * a.bg}, 1.0f, s_T[warp], acc);
      else
        cam_backward_ray_pose(a.vox + vol_off, gvol, a.R, r, a.Z, RayCost{obs_of<true>(a, ri), a.miss}, g0, s_T[warp],
                              acc);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = warp_sum(acc[i]);
      const CamRay u = cam_dir(a.fl[ri.n * a.fN + ri.v * a.fV], ri.h, ri.w, a.H, a.W, a.Z);  // camera-frame u
      const double Rd = (double)a.R, uc[3] = {u.ux, u.uy, u.uz};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
#pragma unroll
        for (int j = 0; j < 3; ++j) part[3 * i + j] = (double)acc[i] * Rd * uc[j];
        part[9 + i] = (double)acc[3 + i] * Rd;
      }
      part[12] = (double)acc[6] * Rd + (double)acc[7];
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < RP_TERMS; ++i) s_part[warp][i] = part[i];
  }
  __syncthreads();
  if (threadIdx.x < RP_TERMS) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < RC_WARPS; ++w) s += s_part[w][threadIdx.x];
    po.part[(view * RP_TERMS + threadIdx.x) * po.bpv + blk] = s;
  }
}

// One CTA per view: sums the view's partials in a fixed order (strided per thread, then a tree), and writes
// grad_rot[i][j] = sum (dV/du'_i) u_j and grad_eye = sum w_k grad_k + (e / |e|) dV/dt(shift), the |e| term once per view.
__global__ void __launch_bounds__(RC_THREADS) render_views_pose_reduce_kernel(const CamArgs a, const PoseOut po) {
  __shared__ double s[RP_TERMS][RC_THREADS];
  const long long view = blockIdx.x;
  const int tid = threadIdx.x;
#pragma unroll 1
  for (int c = 0; c < RP_TERMS; ++c) {
    const double *p = po.part + (view * RP_TERMS + c) * po.bpv;
    double acc = 0.0;
    for (long long b = tid; b < po.bpv; b += RC_THREADS) acc += p[b];
    s[c][tid] = acc;
  }
  __syncthreads();
  for (int w = RC_THREADS / 2; w > 0; w >>= 1) {
    if (tid < w)
      for (int c = 0; c < RP_TERMS; ++c) s[c][tid] += s[c][tid + w];
    __syncthreads();
  }
  if (tid == 0) {
    const long long n = view / a.V, v = view - n * a.V;
    const float *e = a.eye + n * a.eN + v * a.eV;
    const double ex = (double)e[0], ey = (double)e[1], ez = (double)e[2];
    const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)), __dmul_rn(ez, ez)));
    const double sh = s[12][0] / d;
    for (int i = 0; i < 9; ++i) po.grad_rot[view * 9 + i] = (float)s[i][0];
    po.grad_eye[view * 3 + 0] = (float)(s[9][0] + ex * sh);
    po.grad_eye[view * 3 + 1] = (float)(s[10][0] + ey * sh);
    po.grad_eye[view * 3 + 2] = (float)(s[11][0] + ez * sh);
  }
}

// ---- surface normals of the posed views (the *normal*_views entry points; tests/render_normal_ref.py restates them) ----
// The cameras, rays, samples t_k, f_k, taps, p_k, T_k and s_k are the posed views' above, with the same arithmetic.
//   sample normal     g_k = Res d raw / d f at f_k (sample_trilinear_grad, the cell make_taps_at selects, zero padding),
//                     rho_k = sqrt(|g_k|^2 + eps^2),  n_k = -g_k / rho_k  (outward: occupancy falls along n).  A NaN raw
//                     gives p_k = 1e-5 (the clamp's) and n_k = 0.  In fp32: rho = sqrtf(fma(gz,gz, fma(gy,gy,
//                     fma(gx,gx, eps*eps)))), n = -g / rho (one division per component).
//   rendered normal   normal = rot^T (sum_k s_k n_k): the sum in the grid frame, rotated once per ray after the warp
//                     reduction, normal_j = fma(rot[2][j], S_2, fma(rot[1][j], S_1, rot[0][j] S_0)).  Not renormalised;
//                     an escaping ray contributes 0.  Camera frame: x forward, +y towards image -w, +z towards image -h.
//   consistency       obs o [3] in the same camera frame; o = 0 (all three exactly 0) is background.  Otherwise
//                     m = rot o / |o| formed in fp64 ((rot[i][0] o_0 + rot[i][1] o_1) + rot[i][2] o_2, divided by
//                     sqrt((o_0^2 + o_1^2) + o_2^2)) and rounded once to fp32.  Foreground: c_k = 1 - n_k . m (the dot
//                     product an fma chain x, y, z), c_esc = miss; background: c_k = miss, c_esc = 0.
// Both modes are one cost family: c_k = c0 - n_k . a (render: a = -rot G, c0 = 0, per unit upstream G; consistency
// foreground: a = m, c0 = 1), whose gradient in g is d c_k / d g_k = (a - g_k (g_k . a) / rho_k^2) / rho_k.  rot G is
// formed like m (fp64, rounded once).  The grid gradient has two paths through the same 8 taps:
//   p path  dp_k = scale (T_k c_k - A_k / (1 - p_k)), zero where the clamp is active or raw is NaN (the posed walk's);
//   n path  at every sample with s_k != 0 (clamped or not, not NaN): h_k = scale s_k Res d c_k / d g_k, tap i gets
//           h_k . grad_f w_i (the 1-D weights' derivatives, +-1 times the two other axes' weights);
// summed into one atomicAdd per valid tap.  rot, eye, fl, obs and eps are not differentiated.
struct NormArgs {
  CamArgs c;          // posed cameras, Z, miss; c.g0 = upstream grad (render [N,V,3,H,W] dense, loss [N,V,H,W] dense)
  const float *obsn;  // consistency: observed normals [N,V,3,H,W], strides (oN, oV, oC, oH, oW)
  long long oN, oV, oC, oH, oW;
  float eps;
  float *out;         // forward: normal [N,V,3,H,W] or loss [N,V,H,W], dense
};

struct NormalCost {
  float ax, ay, az, c0, esc;
  bool fg;  // false: every stop costs `miss` (stored in c0), the normal does not enter
  __device__ __forceinline__ float at(float nx, float ny, float nz) const {
    return fg ? c0 - fmaf(nz, az, fmaf(ny, ay, nx * ax)) : c0;
  }
};

// fp32(rot v (/ |v| when normalise)) in fp64, the rounding stated above
__device__ __forceinline__ void rot_apply64(const float *__restrict__ rot, float v0, float v1, float v2, bool normalise,
                                            float &o0, float &o1, float &o2) {
  const double x = v0, y = v1, z = v2;
  const double nrm = normalise ? __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z))) : 1.0;
  double r[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const double s = __dadd_rn(__dadd_rn(__dmul_rn((double)__ldg(rot + 3 * i), x), __dmul_rn((double)__ldg(rot + 3 * i + 1), y)),
                               __dmul_rn((double)__ldg(rot + 3 * i + 2), z));
    r[i] = normalise ? __ddiv_rn(s, nrm) : s;
  }
  o0 = (float)r[0];
  o1 = (float)r[1];
  o2 = (float)r[2];
}

// sample k: p_k, the raw interpolant, g_k (grid frame, per unit length, 0 where raw is NaN), rho_k, n_k and the taps
struct NormSample {
  float raw, p, gx, gy, gz, rho, nx, ny, nz, t;
  float f[3];
};
__device__ __forceinline__ void normal_sample(const float *__restrict__ vol, int R, const CamRay &ray, int k, float eps,
                                              Taps &taps, NormSample &s) {
  s.t = cam_sample<true>(ray, k, R, taps, s.f);
  float dx, dy, dz;
  s.raw = sample_trilinear_grad(vol, taps, R, s.f[0], s.f[1], s.f[2], dx, dy, dz);
  s.p = fminf(fmaxf(s.raw, RS_PMIN), RS_PMAX);
  const float Rf = (float)R;
  const bool nan = s.raw != s.raw;
  s.gx = nan ? 0.0f : dx * Rf;
  s.gy = nan ? 0.0f : dy * Rf;
  s.gz = nan ? 0.0f : dz * Rf;
  s.rho = sqrtf(fmaf(s.gz, s.gz, fmaf(s.gy, s.gy, fmaf(s.gx, s.gx, eps * eps))));
  s.nx = -s.gx / s.rho;
  s.ny = -s.gy / s.rho;
  s.nz = -s.gz / s.rho;
}

template <int MODE>
__global__ void __launch_bounds__(RC_THREADS) render_normal_forward_kernel(const NormArgs a) {
  const long long ray = (long long)blockIdx.x * RC_WARPS + (threadIdx.x >> 5);
  if (ray >= a.c.n_rays) return;
  const int lane = threadIdx.x & 31;
  const RayIndex ri = ray_index<true>(a.c, ray);
  const float *vol = a.c.vox + (size_t)ri.n * a.c.R * a.c.R * a.c.R;
  const float *rot = a.c.rot + ri.n * a.c.rN + ri.v * a.c.rV;
  const CamRay r = ray_of<true>(a.c, ri);
  NormalCost cost{0.0f, 0.0f, 0.0f, a.c.miss, 0.0f, false};
  if (MODE == RC_CONSISTENCY) {
    const float *o = a.obsn + ri.n * a.oN + ri.v * a.oV + ri.h * a.oH + ri.w * a.oW;
    const float o0 = o[0], o1 = o[a.oC], o2 = o[2 * a.oC];
    if (o0 != 0.0f || o1 != 0.0f || o2 != 0.0f) {
      rot_apply64(rot, o0, o1, o2, true, cost.ax, cost.ay, cost.az);
      cost.c0 = 1.0f;
      cost.esc = a.c.miss;
      cost.fg = true;
    }
  }
  float carry = 1.0f, acc0 = 0.0f, acc1 = 0.0f, acc2 = 0.0f;
  for (int c = 0; c * 32 < a.c.Z; ++c) {
    const int k = c * 32 + lane;
    NormSample s;
    s.p = 0.0f;  // lanes past the end behave like p = 0 (factor 1, no contribution)
    if (k < a.c.Z) {
      Taps t;
      normal_sample(vol, a.c.R, r, k, a.eps, t, s);
    }
    float total;
    const float before = carry * warp_excl_prod32(1.0f - s.p, total);
    if (k < a.c.Z) {
      const float sk = s.p * before;
      if (MODE == RC_RENDER) {
        acc0 = fmaf(sk, s.nx, acc0);
        acc1 = fmaf(sk, s.ny, acc1);
        acc2 = fmaf(sk, s.nz, acc2);
      } else {
        acc0 = fmaf(sk, cost.at(s.nx, s.ny, s.nz), acc0);
      }
    }
    carry *= total;
    if (carry == 0.0f) break;  // warp-uniform
  }
  acc0 = warp_sum(acc0);
  if (MODE == RC_RENDER) {
    acc1 = warp_sum(acc1);
    acc2 = warp_sum(acc2);
    if (lane < 3) {
      const long long hw = (long long)a.c.H * a.c.W, nv = ray / hw, pix = ray - nv * hw;
      const float v = fmaf(__ldg(rot + 6 + lane), acc2, fmaf(__ldg(rot + 3 + lane), acc1, __ldg(rot + lane) * acc0));
      a.out[(nv * 3 + lane) * hw + pix] = v;
    }
  } else if (lane == 0) {
    a.out[ray] = fmaf(carry, cost.esc, acc0);
  }
}

template <int MODE>
__global__ void __launch_bounds__(RC_THREADS) render_normal_backward_kernel(const NormArgs a) {
  __shared__ float s_T[RC_WARPS][RC_MAX_CHUNKS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ray = (long long)blockIdx.x * RC_WARPS + warp;
  if (ray >= a.c.n_rays) return;
  const RayIndex ri = ray_index<true>(a.c, ray);
  const long long hw = (long long)a.c.H * a.c.W, nv = ray / hw, pix = ray - nv * hw;
  const float *rot = a.c.rot + ri.n * a.c.rN + ri.v * a.c.rV;
  NormalCost cost{0.0f, 0.0f, 0.0f, a.c.miss, 0.0f, false};
  float scale;
  if (MODE == RC_RENDER) {
    const float G0 = a.c.g0[nv * 3 * hw + pix], G1 = a.c.g0[(nv * 3 + 1) * hw + pix], G2 = a.c.g0[(nv * 3 + 2) * hw + pix];
    if (G0 == 0.0f && G1 == 0.0f && G2 == 0.0f) return;  // warp-uniform
    rot_apply64(rot, -G0, -G1, -G2, false, cost.ax, cost.ay, cost.az);
    cost.c0 = 0.0f;
    cost.fg = true;
    scale = 1.0f;
  } else {
    scale = a.c.g0[ray];
    if (scale == 0.0f) return;  // warp-uniform
    const float *o = a.obsn + ri.n * a.oN + ri.v * a.oV + ri.h * a.oH + ri.w * a.oW;
    const float o0 = o[0], o1 = o[a.oC], o2 = o[2 * a.oC];
    if (o0 != 0.0f || o1 != 0.0f || o2 != 0.0f) {
      rot_apply64(rot, o0, o1, o2, true, cost.ax, cost.ay, cost.az);
      cost.c0 = 1.0f;
      cost.esc = a.c.miss;
      cost.fg = true;
    }
  }
  const size_t vol_off = (size_t)ri.n * a.c.R * a.c.R * a.c.R;  // every view of grid n scatters into grad_vox[n]
  const float *vol = a.c.vox + vol_off;
  float *gvol = a.c.grad_vox + vol_off;
  const int R = a.c.R, Z = a.c.Z;
  const CamRay r = ray_of<true>(a.c, ri);
  // first walk: the chunk carries and T_Z (p depends on raw alone, so the plain walk's T_k are the forward's)
  float unused, T_Z;
  int last = 0;
  cam_walk<true>(vol, R, r, Z, LinearCost{0.0f, 0.0f, 0.0f}, unused, T_Z, s_T[warp], &last);
  __syncwarp();
  const float hR = scale * (float)R;
  float suffix = T_Z * cost.esc;
  for (int c = last; c >= 0; --c) {
    const int k = c * 32 + lane;
    const bool live = k < Z;
    NormSample s;
    Taps t;
    s.p = 0.0f;
    float ck = 0.0f;
    if (live) {
      normal_sample(vol, R, r, k, a.eps, t, s);
      ck = cost.at(s.nx, s.ny, s.nz);
    }
    float total;
    const float Tk = s_T[warp][c] * warp_excl_prod32(1.0f - s.p, total);  // the forward's T_k, bit for bit
    const float sk = s.p * Tk;
    float chunk_sum;
    const float Ak = suffix + warp_excl_suffix_sum32(live ? sk * ck : 0.0f, chunk_sum);
    suffix += chunk_sum;
    if (!live || s.raw != s.raw) continue;  // NaN samples pass nothing
    const float dp = (s.raw >= RS_PMIN && s.raw <= RS_PMAX) ? scale * (Tk * ck - Ak / (1.0f - s.p)) : 0.0f;
    float hx = 0.0f, hy = 0.0f, hz = 0.0f;
    if (cost.fg && sk != 0.0f) {
      const float inv = 1.0f / s.rho;
      const float ga = fmaf(s.gz, cost.az, fmaf(s.gy, cost.ay, s.gx * cost.ax));
      const float coef = ga * inv * inv;
      const float w = hR * sk * inv;
      hx = w * fmaf(-s.gx, coef, cost.ax);
      hy = w * fmaf(-s.gy, coef, cost.ay);
      hz = w * fmaf(-s.gz, coef, cost.az);
    }
    if (dp == 0.0f && hx == 0.0f && hy == 0.0f && hz == 0.0f) continue;
    const float x0f = floorf(s.f[0]), y0f = floorf(s.f[1]), z0f = floorf(s.f[2]);
    const float wx[2] = {(x0f + 1.0f) - s.f[0], s.f[0] - x0f};
    const float wy[2] = {(y0f + 1.0f) - s.f[1], s.f[1] - y0f};
    const float wz[2] = {(z0f + 1.0f) - s.f[2], s.f[2] - z0f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (!(t.valid & (1u << i))) continue;
      const int bx = (i >> 2) & 1, by = (i >> 1) & 1, bz = i & 1;
      const float dwx = (bx ? 1.0f : -1.0f) * (wy[by] * wz[bz]);
      const float dwy = (by ? 1.0f : -1.0f) * (wx[bx] * wz[bz]);
      const float dwz = (bz ? 1.0f : -1.0f) * (wx[bx] * wy[by]);
      const float v = fmaf(hz, dwz, fmaf(hy, dwy, fmaf(hx, dwx, dp * t.w[i])));
      if (v != 0.0f) atomicAdd(gvol + t.base + tap_offset(i, R), v);
    }
  }
}

// ---- depth and normal sketches together (the sketch_consistency_views entry points; tests/sketch_pose_ref.py restates
// them) --------------------------------------------------------------------------------------------------------------
// The cameras, rays, samples t_k, f_k, p_k, T_k, s_k are ray_consistency_views', bit for bit, and the sample normal
// n_k = -g_k / rho_k is render_normal_views'.  Each ray's cost is a weighted sum of the two consistency costs, each term
// with its own background rule:
//   depth   obs_d > 0: c^d_k = |t_k - obs_d|, c^d_esc = miss;   obs_d <= 0: c^d_k = miss, c^d_esc = 0
//   normal  obs_n != 0: c^n_k = 1 - n_k . m, c^n_esc = miss (m as normal_consistency_views');  obs_n = 0: miss, 0
//   c_k = fma(wn, c^n_k, wd c^d_k),   c_esc = fma(wn, c^n_esc, wd c^d_esc)
// so in exact arithmetic a ray's loss is wd L_depth + wn L_normal.  The grid gradient is the normal backward's two
// paths with this cost: the p path dp_k (clamp and NaN rules as there) and the n path h_k = scale wn s_k Res dc^n/dg_k.
// Pose gradients (the _backward_pose entry point) keep the definition of the file header; per sample, the position
// gradient is
//   q_k = w_k g_k + Res Hf_k h_k     (w_k = dp_k; g_k = Res d raw / d f; Hf_k = d2 raw / df2 in the cell make_taps_at
//                                     selects, zero diagonal; the n path at every non-NaN sample with s_k != 0)
// i.e. w_k grad_k + Res^2 Hf_k b_k with b_k = scale wn s_k (m - g (g . m) / rho^2) / rho.  From q_k the per-ray terms
//   dV/du' = sum_k t_k q_k,   dV/dt(shift) = sum_k (q_k . u' + s_k c'_k)  (c'_k = scale wd sign(t_k - obs_d): the normal
//   cost does not depend on t),   dV/de = sum_k q_k + (e / |e|) dV/dt(shift)
// and the frame term of m = rot o / |o|: a foreground-normal ray adds -scale wn S_i o_j / |o| to grad_rot[i][j], with
// S = sum_k s_k n_k (the ray's grid-frame sum, as render_normal_views').  The terms go to the pose backward's RP_TERMS
// per-CTA partials and render_views_pose_reduce_kernel sums them, so they are bitwise repeatable.
struct SketchArgs {
  NormArgs n;      // n.c: posed cameras, Z, miss, obs_d (c.obs, strides c.oN, c.oV, c.oH, c.oW), c.g0 = grad_loss,
                   // c.grad_vox; n.obsn: obs_n; n.eps; n.out = loss
  float wd, wn;
};

struct SketchCost {
  RayCost d;
  NormalCost n;
  float wd, wn;
  __device__ __forceinline__ float at(float t, float nx, float ny, float nz) const {
    return fmaf(wn, n.at(nx, ny, nz), wd * d.at(t));
  }
  __device__ __forceinline__ float esc() const { return fmaf(wn, n.esc, wd * d.esc()); }
  __device__ __forceinline__ float slope(float t) const { return wd * d.slope(t); }  // d c_k / d t_k
};

// the ray's costs; o = its observed normal (camera frame)
__device__ __forceinline__ SketchCost sketch_cost(const SketchArgs &a, const RayIndex &ri, const float *rot, float (&o)[3]) {
  SketchCost c;
  c.d = RayCost{obs_of<true>(a.n.c, ri), a.n.c.miss};
  c.n = NormalCost{0.0f, 0.0f, 0.0f, a.n.c.miss, 0.0f, false};
  c.wd = a.wd;
  c.wn = a.wn;
  const float *op = a.n.obsn + ri.n * a.n.oN + ri.v * a.n.oV + ri.h * a.n.oH + ri.w * a.n.oW;
  o[0] = op[0];
  o[1] = op[a.n.oC];
  o[2] = op[2 * a.n.oC];
  if (o[0] != 0.0f || o[1] != 0.0f || o[2] != 0.0f) {
    rot_apply64(rot, o[0], o[1], o[2], true, c.n.ax, c.n.ay, c.n.az);
    c.n.c0 = 1.0f;
    c.n.esc = a.n.c.miss;
    c.n.fg = true;
  }
  return c;
}

// normal_sample, and with HESS the interpolant's mixed second partials in f (0 otherwise)
template <bool HESS>
__device__ __forceinline__ void sketch_sample(const float *__restrict__ vol, int R, const CamRay &ray, int k, float eps,
                                              Taps &taps, NormSample &s, float &hxy, float &hxz, float &hyz) {
  if (!HESS) {
    normal_sample(vol, R, ray, k, eps, taps, s);
    hxy = hxz = hyz = 0.0f;
    return;
  }
  s.t = cam_sample<true>(ray, k, R, taps, s.f);
  float dx, dy, dz;
  s.raw = sample_trilinear_hess(vol, taps, R, s.f[0], s.f[1], s.f[2], dx, dy, dz, hxy, hxz, hyz);
  s.p = fminf(fmaxf(s.raw, RS_PMIN), RS_PMAX);
  const float Rf = (float)R;
  const bool nan = s.raw != s.raw;
  s.gx = nan ? 0.0f : dx * Rf;
  s.gy = nan ? 0.0f : dy * Rf;
  s.gz = nan ? 0.0f : dz * Rf;
  s.rho = sqrtf(fmaf(s.gz, s.gz, fmaf(s.gy, s.gy, fmaf(s.gx, s.gx, eps * eps))));
  s.nx = -s.gx / s.rho;
  s.ny = -s.gy / s.rho;
  s.nz = -s.gz / s.rho;
}

__global__ void __launch_bounds__(RC_THREADS) sketch_consistency_forward_kernel(const SketchArgs a) {
  const CamArgs &c = a.n.c;
  const long long ray = (long long)blockIdx.x * RC_WARPS + (threadIdx.x >> 5);
  if (ray >= c.n_rays) return;
  const int lane = threadIdx.x & 31;
  const RayIndex ri = ray_index<true>(c, ray);
  const float *vol = c.vox + (size_t)ri.n * c.R * c.R * c.R;
  const CamRay r = ray_of<true>(c, ri);
  float o[3];
  const SketchCost cost = sketch_cost(a, ri, c.rot + ri.n * c.rN + ri.v * c.rV, o);
  float carry = 1.0f, acc = 0.0f;
  for (int ch = 0; ch * 32 < c.Z; ++ch) {
    const int k = ch * 32 + lane;
    NormSample s;
    s.p = 0.0f;  // lanes past the end behave like p = 0 (factor 1, no contribution)
    if (k < c.Z) {
      Taps t;
      normal_sample(vol, c.R, r, k, a.n.eps, t, s);
    }
    float total;
    const float before = carry * warp_excl_prod32(1.0f - s.p, total);
    if (k < c.Z) acc = fmaf(s.p * before, cost.at(s.t, s.nx, s.ny, s.nz), acc);
    carry *= total;
    if (carry == 0.0f) break;  // warp-uniform
  }
  acc = warp_sum(acc);
  if (lane == 0) a.n.out[ray] = fmaf(carry, cost.esc(), acc);
}

// One ray's two walks: the grid gradient into gvol (skipped when null) and, with POSE, the ray's pose partials
// (RP_TERMS, the layout of render_views_pose_backward_kernel) in part, identical in every lane.
template <bool POSE>
__device__ __forceinline__ void sketch_backward_ray(const SketchArgs &a, long long ray, float scale, float *chunk_T,
                                                    double (&part)[RP_TERMS]) {
  const CamArgs &c = a.n.c;
  const int lane = threadIdx.x & 31;
  const RayIndex ri = ray_index<true>(c, ray);
  const float *rot = c.rot + ri.n * c.rN + ri.v * c.rV;
  float o[3];
  const SketchCost cost = sketch_cost(a, ri, rot, o);
  const size_t vol_off = (size_t)ri.n * c.R * c.R * c.R;  // every view of grid n scatters into grad_vox[n]
  const float *vol = c.vox + vol_off;
  float *gvol = POSE && !c.grad_vox ? nullptr : c.grad_vox + vol_off;  // null: pose only
  const int R = c.R, Z = c.Z;
  const float Rf = (float)R;
  const CamRay r = ray_of<true>(c, ri);
  // first walk: the chunk carries and T_Z (p depends on raw alone, so the plain walk's T_k are the forward's)
  float unused, T_Z;
  int last = 0;
  cam_walk<true>(vol, R, r, Z, LinearCost{0.0f, 0.0f, 0.0f}, unused, T_Z, chunk_T, &last);
  __syncwarp();
  const float hR = scale * a.wn * Rf;
  const float ux = (float)r.ux, uy = (float)r.uy, uz = (float)r.uz;
  // acc[0..2] = sum_k t_k q_k, acc[3..5] = sum_k q_k, acc[6] = sum_k q_k . u', acc[7] = sum_k s_k c'_k, acc[8..10] = S
  float acc[11];
#pragma unroll
  for (int i = 0; i < 11; ++i) acc[i] = 0.0f;
  float suffix = T_Z * cost.esc();
  for (int ch = last; ch >= 0; --ch) {
    const int k = ch * 32 + lane;
    const bool live = k < Z;
    NormSample s;
    Taps t;
    s.p = 0.0f;
    float ck = 0.0f, hxy = 0.0f, hxz = 0.0f, hyz = 0.0f;
    if (live) {
      sketch_sample<POSE>(vol, R, r, k, a.n.eps, t, s, hxy, hxz, hyz);
      ck = cost.at(s.t, s.nx, s.ny, s.nz);
    }
    float total;
    const float Tk = chunk_T[ch] * warp_excl_prod32(1.0f - s.p, total);  // the forward's T_k, bit for bit
    const float sk = s.p * Tk;
    float chunk_sum;
    const float Ak = suffix + warp_excl_suffix_sum32(live ? sk * ck : 0.0f, chunk_sum);
    suffix += chunk_sum;
    if (POSE && live) {
      acc[7] = fmaf(sk, scale * cost.slope(s.t), acc[7]);
      acc[8] = fmaf(sk, s.nx, acc[8]);
      acc[9] = fmaf(sk, s.ny, acc[9]);
      acc[10] = fmaf(sk, s.nz, acc[10]);
    }
    if (!live || s.raw != s.raw) continue;  // NaN samples pass nothing
    const float dp = (s.raw >= RS_PMIN && s.raw <= RS_PMAX) ? scale * (Tk * ck - Ak / (1.0f - s.p)) : 0.0f;
    float hx = 0.0f, hy = 0.0f, hz = 0.0f;
    if (cost.n.fg && sk != 0.0f) {
      const float inv = 1.0f / s.rho;
      const float ga = fmaf(s.gz, cost.n.az, fmaf(s.gy, cost.n.ay, s.gx * cost.n.ax));
      const float coef = ga * inv * inv;
      const float w = hR * sk * inv;
      hx = w * fmaf(-s.gx, coef, cost.n.ax);
      hy = w * fmaf(-s.gy, coef, cost.n.ay);
      hz = w * fmaf(-s.gz, coef, cost.n.az);
    }
    if (dp == 0.0f && hx == 0.0f && hy == 0.0f && hz == 0.0f) continue;
    if (POSE) {
      const float qx = fmaf(dp, s.gx, Rf * fmaf(hxz, hz, hxy * hy));
      const float qy = fmaf(dp, s.gy, Rf * fmaf(hyz, hz, hxy * hx));
      const float qz = fmaf(dp, s.gz, Rf * fmaf(hyz, hy, hxz * hx));
      acc[0] = fmaf(qx, s.t, acc[0]);
      acc[1] = fmaf(qy, s.t, acc[1]);
      acc[2] = fmaf(qz, s.t, acc[2]);
      acc[3] += qx;
      acc[4] += qy;
      acc[5] += qz;
      acc[6] = fmaf(qz, uz, fmaf(qy, uy, fmaf(qx, ux, acc[6])));
      if (!gvol) continue;
    }
    const float x0f = floorf(s.f[0]), y0f = floorf(s.f[1]), z0f = floorf(s.f[2]);
    const float wx[2] = {(x0f + 1.0f) - s.f[0], s.f[0] - x0f};
    const float wy[2] = {(y0f + 1.0f) - s.f[1], s.f[1] - y0f};
    const float wz[2] = {(z0f + 1.0f) - s.f[2], s.f[2] - z0f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (!(t.valid & (1u << i))) continue;
      const int bx = (i >> 2) & 1, by = (i >> 1) & 1, bz = i & 1;
      const float dwx = (bx ? 1.0f : -1.0f) * (wy[by] * wz[bz]);
      const float dwy = (by ? 1.0f : -1.0f) * (wx[bx] * wz[bz]);
      const float dwz = (bz ? 1.0f : -1.0f) * (wx[bx] * wy[by]);
      const float v = fmaf(hz, dwz, fmaf(hy, dwy, fmaf(hx, dwx, dp * t.w[i])));
      if (v != 0.0f) atomicAdd(gvol + t.base + tap_offset(i, R), v);
    }
  }
  if constexpr (POSE) {
#pragma unroll
    for (int i = 0; i < 11; ++i) acc[i] = warp_sum(acc[i]);
    const CamRay u = cam_dir(c.fl[ri.n * c.fN + ri.v * c.fV], ri.h, ri.w, c.H, c.W, c.Z);  // camera-frame u
    const double uc[3] = {u.ux, u.uy, u.uz};
    double oh[3] = {0.0, 0.0, 0.0}, fs = 0.0;  // the frame term's o / |o| (fp64) and -scale wn
    if (cost.n.fg) {
      const double x = o[0], y = o[1], z = o[2];
      const double nrm = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
      oh[0] = x / nrm;
      oh[1] = y / nrm;
      oh[2] = z / nrm;
      fs = -(double)scale * (double)a.wn;
    }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int j = 0; j < 3; ++j) part[3 * i + j] = (double)acc[i] * uc[j] + fs * (double)acc[8 + i] * oh[j];
      part[9 + i] = (double)acc[3 + i];
    }
    part[12] = (double)acc[6] + (double)acc[7];
  }
}

// POSE = false: one warp per ray over [N, V, H, W], the grid gradient only.  POSE = true: the layout of
// render_views_pose_backward_kernel (CTAs never straddle views; each writes its 8 rays' RP_TERMS fp64 sums, in warp
// order, to the workspace; grad_vox optional).
template <bool POSE>
__global__ void __launch_bounds__(RC_THREADS) sketch_consistency_backward_kernel(const SketchArgs a, const PoseOut po) {
  __shared__ float s_T[RC_WARPS][RC_MAX_CHUNKS];
  const int warp = threadIdx.x >> 5;
  double part[RP_TERMS];
  if constexpr (!POSE) {
    const long long ray = (long long)blockIdx.x * RC_WARPS + warp;
    if (ray >= a.n.c.n_rays) return;
    const float scale = a.n.c.g0[ray];
    if (scale != 0.0f) sketch_backward_ray<false>(a, ray, scale, s_T[warp], part);  // warp-uniform
    return;
  }
  __shared__ double s_part[RC_WARPS][RP_TERMS];
  const long long hw = (long long)a.n.c.H * a.n.c.W;
  const long long view = blockIdx.x / po.bpv, blk = blockIdx.x - view * po.bpv;
  const long long pix = blk * RC_WARPS + warp;
#pragma unroll
  for (int i = 0; i < RP_TERMS; ++i) part[i] = 0.0;
  if (pix < hw) {
    const long long ray = view * hw + pix;
    const float scale = a.n.c.g0[ray];
    if (scale != 0.0f) sketch_backward_ray<true>(a, ray, scale, s_T[warp], part);  // warp-uniform
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int i = 0; i < RP_TERMS; ++i) s_part[warp][i] = part[i];
  }
  __syncthreads();
  if (threadIdx.x < RP_TERMS) {
    double s = 0.0;
#pragma unroll
    for (int w = 0; w < RC_WARPS; ++w) s += s_part[w][threadIdx.x];
    po.part[(view * RP_TERMS + threadIdx.x) * po.bpv + blk] = s;
  }
}

static bool aligned4(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 3u) == 0; }

constexpr long long RC_MAX_RAYS = 1ll << 34;

// the checks every entry point shares: rays over [N, V, H, W] (V = 1: the fixed camera), and the camera's pointers cams
// (fl and camdist, or fl, rot and eye; named in cam_names)
static int rc_check(const char *what, const float *vox, int64_t N, int64_t V, int res, int64_t H, int64_t W, int Z,
                    std::initializer_list<const float *> cams, const char *cam_names, CamArgs &a) {
  bool cams_set = true, cams_aligned = true;
  for (const float *p : cams) {
    cams_set = cams_set && p;
    cams_aligned = cams_aligned && aligned4(p);
  }
  GB_REQUIRE(vox && cams_set, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(res >= 2 && res <= RC_MAX_RES, GENRE_B200_EINVAL, "%s: resolution %d unsupported (2..%d)", what, res,
             RC_MAX_RES);
  GB_REQUIRE(H >= 1 && W >= 1 && H <= RC_MAX_HW && W <= RC_MAX_HW, GENRE_B200_EINVAL,
             "%s: image size %lld x %lld unsupported (1..%d per side)", what, (long long)H, (long long)W, RC_MAX_HW);
  GB_REQUIRE(Z >= 1 && Z <= RC_MAX_Z, GENRE_B200_EINVAL, "%s: z_res %d unsupported (1..%d)", what, Z, RC_MAX_Z);
  GB_REQUIRE(V >= 1 && V <= RC_MAX_RAYS, GENRE_B200_EINVAL, "%s: %lld views unsupported (1 .. 2^34)", what, (long long)V);
  GB_REQUIRE(N >= 1 && N <= RC_MAX_RAYS / V && (N * V * H * W + RC_WARPS - 1) / RC_WARPS < (1ll << 31), GENRE_B200_EINVAL,
             "%s: batch %lld unsupported (1 .. 2^34 / (%sH W) rays)", what, (long long)N, V == 1 ? "" : "V ");
  GB_REQUIRE(aligned4(vox) && cams_aligned, GENRE_B200_EALIGN, "%s: vox, %s must be 4-byte aligned", what, cam_names);
  a = CamArgs{};
  a.vox = vox;
  a.R = res;
  a.H = (int)H;
  a.W = (int)W;
  a.Z = Z;
  a.V = V;
  a.n_rays = (long long)N * V * H * W;
  return 0;
}

// the posed views' checks and camera arguments
static int rv_check(const char *what, const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int Z,
                    const float *fl, int64_t fN, int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye,
                    int64_t eN, int64_t eV, CamArgs &a) {
  if (int rc = rc_check(what, vox, N, V, res, H, W, Z, {fl, rot, eye}, "fl, rot and eye", a)) return rc;
  a.fl = fl;
  a.fN = fN;
  a.fV = fV;
  a.rot = rot;
  a.rN = rN;
  a.rV = rV;
  a.eye = eye;
  a.eN = eN;
  a.eV = eV;
  return 0;
}

static unsigned rc_grid(const CamArgs &a) { return (unsigned)((a.n_rays + RC_WARPS - 1) / RC_WARPS); }

static long long rp_bpv(int64_t H, int64_t W) { return ((long long)H * W + RC_WARPS - 1) / RC_WARPS; }

// the pose outputs' and the workspace's checks; po.bpv is the CTAs per view
static int rp_check(const char *what, const CamArgs &a, int64_t N, int64_t V, float *grad_vox, float *grad_rot,
                    float *grad_eye, void *workspace, size_t workspace_bytes, PoseOut &po) {
  const long long bpv = rp_bpv(a.H, a.W);
  GB_REQUIRE(bpv <= ((1ll << 31) - 1) / ((long long)N * V), GENRE_B200_EINVAL,
             "%s: %lld views of %lld CTAs unsupported (fewer than 2^31 CTAs)", what, (long long)(N * V), bpv);
  GB_REQUIRE(grad_rot && grad_eye && workspace, GENRE_B200_EINVAL, "%s: null grad_rot, grad_eye or workspace", what);
  GB_REQUIRE(aligned4(grad_rot) && aligned4(grad_eye) && (grad_vox == nullptr || aligned4(grad_vox)), GENRE_B200_EALIGN,
             "%s: grad_vox, grad_rot and grad_eye must be 4-byte aligned", what);
  GB_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, GENRE_B200_EALIGN,
             "%s: workspace must be 8-byte aligned", what);
  const size_t need = (size_t)N * V * RP_TERMS * bpv * sizeof(double);
  GB_REQUIRE(workspace_bytes >= need, GENRE_B200_EWORKSPACE, "%s: workspace too small (%zu bytes, %zu needed)", what,
             workspace_bytes, need);
  po.grad_rot = grad_rot;
  po.grad_eye = grad_eye;
  po.part = static_cast<double *>(workspace);
  po.bpv = bpv;
  return 0;
}

template <int MODE>
static int rp_launch(const char *what, const CamArgs &a, const PoseOut &po, void *stream) {
  const long long views = a.n_rays / ((long long)a.H * a.W);
  render_views_pose_backward_kernel<MODE><<<(unsigned)(views * po.bpv), RC_THREADS, 0, as_stream(stream)>>>(a, po);
  if (int rc = check_launch(what)) return rc;
  render_views_pose_reduce_kernel<<<(unsigned)views, RC_THREADS, 0, as_stream(stream)>>>(a, po);
  return check_launch(what);
}

}  // namespace gb

using namespace gb;

extern "C" int genre_b200_render_camera_forward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                                const float *fl, int64_t fN, const float *camdist, int64_t dN, float bg,
                                                float *depth, float *silhou, void *stream) {
  CamArgs a;
  if (int rc = rc_check("render_camera", vox, N, 1, res, H, W, z_res, {fl, camdist}, "fl and camdist", a)) return rc;
  GB_REQUIRE(depth && silhou, GENRE_B200_EINVAL, "render_camera: null output");
  GB_REQUIRE(aligned4(depth) && aligned4(silhou), GENRE_B200_EALIGN, "render_camera: outputs must be 4-byte aligned");
  a.fl = fl;
  a.cd = camdist;
  a.fN = fN;
  a.dN = dN;
  a.bg = bg;
  a.out0 = depth;
  a.out1 = silhou;
  render_camera_forward_kernel<RC_RENDER, false><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("render_camera forward kernel");
}

extern "C" int genre_b200_render_camera_backward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                                 const float *fl, int64_t fN, const float *camdist, int64_t dN, float bg,
                                                 const float *grad_depth, const float *grad_silhou, float *grad_vox,
                                                 void *stream) {
  CamArgs a;
  if (int rc = rc_check("render_camera backward", vox, N, 1, res, H, W, z_res, {fl, camdist}, "fl and camdist", a)) return rc;
  GB_REQUIRE(grad_depth && grad_silhou && grad_vox, GENRE_B200_EINVAL, "render_camera backward: null pointer");
  GB_REQUIRE(aligned4(grad_depth) && aligned4(grad_silhou) && aligned4(grad_vox), GENRE_B200_EALIGN,
             "render_camera backward: gradients must be 4-byte aligned");
  a.fl = fl;
  a.cd = camdist;
  a.fN = fN;
  a.dN = dN;
  a.bg = bg;
  a.g0 = grad_depth;
  a.g1 = grad_silhou;
  a.grad_vox = grad_vox;
  render_camera_backward_kernel<RC_RENDER, false><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("render_camera backward kernel");
}

extern "C" int genre_b200_ray_consistency_forward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                                  const float *fl, int64_t fN, const float *camdist, int64_t dN,
                                                  const float *obs, int64_t oN, int64_t oH, int64_t oW, float miss_cost,
                                                  float *loss, void *stream) {
  CamArgs a;
  if (int rc = rc_check("ray_consistency", vox, N, 1, res, H, W, z_res, {fl, camdist}, "fl and camdist", a)) return rc;
  GB_REQUIRE(obs && loss, GENRE_B200_EINVAL, "ray_consistency: null pointer");
  GB_REQUIRE(aligned4(obs) && aligned4(loss), GENRE_B200_EALIGN, "ray_consistency: obs and loss must be 4-byte aligned");
  a.fl = fl;
  a.cd = camdist;
  a.fN = fN;
  a.dN = dN;
  a.obs = obs;
  a.oN = oN;
  a.oH = oH;
  a.oW = oW;
  a.miss = miss_cost;
  a.out0 = loss;
  render_camera_forward_kernel<RC_CONSISTENCY, false><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("ray_consistency forward kernel");
}

extern "C" int genre_b200_ray_consistency_backward(const float *vox, int64_t N, int res, int64_t H, int64_t W, int z_res,
                                                   const float *fl, int64_t fN, const float *camdist, int64_t dN,
                                                   const float *obs, int64_t oN, int64_t oH, int64_t oW, float miss_cost,
                                                   const float *grad_loss, float *grad_vox, void *stream) {
  CamArgs a;
  if (int rc = rc_check("ray_consistency backward", vox, N, 1, res, H, W, z_res, {fl, camdist}, "fl and camdist", a)) return rc;
  GB_REQUIRE(obs && grad_loss && grad_vox, GENRE_B200_EINVAL, "ray_consistency backward: null pointer");
  GB_REQUIRE(aligned4(obs) && aligned4(grad_loss) && aligned4(grad_vox), GENRE_B200_EALIGN,
             "ray_consistency backward: obs and gradients must be 4-byte aligned");
  a.fl = fl;
  a.cd = camdist;
  a.fN = fN;
  a.dN = dN;
  a.obs = obs;
  a.oN = oN;
  a.oH = oH;
  a.oW = oW;
  a.miss = miss_cost;
  a.g0 = grad_loss;
  a.grad_vox = grad_vox;
  render_camera_backward_kernel<RC_CONSISTENCY, false><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("ray_consistency backward kernel");
}

extern "C" int genre_b200_render_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                               int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                               int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, float bg,
                                               float *depth, float *silhou, void *stream) {
  CamArgs a;
  if (int rc = rv_check("render_views", vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, a)) return rc;
  GB_REQUIRE(depth && silhou, GENRE_B200_EINVAL, "render_views: null output");
  GB_REQUIRE(aligned4(depth) && aligned4(silhou), GENRE_B200_EALIGN, "render_views: outputs must be 4-byte aligned");
  a.bg = bg;
  a.out0 = depth;
  a.out1 = silhou;
  render_camera_forward_kernel<RC_RENDER, true><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("render_views forward kernel");
}

extern "C" int genre_b200_render_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W,
                                                int z_res, const float *fl, int64_t fN, int64_t fV, const float *rot,
                                                int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, float bg,
                                                const float *grad_depth, const float *grad_silhou, float *grad_vox,
                                                void *stream) {
  CamArgs a;
  if (int rc = rv_check("render_views backward", vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, a))
    return rc;
  GB_REQUIRE(grad_depth && grad_silhou && grad_vox, GENRE_B200_EINVAL, "render_views backward: null pointer");
  GB_REQUIRE(aligned4(grad_depth) && aligned4(grad_silhou) && aligned4(grad_vox), GENRE_B200_EALIGN,
             "render_views backward: gradients must be 4-byte aligned");
  a.bg = bg;
  a.g0 = grad_depth;
  a.g1 = grad_silhou;
  a.grad_vox = grad_vox;
  render_camera_backward_kernel<RC_RENDER, true><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("render_views backward kernel");
}

extern "C" int genre_b200_ray_consistency_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                        int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                        const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                        int64_t eN, int64_t eV, const float *obs, int64_t oN, int64_t oV,
                                                        int64_t oH, int64_t oW, float miss_cost, float *loss,
                                                        void *stream) {
  CamArgs a;
  if (int rc = rv_check("ray_consistency_views", vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, a))
    return rc;
  GB_REQUIRE(obs && loss, GENRE_B200_EINVAL, "ray_consistency_views: null pointer");
  GB_REQUIRE(aligned4(obs) && aligned4(loss), GENRE_B200_EALIGN,
             "ray_consistency_views: obs and loss must be 4-byte aligned");
  a.obs = obs;
  a.oN = oN;
  a.oV = oV;
  a.oH = oH;
  a.oW = oW;
  a.miss = miss_cost;
  a.out0 = loss;
  render_camera_forward_kernel<RC_CONSISTENCY, true><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("ray_consistency_views forward kernel");
}

extern "C" int genre_b200_ray_consistency_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                         int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                         const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                         int64_t eN, int64_t eV, const float *obs, int64_t oN, int64_t oV,
                                                         int64_t oH, int64_t oW, float miss_cost, const float *grad_loss,
                                                         float *grad_vox, void *stream) {
  CamArgs a;
  if (int rc = rv_check("ray_consistency_views backward", vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN,
                        eV, a))
    return rc;
  GB_REQUIRE(obs && grad_loss && grad_vox, GENRE_B200_EINVAL, "ray_consistency_views backward: null pointer");
  GB_REQUIRE(aligned4(obs) && aligned4(grad_loss) && aligned4(grad_vox), GENRE_B200_EALIGN,
             "ray_consistency_views backward: obs and gradients must be 4-byte aligned");
  a.obs = obs;
  a.oN = oN;
  a.oV = oV;
  a.oH = oH;
  a.oW = oW;
  a.miss = miss_cost;
  a.g0 = grad_loss;
  a.grad_vox = grad_vox;
  render_camera_backward_kernel<RC_CONSISTENCY, true><<<rc_grid(a), RC_THREADS, 0, as_stream(stream)>>>(a);
  return check_launch("ray_consistency_views backward kernel");
}

extern "C" size_t genre_b200_render_views_pose_workspace_bytes(int64_t N, int64_t V, int64_t H, int64_t W) {
  if (N < 1 || V < 1 || H < 1 || W < 1) return 0;
  return (size_t)N * V * RP_TERMS * rp_bpv(H, W) * sizeof(double);
}

extern "C" int genre_b200_render_views_backward_pose(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                     int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                     const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                     int64_t eN, int64_t eV, float bg, const float *grad_depth,
                                                     const float *grad_silhou, float *grad_vox, float *grad_rot,
                                                     float *grad_eye, void *workspace, size_t workspace_bytes,
                                                     void *stream) {
  CamArgs a;
  PoseOut po;
  const char *what = "render_views backward_pose";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, a)) return rc;
  GB_REQUIRE(grad_depth && grad_silhou, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(aligned4(grad_depth) && aligned4(grad_silhou), GENRE_B200_EALIGN,
             "%s: gradients must be 4-byte aligned", what);
  if (int rc = rp_check(what, a, N, V, grad_vox, grad_rot, grad_eye, workspace, workspace_bytes, po)) return rc;
  a.bg = bg;
  a.g0 = grad_depth;
  a.g1 = grad_silhou;
  a.grad_vox = grad_vox;
  return rp_launch<RC_RENDER>("render_views backward_pose kernels", a, po, stream);
}

extern "C" int genre_b200_ray_consistency_views_backward_pose(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV, const float *obs,
    int64_t oN, int64_t oV, int64_t oH, int64_t oW, float miss_cost, const float *grad_loss, float *grad_vox,
    float *grad_rot, float *grad_eye, void *workspace, size_t workspace_bytes, void *stream) {
  CamArgs a;
  PoseOut po;
  const char *what = "ray_consistency_views backward_pose";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, a)) return rc;
  GB_REQUIRE(obs && grad_loss, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(aligned4(obs) && aligned4(grad_loss), GENRE_B200_EALIGN, "%s: obs and grad_loss must be 4-byte aligned",
             what);
  if (int rc = rp_check(what, a, N, V, grad_vox, grad_rot, grad_eye, workspace, workspace_bytes, po)) return rc;
  a.obs = obs;
  a.oN = oN;
  a.oV = oV;
  a.oH = oH;
  a.oW = oW;
  a.miss = miss_cost;
  a.g0 = grad_loss;
  a.grad_vox = grad_vox;
  return rp_launch<RC_CONSISTENCY>("ray_consistency_views backward_pose kernels", a, po, stream);
}

// ---- surface normals of the posed views ----------------------------------------------------------------------------
static int rn_check(const char *what, float eps, NormArgs &n) {
  GB_REQUIRE(eps > 0.0f && eps <= 3.4e38f, GENRE_B200_EINVAL, "%s: eps %g must be positive and finite", what, (double)eps);
  n.eps = eps;
  return 0;
}

template <int MODE, bool FORWARD>
static int rn_launch(const char *what, const NormArgs &n, void *stream) {
  const unsigned grid = rc_grid(n.c);
  if (FORWARD)
    render_normal_forward_kernel<MODE><<<grid, RC_THREADS, 0, as_stream(stream)>>>(n);
  else
    render_normal_backward_kernel<MODE><<<grid, RC_THREADS, 0, as_stream(stream)>>>(n);
  return check_launch(what);
}

extern "C" int genre_b200_render_normal_views_forward(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                      int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                      const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                      int64_t eN, int64_t eV, float eps, float *normal, void *stream) {
  NormArgs n{};
  const char *what = "render_normal_views";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, n.c)) return rc;
  if (int rc = rn_check(what, eps, n)) return rc;
  GB_REQUIRE(normal, GENRE_B200_EINVAL, "%s: null output", what);
  GB_REQUIRE(aligned4(normal), GENRE_B200_EALIGN, "%s: normal must be 4-byte aligned", what);
  n.out = normal;
  return rn_launch<RC_RENDER, true>("render_normal_views forward kernel", n, stream);
}

extern "C" int genre_b200_render_normal_views_backward(const float *vox, int64_t N, int res, int64_t V, int64_t H,
                                                       int64_t W, int z_res, const float *fl, int64_t fN, int64_t fV,
                                                       const float *rot, int64_t rN, int64_t rV, const float *eye,
                                                       int64_t eN, int64_t eV, float eps, const float *grad_normal,
                                                       float *grad_vox, void *stream) {
  NormArgs n{};
  const char *what = "render_normal_views backward";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, n.c)) return rc;
  if (int rc = rn_check(what, eps, n)) return rc;
  GB_REQUIRE(grad_normal && grad_vox, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(aligned4(grad_normal) && aligned4(grad_vox), GENRE_B200_EALIGN, "%s: gradients must be 4-byte aligned",
             what);
  n.c.g0 = grad_normal;
  n.c.grad_vox = grad_vox;
  return rn_launch<RC_RENDER, false>("render_normal_views backward kernel", n, stream);
}

static int nc_obs(const char *what, const float *obs_normal, int64_t oN, int64_t oV, int64_t oC, int64_t oH, int64_t oW,
                  float miss_cost, NormArgs &n) {
  GB_REQUIRE(obs_normal, GENRE_B200_EINVAL, "%s: null obs_normal", what);
  GB_REQUIRE(aligned4(obs_normal), GENRE_B200_EALIGN, "%s: obs_normal must be 4-byte aligned", what);
  n.obsn = obs_normal;
  n.oN = oN;
  n.oV = oV;
  n.oC = oC;
  n.oH = oH;
  n.oW = oW;
  n.c.miss = miss_cost;
  return 0;
}

extern "C" int genre_b200_normal_consistency_views_forward(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_normal, int64_t oN, int64_t oV, int64_t oC, int64_t oH, int64_t oW, float miss_cost, float eps,
    float *loss, void *stream) {
  NormArgs n{};
  const char *what = "normal_consistency_views";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, n.c)) return rc;
  if (int rc = rn_check(what, eps, n)) return rc;
  if (int rc = nc_obs(what, obs_normal, oN, oV, oC, oH, oW, miss_cost, n)) return rc;
  GB_REQUIRE(loss, GENRE_B200_EINVAL, "%s: null output", what);
  GB_REQUIRE(aligned4(loss), GENRE_B200_EALIGN, "%s: loss must be 4-byte aligned", what);
  n.out = loss;
  return rn_launch<RC_CONSISTENCY, true>("normal_consistency_views forward kernel", n, stream);
}

extern "C" int genre_b200_normal_consistency_views_backward(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_normal, int64_t oN, int64_t oV, int64_t oC, int64_t oH, int64_t oW, float miss_cost, float eps,
    const float *grad_loss, float *grad_vox, void *stream) {
  NormArgs n{};
  const char *what = "normal_consistency_views backward";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, n.c)) return rc;
  if (int rc = rn_check(what, eps, n)) return rc;
  if (int rc = nc_obs(what, obs_normal, oN, oV, oC, oH, oW, miss_cost, n)) return rc;
  GB_REQUIRE(grad_loss && grad_vox, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(aligned4(grad_loss) && aligned4(grad_vox), GENRE_B200_EALIGN, "%s: gradients must be 4-byte aligned", what);
  n.c.g0 = grad_loss;
  n.c.grad_vox = grad_vox;
  return rn_launch<RC_CONSISTENCY, false>("normal_consistency_views backward kernel", n, stream);
}

// ---- depth and normal sketches together -----------------------------------------------------------------------------
static int sk_check(const char *what, const float *obs_depth, int64_t odN, int64_t odV, int64_t odH, int64_t odW,
                    const float *obs_normal, int64_t onN, int64_t onV, int64_t onC, int64_t onH, int64_t onW, float wd,
                    float wn, float miss_cost, float eps, SketchArgs &s) {
  if (int rc = rn_check(what, eps, s.n)) return rc;
  if (int rc = nc_obs(what, obs_normal, onN, onV, onC, onH, onW, miss_cost, s.n)) return rc;
  GB_REQUIRE(obs_depth, GENRE_B200_EINVAL, "%s: null obs_depth", what);
  GB_REQUIRE(aligned4(obs_depth), GENRE_B200_EALIGN, "%s: obs_depth must be 4-byte aligned", what);
  const float fmax = 3.402823466e38f;
  GB_REQUIRE(wd >= 0.0f && wd <= fmax && wn >= 0.0f && wn <= fmax && (wd > 0.0f || wn > 0.0f), GENRE_B200_EINVAL,
             "%s: weights %g, %g must be finite and >= 0, one of them > 0", what, (double)wd, (double)wn);
  s.n.c.obs = obs_depth;
  s.n.c.oN = odN;
  s.n.c.oV = odV;
  s.n.c.oH = odH;
  s.n.c.oW = odW;
  s.wd = wd;
  s.wn = wn;
  return 0;
}

extern "C" int genre_b200_sketch_consistency_views_forward(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_depth, int64_t odN, int64_t odV, int64_t odH, int64_t odW, const float *obs_normal, int64_t onN,
    int64_t onV, int64_t onC, int64_t onH, int64_t onW, float depth_weight, float normal_weight, float miss_cost,
    float eps, float *loss, void *stream) {
  SketchArgs s{};
  const char *what = "sketch_consistency_views";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, s.n.c)) return rc;
  if (int rc = sk_check(what, obs_depth, odN, odV, odH, odW, obs_normal, onN, onV, onC, onH, onW, depth_weight,
                        normal_weight, miss_cost, eps, s))
    return rc;
  GB_REQUIRE(loss, GENRE_B200_EINVAL, "%s: null output", what);
  GB_REQUIRE(aligned4(loss), GENRE_B200_EALIGN, "%s: loss must be 4-byte aligned", what);
  s.n.out = loss;
  sketch_consistency_forward_kernel<<<rc_grid(s.n.c), RC_THREADS, 0, as_stream(stream)>>>(s);
  return check_launch("sketch_consistency_views forward kernel");
}

extern "C" int genre_b200_sketch_consistency_views_backward(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_depth, int64_t odN, int64_t odV, int64_t odH, int64_t odW, const float *obs_normal, int64_t onN,
    int64_t onV, int64_t onC, int64_t onH, int64_t onW, float depth_weight, float normal_weight, float miss_cost,
    float eps, const float *grad_loss, float *grad_vox, void *stream) {
  SketchArgs s{};
  const char *what = "sketch_consistency_views backward";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, s.n.c)) return rc;
  if (int rc = sk_check(what, obs_depth, odN, odV, odH, odW, obs_normal, onN, onV, onC, onH, onW, depth_weight,
                        normal_weight, miss_cost, eps, s))
    return rc;
  GB_REQUIRE(grad_loss && grad_vox, GENRE_B200_EINVAL, "%s: null pointer", what);
  GB_REQUIRE(aligned4(grad_loss) && aligned4(grad_vox), GENRE_B200_EALIGN, "%s: gradients must be 4-byte aligned", what);
  s.n.c.g0 = grad_loss;
  s.n.c.grad_vox = grad_vox;
  sketch_consistency_backward_kernel<false><<<rc_grid(s.n.c), RC_THREADS, 0, as_stream(stream)>>>(s, PoseOut{});
  return check_launch("sketch_consistency_views backward kernel");
}

extern "C" int genre_b200_sketch_consistency_views_backward_pose(
    const float *vox, int64_t N, int res, int64_t V, int64_t H, int64_t W, int z_res, const float *fl, int64_t fN,
    int64_t fV, const float *rot, int64_t rN, int64_t rV, const float *eye, int64_t eN, int64_t eV,
    const float *obs_depth, int64_t odN, int64_t odV, int64_t odH, int64_t odW, const float *obs_normal, int64_t onN,
    int64_t onV, int64_t onC, int64_t onH, int64_t onW, float depth_weight, float normal_weight, float miss_cost,
    float eps, const float *grad_loss, float *grad_vox, float *grad_rot, float *grad_eye, void *workspace,
    size_t workspace_bytes, void *stream) {
  SketchArgs s{};
  PoseOut po;
  const char *what = "sketch_consistency_views backward_pose";
  if (int rc = rv_check(what, vox, N, res, V, H, W, z_res, fl, fN, fV, rot, rN, rV, eye, eN, eV, s.n.c)) return rc;
  if (int rc = sk_check(what, obs_depth, odN, odV, odH, odW, obs_normal, onN, onV, onC, onH, onW, depth_weight,
                        normal_weight, miss_cost, eps, s))
    return rc;
  GB_REQUIRE(grad_loss, GENRE_B200_EINVAL, "%s: null grad_loss", what);
  GB_REQUIRE(aligned4(grad_loss), GENRE_B200_EALIGN, "%s: grad_loss must be 4-byte aligned", what);
  if (int rc = rp_check(what, s.n.c, N, V, grad_vox, grad_rot, grad_eye, workspace, workspace_bytes, po)) return rc;
  s.n.c.g0 = grad_loss;
  s.n.c.grad_vox = grad_vox;
  const long long views = (long long)N * V;
  sketch_consistency_backward_kernel<true><<<(unsigned)(views * po.bpv), RC_THREADS, 0, as_stream(stream)>>>(s, po);
  if (int rc = check_launch("sketch_consistency_views backward_pose kernel")) return rc;
  render_views_pose_reduce_kernel<<<(unsigned)views, RC_THREADS, 0, as_stream(stream)>>>(s.n.c, po);
  return check_launch("sketch_consistency_views pose reduce kernel");
}
