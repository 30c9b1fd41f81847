// Tiled software RGB-D camera: stands in for `sim.render(width, height, camera_name, depth=True)` + `depth_2_meters`
// (reference: MujocoController.py:708-740).  Output already has the reference's U/D + L/R flip applied and depth is
// linear eye-space z in metres (SURVEY A.3).
//
// Two kernels: (1) one warp (CTA in the big-scene build) per env runs the kinematics stage and writes every geom's world frame
// ([N, ngeom, 12] f64) and its screen-space box ([N, ngeom] short4) to HBM; (2) one 16x16-pixel tile per CTA: the geoms whose box meets
// the tile go into a shared-memory list, then every thread casts its pixel's ray against the listed geoms whose box contains the pixel
// (plane / sphere / box / capsule / cylinder analytic, mesh geoms as convex polytopes = hull face planes).  Writes are coalesced:
// depth f32 rows of 16 pixels, rgb u8x3.
#pragma once
#include "ge_physics.cuh"

namespace ge {

struct RenderCtx { double* gframes; short4* gbox; double* fpx; size_t cap_envs; };

static inline void render_init(RenderCtx& r, const DevModel&, const char*) { r.gframes = nullptr; r.gbox = nullptr; r.fpx = nullptr; r.cap_envs = 0; }
static inline void render_free(RenderCtx& r) { if (r.gframes) cudaFree(r.gframes); if (r.gbox) cudaFree(r.gbox); if (r.fpx) cudaFree(r.fpx); r.gframes = nullptr; r.gbox = nullptr; r.fpx = nullptr; }

// Also writes every geom's screen-space box for camera `cam` (r02): pixel (c, r) sees direction ((W/2 - c - 1/2) / f, (H/2 - r - 1/2) / f, -1)
// in the camera frame, so a camera-frame point p lands on c = W/2 - 1/2 - f p.x / (-p.z); the box of the 8 OBB corners, one pixel of
// slack on every side, clamped to the image (x0 > x1: not visible at all; planes and geoms reaching behind the camera: whole image).
__global__ void __launch_bounds__(GE_LANES) k_render_fk(const double* qpos, int n_env, double* gframes, short4* gbox, double* fpx, int cam, int W, int H) {
  extern __shared__ double smem[];
  const DevModel& m = c_m; const Layout& L = c_L;
  int env = blockIdx.x, lane = threadIdx.x;
  if (env >= n_env) return;
  double* ws = smem;
  LANE_LOOP(i, m.nq) ws[L.qpos + i] = qpos[(size_t)env * m.nq + i];
  gsync();
  stage_fk(ws, lane);
  double* out = gframes + (size_t)env * m.ngeom * 12;
  const double *cp = m.cam_pos0 + 3 * cam, *cm = m.cam_mat0 + 9 * cam;
  const double f = 0.5 * H / tan(m.cam_fovy[cam] * 3.14159265358979323846 / 360.0);  // focal length in pixels (MujocoController.py:742-758)
  if (env == 0 && lane == 0) *fpx = f;                                                 // (k_render reads it instead of one tan per thread)
  LANE_LOOP(g, m.ngeom) {
    const double *gp = ws + L.gpos + 3 * g, *R = ws + L.gmat + 9 * g;
    for (int k = 0; k < 3; k++) out[12 * g + k] = gp[k];
    for (int k = 0; k < 9; k++) out[12 * g + 3 + k] = R[k];
    short4 bb = make_short4(0, 0, (short)(W - 1), (short)(H - 1));
    if (m.geom_type[g] != G_PLANE) {
      const double* hf = m.geom_obbhalf + 3 * g;
      double t[3], cw[3];
      m3mulv(t, R, m.geom_obbcenter + 3 * g); v3add(cw, gp, t); v3sub(t, cw, cp);  // OBB centre relative to the camera, world axes
      double xmin = 1e300, xmax = -1e300, ymin = 1e300, ymax = -1e300;
      bool front = true;
      for (int k = 0; k < 8; k++) {
        double off[3] = {(k & 1) ? hf[0] : -hf[0], (k & 2) ? hf[1] : -hf[1], (k & 4) ? hf[2] : -hf[2]}, ow[3], q[3];
        m3mulv(ow, R, off); v3add(ow, ow, t);
        m3Tmulv(q, cm, ow);
        if (-q[2] < 1e-6) { front = false; break; }
        double u = 0.5 * W - 0.5 - f * q[0] / (-q[2]), v = 0.5 * H - 0.5 - f * q[1] / (-q[2]);
        xmin = fmin(xmin, u); xmax = fmax(xmax, u); ymin = fmin(ymin, v); ymax = fmax(ymax, v);
      }
      if (front) {
        int x0 = (int)floor(fmax(xmin, -2.0)) - 1, x1 = (int)ceil(fmin(xmax, (double)W + 1)) + 1;
        int y0 = (int)floor(fmax(ymin, -2.0)) - 1, y1 = (int)ceil(fmin(ymax, (double)H + 1)) + 1;
        if (x1 < 0 || x0 > W - 1 || y1 < 0 || y0 > H - 1) bb = make_short4(1, 1, 0, 0);
        else bb = make_short4((short)max(x0, 0), (short)max(y0, 0), (short)min(x1, W - 1), (short)min(y1, H - 1));
      }
    }
    gbox[(size_t)env * m.ngeom + g] = bb;
  }
}

__device__ __forceinline__ double ray_geom(int g, const double* fr, const double* o, const double* dir, double* nrm) {
  const DevModel& m = c_m;
  const double *gp = fr, *R = fr + 3, *size = m.geom_size + 3 * g;
  double ol[3], dl[3], t[3];
  v3sub(t, o, gp); m3Tmulv(ol, R, t); m3Tmulv(dl, R, dir);
  int type = m.geom_type[g];
  double tn = -1e300, tf = 1e300, nl[3] = {0, 0, 1};
  if (type == G_PLANE) {
    if (dl[2] >= -1e-12) return -1;
    double tt = -ol[2] / dl[2];
    if (tt <= 0) return -1;
    m3col(nrm, R, 2);
    return tt;
  } else if (type == G_SPHERE) {
    double b = v3dot(ol, dl), c = v3dot(ol, ol) - size[0] * size[0], a = v3dot(dl, dl);
    double disc = b * b - a * c;
    if (disc < 0) return -1;
    double tt = (-b - sqrt(disc)) / a;
    if (tt <= 0) return -1;
    v3addscl(nl, ol, dl, tt); v3normalize(nl);
    m3mulv(nrm, R, nl);
    return tt;
  } else if (type == G_BOX) {
    for (int k = 0; k < 3; k++) {
      if (fabs(dl[k]) < 1e-14) { if (fabs(ol[k]) > size[k]) return -1; continue; }
      double t1 = (-size[k] - ol[k]) / dl[k], t2 = (size[k] - ol[k]) / dl[k], s = -1;
      if (t1 > t2) { double x = t1; t1 = t2; t2 = x; s = 1; }
      if (t1 > tn) { tn = t1; v3set(nl, 0, 0, 0); if (k == 0) nl[0] = s; else if (k == 1) nl[1] = s; else nl[2] = s; }
      if (t2 < tf) tf = t2;
    }
    if (tn > tf || tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  } else if (type == G_MESH) {
    int k = m.geom_meshid[g];
    double oc[3];
    v3sub(oc, ol, m.geom_obbcenter + 3 * g);
    double b = v3dot(oc, dl), c = v3dot(oc, oc) - m.geom_rbound[g] * m.geom_rbound[g], a = v3dot(dl, dl);
    if (b * b - a * c < 0) return -1;
    const double* pl = m.mesh_faceplane + 4 * m.mesh_faceadr[k];
    int nf = m.mesh_facenum[k];
    for (int f = 0; f < nf; f++, pl += 4) {
      double p0 = __ldg(pl), p1 = __ldg(pl + 1), p2 = __ldg(pl + 2), p3 = __ldg(pl + 3);
      double dn = p0 * dl[0] + p1 * dl[1] + p2 * dl[2], on = p0 * ol[0] + p1 * ol[1] + p2 * ol[2] - p3;
      if (fabs(dn) < 1e-14) { if (on > 0) return -1; continue; }
      double tt = -on / dn;
      if (dn < 0) { if (tt > tn) { tn = tt; nl[0] = p0; nl[1] = p1; nl[2] = p2; } }
      else if (tt < tf) tf = tt;
      if (tn > tf) return -1;
    }
    if (tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  } else if (type == G_CYLINDER) {  // infinite cylinder and the slab |z| <= h, intersected like the box slabs
    double r = size[0], h = size[1];
    double a = dl[0] * dl[0] + dl[1] * dl[1], b = ol[0] * dl[0] + ol[1] * dl[1], c = ol[0] * ol[0] + ol[1] * ol[1] - r * r;
    if (a < 1e-14) { if (c > 0) return -1; }
    else {
      double disc = b * b - a * c;
      if (disc < 0) return -1;
      double sq = sqrt(disc);
      tn = (-b - sq) / a; tf = (-b + sq) / a;
      v3set(nl, (ol[0] + tn * dl[0]) / r, (ol[1] + tn * dl[1]) / r, 0);
    }
    if (fabs(dl[2]) < 1e-14) { if (fabs(ol[2]) > h) return -1; }
    else {
      double t1 = (-h - ol[2]) / dl[2], t2 = (h - ol[2]) / dl[2], s = -1;
      if (t1 > t2) { double x = t1; t1 = t2; t2 = x; s = 1; }
      if (t1 > tn) { tn = t1; v3set(nl, 0, 0, s); }
      if (t2 < tf) tf = t2;
    }
    if (tn > tf || tn <= 0) return -1;
    m3mulv(nrm, R, nl);
    return tn;
  } else if (type == G_CAPSULE) {  // side wall where |z| <= h, otherwise the outward half of either end sphere
    double r = size[0], h = size[1], best = -1;
    double a = dl[0] * dl[0] + dl[1] * dl[1], b = ol[0] * dl[0] + ol[1] * dl[1], c = ol[0] * ol[0] + ol[1] * ol[1] - r * r;
    if (a >= 1e-14) {
      double disc = b * b - a * c;
      if (disc >= 0) {
        double t1 = (-b - sqrt(disc)) / a, z = ol[2] + t1 * dl[2];
        if (t1 > 0 && fabs(z) <= h) { best = t1; v3set(nl, (ol[0] + t1 * dl[0]) / r, (ol[1] + t1 * dl[1]) / r, 0); }
      }
    }
    for (int s = 0; s < 2; s++) {
      double sg = s ? -1.0 : 1.0, oc[3] = {ol[0], ol[1], ol[2] - sg * h};
      double bb = v3dot(oc, dl), cc = v3dot(oc, oc) - r * r, aa = v3dot(dl, dl), disc = bb * bb - aa * cc;
      if (disc < 0) continue;
      double t1 = (-bb - sqrt(disc)) / aa;
      if (t1 <= 0 || sg * (oc[2] + t1 * dl[2]) < 0) continue;
      if (best < 0 || t1 < best) { best = t1; v3addscl(nl, oc, dl, t1); v3scl(nl, nl, 1.0 / r); }
    }
    if (best <= 0) return -1;
    m3mulv(nrm, R, nl);
    return best;
  }
  return -1;
}

#define RTILE 16
#define RTILE_LIST 256  // geoms a tile can list (ge_create rejects scenes with more)
__global__ void __launch_bounds__(RTILE * RTILE) k_render(const double* gframes, const short4* gbox, const double* fpx, int n_env, int cam, int W, int H, unsigned char* rgb,
                                                          float* depth) {
  const DevModel& m = c_m;
  __shared__ int s_list[RTILE_LIST];
  __shared__ short4 s_bb[RTILE_LIST];  // screen-space box (pixel columns x..z, rows y..w) of the listed geom
  __shared__ int s_n;
  int env = blockIdx.y, tiles_x = (W + RTILE - 1) / RTILE;
  int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
  int tid = threadIdx.y * RTILE + threadIdx.x;
  const double* fr = gframes + (size_t)env * m.ngeom * 12;
  const double *cp = m.cam_pos0 + 3 * cam, *cm = m.cam_mat0 + 9 * cam;
  if (tid == 0) s_n = 0;
  __syncthreads();
  // The tile lists the geoms whose screen box (k_render_fk) meets its pixel range, and keeps the box so that each pixel also skips the
  // geoms whose box it lies outside of.  The boxes only drop geoms no ray of the tile / pixel can hit: the image is the same as with
  // the full list.  A bounding-cone test against bounding spheres alone lets the table top, legs and bin walls
  // (spheres of 0.35-0.5 m) through for every tile.  The boxes are computed once per env: computed here, per tile, most threads would
  // wait at this barrier.
  {
    const int c0i = tx * RTILE, c1i = min(W, c0i + RTILE), r0i = ty * RTILE, r1i = min(H, r0i + RTILE);
    const short4* gb = gbox + (size_t)env * m.ngeom;
    for (int g = tid; g < m.ngeom; g += RTILE * RTILE) {
      const short4 bb = gb[g];
      if (bb.z < c0i || bb.x > c1i - 1 || bb.w < r0i || bb.y > r1i - 1) continue;
      int k = atomicAdd(&s_n, 1);
      if (k < RTILE_LIST) { s_list[k] = g; s_bb[k] = bb; }
    }
  }
  __syncthreads();
  const double f = *fpx;
  int c = tx * RTILE + threadIdx.x, r = ty * RTILE + threadIdx.y;
  if (c >= W || r >= H) return;
  int n = s_n < RTILE_LIST ? s_n : RTILE_LIST;
  double dc[3] = {(0.5 * W - c - 0.5) / f, (0.5 * H - r - 0.5) / f, -1.0}, dir[3];
  m3mulv(dir, cm, dc);
  double best = 1e300, bn[3] = {0, 0, 1};
  int bg = -1;
  for (int k = 0; k < n; k++) {
    const short4 bb = s_bb[k];
    if (c < bb.x || c > bb.z || r < bb.y || r > bb.w) continue;
    int g = s_list[k];
    double nr[3];
    double t = ray_geom(g, fr + 12 * g, cp, dir, nr);
    if (t > 0 && (t < best || (t == best && g < bg))) { best = t; bg = g; v3copy(bn, nr); }
  }
  size_t px = ((size_t)env * H + r) * W + c;
  if (bg < 0) { depth[px] = (float)(m.zfar * m.extent); rgb[3 * px] = rgb[3 * px + 1] = rgb[3 * px + 2] = 0; return; }
  depth[px] = (float)best;
  double light[3] = {-1, 1, -2.565};
  v3normalize(light);
  double lam = -v3dot(bn, light);
  if (lam < 0) lam = 0;
  double shade = 0.4 + 0.6 * lam;
  const double* col = m.geom_rgba + 4 * bg;
  double base[3] = {col[0], col[1], col[2]};
  if (m.geom_type[bg] == G_PLANE) {
    double hit[3];
    v3addscl(hit, cp, dir, best);
    int cx = (int)floor(hit[0] / 0.25), cy = (int)floor(hit[1] / 0.25);
    if ((cx + cy) & 1) { base[0] = 0.1; base[1] = 0.2; base[2] = 0.3; } else { base[0] = 0.2; base[1] = 0.3; base[2] = 0.4; }
  }
  for (int k = 0; k < 3; k++) { double v = base[k] * shade * 255.0 + 0.5; rgb[3 * px + k] = (unsigned char)(v > 255 ? 255 : v); }
}

static inline int render_launch(RenderCtx& rc, const DevModel& m, const Layout& L, const double* qpos, int n_env, int cam, int W, int H,
                                unsigned char* rgb, float* depth, cudaStream_t stream, int64_t* launches) {
  if (rc.cap_envs < (size_t)n_env) {
    if (rc.gframes) cudaFree(rc.gframes);
    if (rc.gbox) cudaFree(rc.gbox);
    rc.gframes = nullptr; rc.gbox = nullptr;
    if (cudaMalloc(&rc.gframes, sizeof(double) * 12 * m.ngeom * (size_t)n_env) != cudaSuccess) return -1;
    if (cudaMalloc(&rc.gbox, sizeof(short4) * m.ngeom * (size_t)n_env) != cudaSuccess) return -1;
    if (!rc.fpx && cudaMalloc(&rc.fpx, sizeof(double)) != cudaSuccess) return -1;
    rc.cap_envs = n_env;
  }
  k_render_fk<<<n_env, GE_LANES, L.fk_bytes, stream>>>(qpos, n_env, rc.gframes, rc.gbox, rc.fpx, cam, W, H);
  int tiles = ((W + RTILE - 1) / RTILE) * ((H + RTILE - 1) / RTILE);
  dim3 grid(tiles, n_env), blk(RTILE, RTILE);
  k_render<<<grid, blk, 0, stream>>>(rc.gframes, rc.gbox, rc.fpx, n_env, cam, W, H, rgb, depth);
  *launches += 2;
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace ge
