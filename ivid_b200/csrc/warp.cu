// RGBD novel-view warp on the device: mesh construction, visibility-buffer rasterisation, per-view shading +
// cross-view aggregation, SSAA resolve and condition-map post-filters.  Replaces the CPU numpy mesh build, the OpenGL
// rasteriser / GLSL shaders and the CPU PIL/cv2 post-filters of the reference (per view, per sample round trips
// GPU->CPU->GL->CPU->GPU: SURVEY.md §1) with kernels that keep the RGBD views resident in HBM.
//   reference: rgbd_3d/utils.py:38-58,89-134,137-141,144-274   linearize_depth, unproject, triangulate, depth_to_mesh
//              rgbd_3d/moderngl_renderer.py:260-340 + shaders/aggregation.{vsh,fsh,csh}, clear.csh   render + aggregate
//              rgbd_3d/utils.py:61-67,311-332,420-477           project_depth, depth_edge, aggregate_conditions
// Rasterisation follows the rules fixed in oracle/raster_ref.c (fp32 vertex stage, 1/256-pixel snapping, exact 64-bit
// edge functions, strict '<' depth).  Instead of GL's sequential depth test, every fragment does a 64-bit atomicMin of
// (depth bits << 32 | primitive id) into a per-(sample, source view) visibility buffer: equal depth resolves to the
// lower primitive id == the first triangle drawn, i.e. exactly the sequential '<' result, with coalesced 8-byte
// traffic.  Shading happens once per pixel in the resolve kernel (deferred), fused with the aggregation.csh rule.
// This translation unit is compiled with -fmad=false so fp32 arithmetic rounds like the CPU oracle.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "../../include/ivid_b200.h"
#include "host_util.h"

namespace ivid {

// ----------------------------------------------------------------------------------------------------------------------
// shared device helpers
// ----------------------------------------------------------------------------------------------------------------------
struct WVtx {
  float clip[4];
  float pos[3];
  float nrm[3];
  float uv[2];
  float edge, pad, ero;
};
constexpr int kVtxFloats = sizeof(WVtx) / sizeof(float);

__device__ __forceinline__ void wv_lerp(const WVtx& a, const WVtx& b, float t, WVtx& o) {
  const float* pa = reinterpret_cast<const float*>(&a);
  const float* pb = reinterpret_cast<const float*>(&b);
  float* po = reinterpret_cast<float*>(&o);
#pragma unroll
  for (int i = 0; i < kVtxFloats; ++i) po[i] = pa[i] + (pb[i] - pa[i]) * t;
}

__device__ __forceinline__ void load_vertex(const float* __restrict__ verts, uint32_t vi, const float* __restrict__ mvp, WVtx& v) {
  const float* a = verts + static_cast<size_t>(vi) * 9;
#pragma unroll
  for (int r = 0; r < 4; ++r) v.clip[r] = ((mvp[r * 4 + 0] * a[0] + mvp[r * 4 + 1] * a[1]) + mvp[r * 4 + 2] * a[2]) + mvp[r * 4 + 3];
  v.pos[0] = a[0]; v.pos[1] = a[1]; v.pos[2] = a[2];
  const float nl = sqrtf((a[3] * a[3] + a[4] * a[4]) + a[5] * a[5]);
  v.nrm[0] = a[3] / nl; v.nrm[1] = a[4] / nl; v.nrm[2] = a[5] / nl;
  v.uv[0] = a[6]; v.uv[1] = a[7];
  const int flag = static_cast<int>(a[8]);
  v.edge = static_cast<float>(flag & 1); v.pad = static_cast<float>((flag >> 1) & 1); v.ero = static_cast<float>((flag >> 2) & 1);
}

// clip against z + w >= 0; returns 0, 3 or 4 polygon vertices
__device__ __forceinline__ int clip_near(const WVtx (&in)[3], WVtx (&out)[4]) {
  float d[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) d[i] = in[i].clip[2] + in[i].clip[3];
  if (d[0] >= 0.f && d[1] >= 0.f && d[2] >= 0.f) { out[0] = in[0]; out[1] = in[1]; out[2] = in[2]; return 3; }
  if (d[0] < 0.f && d[1] < 0.f && d[2] < 0.f) return 0;
  int n = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int j = (i + 1) % 3;
    if (d[i] >= 0.f) out[n++] = in[i];
    if ((d[i] >= 0.f) != (d[j] >= 0.f)) {
      const float t = d[i] / (d[i] - d[j]);
      wv_lerp(in[i], in[j], t, out[n++]);
    }
  }
  return n;
}

struct TriSetup {
  long long X[3], Y[3];
  float zw[3], iw[3];
  long long area;
};

__device__ __forceinline__ void tri_setup(const WVtx* v, int S, TriSetup& t) {
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float w = v[i].clip[3];
    const float xn = v[i].clip[0] / w, yn = v[i].clip[1] / w, zn = v[i].clip[2] / w;
    const float xw = (xn * 0.5f + 0.5f) * static_cast<float>(S), yw = (yn * 0.5f + 0.5f) * static_cast<float>(S);
    t.X[i] = static_cast<long long>(floorf(xw * 256.f + 0.5f));
    t.Y[i] = static_cast<long long>(floorf(yw * 256.f + 0.5f));
    t.zw[i] = zn * 0.5f + 0.5f;
    t.iw[i] = 1.0f / w;
  }
  t.area = (t.X[1] - t.X[0]) * (t.Y[2] - t.Y[0]) - (t.Y[1] - t.Y[0]) * (t.X[2] - t.X[0]);
}

// coverage + barycentrics of pixel (px,py); returns false if the pixel centre is outside
__device__ __forceinline__ bool tri_eval(const TriSetup& t, long long px, long long py, float& l0, float& l1, float& l2) {
  const long long sgn = t.area > 0 ? 1 : -1;
  const long long cx = px * 256 + 128, cy = py * 256 + 128;
  long long E[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int a = (i + 1) % 3, b = (i + 2) % 3;
    const long long dx = (t.X[b] - t.X[a]) * sgn, dy = (t.Y[b] - t.Y[a]) * sgn;
    const long long e = ((t.X[b] - t.X[a]) * (cy - t.Y[a]) - (t.Y[b] - t.Y[a]) * (cx - t.X[a])) * sgn;
    const bool tie_ok = (dy > 0) || (dy == 0 && dx < 0);
    if (e < 0 || (e == 0 && !tie_ok)) return false;
    E[i] = e;
  }
  const float farea = static_cast<float>(sgn * t.area);
  l0 = static_cast<float>(E[0]) / farea;
  l1 = static_cast<float>(E[1]) / farea;
  l2 = static_cast<float>(E[2]) / farea;
  return true;
}

struct ViewRef {            // one source view of one sample
  const float* verts;       // [V][9]
  const uint32_t* faces;    // [F][3]
  const float* tex;         // [T][T][3]
  float cam[3];             // source camera position (world)
};

// ----------------------------------------------------------------------------------------------------------------------
// rasterise: one thread per triangle, 64-bit atomicMin visibility buffer
// ----------------------------------------------------------------------------------------------------------------------
struct RasterParams {
  const ViewRef* views;       // [B][nviews]
  const float* mvp;           // [B][16] row-major P*MV of the target view
  unsigned long long* vis;    // [B][nviews][S*S]
  int nviews, F, S;
  int simple;                 // 1: SimpleRenderer (simple.fsh): no back-face padding discard
};

// One set-up sub-triangle, flattened to 32-bit words so a lane can broadcast it to its warp with shuffles.
// The three edge functions are kept in coefficient form  E_i(cx, cy) = ea_i*cx + eb_i*cy + ec_i  (exact 64-bit integers, the
// expansion of tri_eval's ((Xb-Xa)*(cy-Ya) - (Yb-Ya)*(cx-Xa))*sgn), so a pixel costs two multiplies per edge.
struct RTri {
  long long ea[3], eb[3], ec[3];
  float zw[3], iw[3], pad[3];
  float farea;                 // |area| as float (barycentric denominator)
  int front;                   // area > 0
  int tie;                     // bit i: an E_i == 0 pixel centre belongs to the triangle (top-left style rule)
  int px0, px1, py0, py1;
  uint32_t prim;
  int valid;
};
constexpr int kRTriWords = sizeof(RTri) / 4;

__device__ __forceinline__ void rtri_make(const WVtx* v, int S, uint32_t prim, RTri& r) {
  TriSetup t;
  tri_setup(v, S, t);
  r.valid = 0;
  if (t.area == 0) return;
  const long long sgn = t.area > 0 ? 1 : -1;
  r.tie = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int a = (i + 1) % 3, c = (i + 2) % 3;
    const long long dx = (t.X[c] - t.X[a]) * sgn, dy = (t.Y[c] - t.Y[a]) * sgn;
    r.ea[i] = -dy;
    r.eb[i] = dx;
    r.ec[i] = -(r.ea[i] * t.X[a] + r.eb[i] * t.Y[a]);
    if ((dy > 0) || (dy == 0 && dx < 0)) r.tie |= 1 << i;
    r.zw[i] = t.zw[i]; r.iw[i] = t.iw[i]; r.pad[i] = v[i].pad;
  }
  r.farea = static_cast<float>(sgn * t.area);
  r.front = t.area > 0 ? 1 : 0;
  r.prim = prim;
  const long long minx = min(t.X[0], min(t.X[1], t.X[2])), maxx = max(t.X[0], max(t.X[1], t.X[2]));
  const long long miny = min(t.Y[0], min(t.Y[1], t.Y[2])), maxy = max(t.Y[0], max(t.Y[1], t.Y[2]));
  if (maxx < 128 || maxy < 128) return;
  long long px0 = minx <= 128 ? 0 : (minx - 128 + 255) / 256, px1 = (maxx - 128) / 256;
  long long py0 = miny <= 128 ? 0 : (miny - 128 + 255) / 256, py1 = (maxy - 128) / 256;
  if (px1 > S - 1) px1 = S - 1;
  if (py1 > S - 1) py1 = S - 1;
  if (px0 > px1 || py0 > py1) return;
  r.px0 = static_cast<int>(px0); r.px1 = static_cast<int>(px1); r.py0 = static_cast<int>(py0); r.py1 = static_cast<int>(py1);
  r.valid = 1;
}

// a covered pixel: depth, (aggregation mode) back-face padding discard, visibility key.  fE = the three edge values as floats
__device__ __forceinline__ void rtri_cover(const RTri& r, float fE0, float fE1, float fE2, int px, int py, int S, unsigned long long* vis, int simple) {
  const float l0 = fE0 / r.farea, l1 = fE1 / r.farea, l2 = fE2 / r.farea;
  const float z = (l0 * r.zw[0] + l1 * r.zw[1]) + l2 * r.zw[2];
  if (!(z > 0.f && z < 1.f)) return;
  if (!simple && !r.front) {
    const float b0 = l0 * r.iw[0], b1 = l1 * r.iw[1], b2 = l2 * r.iw[2];
    const float bs = (b0 + b1) + b2;
    const float pad = ((b0 / bs) * r.pad[0] + (b1 / bs) * r.pad[1]) + (b2 / bs) * r.pad[2];
    if (pad > 0.001f) return;      // back-facing frustum padding is discarded (aggregation.fsh:23)
  }
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(z)) << 32) | r.prim;
  atomicMin(vis + static_cast<size_t>(py) * S + px, key);
}

__device__ __forceinline__ void rtri_pixel(const RTri& r, int px, int py, int S, unsigned long long* vis, int simple) {
  const long long cx = static_cast<long long>(px) * 256 + 128, cy = static_cast<long long>(py) * 256 + 128;
  long long E[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const long long e = r.ea[i] * cx + r.eb[i] * cy + r.ec[i];
    if (e < 0 || (e == 0 && !((r.tie >> i) & 1))) return;
    E[i] = e;
  }
  rtri_cover(r, static_cast<float>(E[0]), static_cast<float>(E[1]), static_cast<float>(E[2]), px, py, S, vis, simple);
}

// Small bounding boxes (<= 48 pixels) of triangles whose edge coefficients fit 15 bits: the same exact integer edge functions,
// evaluated once at the first pixel centre in 64 bits and then stepped in 32 bits (|E| < 2^31 inside the box: (|ea| + |eb|) <
// 2^16 times at most 49 * 256 sub-pixels), one add per edge and pixel instead of two 64-bit multiply-adds.  float(int32 E) ==
// float(int64 E) for the same integer, so the covered pixels get bit-identical barycentrics.
__device__ __forceinline__ void rtri_scan_small32(const RTri& r, int S, unsigned long long* vis, int simple) {
  const long long cx0 = static_cast<long long>(r.px0) * 256 + 128, cy0 = static_cast<long long>(r.py0) * 256 + 128;
  int erow[3], sx[3], sy[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    erow[i] = static_cast<int>(r.ea[i] * cx0 + r.eb[i] * cy0 + r.ec[i]);
    sx[i] = static_cast<int>(r.ea[i]) * 256;
    sy[i] = static_cast<int>(r.eb[i]) * 256;
  }
  for (int py = r.py0; py <= r.py1; ++py) {
    int e0 = erow[0], e1 = erow[1], e2 = erow[2];
    for (int px = r.px0; px <= r.px1; ++px) {
      const bool in0 = e0 > 0 || (e0 == 0 && (r.tie & 1)), in1 = e1 > 0 || (e1 == 0 && (r.tie & 2)), in2 = e2 > 0 || (e2 == 0 && (r.tie & 4));
      if (in0 && in1 && in2) rtri_cover(r, static_cast<float>(e0), static_cast<float>(e1), static_cast<float>(e2), px, py, S, vis, simple);
      e0 += sx[0]; e1 += sx[1]; e2 += sx[2];
    }
    erow[0] += sy[0]; erow[1] += sy[1]; erow[2] += sy[2];
  }
}

// Small triangles (the common 3x3-pixel case) are scanned by their own lane; triangles with a large bounding box (the
// frustum ring and faces stretched across depth discontinuities) are broadcast to the warp and scanned by all 32 lanes.
// `stash` = this warp's 32 rows of a shared-memory table: a lane parks its big triangle there and the warp reads the leader's row
// (a broadcast load) instead of keeping two set-up triangles in registers and shuffling 36 words per triangle.
__device__ __forceinline__ void rtri_raster(RTri& r, int S, unsigned long long* vis, int lane, int simple, uint32_t (*stash)[kRTriWords]) {
  constexpr int kSmall = 48;
  const int w = r.valid ? (r.px1 - r.px0 + 1) : 0, h = r.valid ? (r.py1 - r.py0 + 1) : 0;
  const bool big = r.valid && (w * h > kSmall);
  if (r.valid && !big) {
    bool fit = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) fit = fit && r.ea[i] > -32768 && r.ea[i] < 32768 && r.eb[i] > -32768 && r.eb[i] < 32768;
    // the first-pixel edge values must also fit 31 bits (they do whenever the box lies within ~2^15 sub-pixels of the triangle,
    // i.e. always for on-screen boxes of such triangles; checked, not assumed)
    const long long cx0 = static_cast<long long>(r.px0) * 256 + 128, cy0 = static_cast<long long>(r.py0) * 256 + 128;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const long long e = r.ea[i] * cx0 + r.eb[i] * cy0 + r.ec[i];
      fit = fit && e > -(1ll << 29) && e < (1ll << 29);
    }
    if (fit) {
      rtri_scan_small32(r, S, vis, simple);
    } else {
      for (int py = r.py0; py <= r.py1; ++py)
        for (int px = r.px0; px <= r.px1; ++px) rtri_pixel(r, px, py, S, vis, simple);
    }
  }
  unsigned mask = __ballot_sync(0xffffffffu, big);
  if (mask == 0u) return;
  if (big) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
    for (int i = 0; i < kRTriWords; ++i) stash[lane][i] = src[i];
  }
  __syncwarp();
  while (mask) {
    const int leader = __ffs(mask) - 1;
    mask &= mask - 1;
    // the leader's record is read in place (warp-uniform addresses: broadcast loads), which keeps the kernel at 96 registers
    // (5 blocks per SM) instead of 122 with a register copy
    const RTri& b = *reinterpret_cast<const RTri*>(stash[leader]);
    // 8x8-pixel tiles of the bounding box; a tile is skipped when one edge function is negative at its most-inside corner
    // (exact integer test, so the surviving pixels are decided by the same arithmetic as the small path).  The tiles are
    // TESTED 32 at a time (one tile per lane: the frustum-ring slivers have bounding boxes of thousands of tiles of which a
    // few dozen survive); the survivors are then scanned by the whole warp, 2 pixels per lane.
    const int tx0 = b.px0 >> 3, tx1 = b.px1 >> 3, ty0 = b.py0 >> 3, ty1 = b.py1 >> 3;
    const int ntx = tx1 - tx0 + 1, nt = ntx * (ty1 - ty0 + 1);
    for (int base = 0; base < nt; base += 32) {
      const int ti = base + lane;
      int tx = 0, ty = 0;
      bool keep = false;
      if (ti < nt) {
        ty = ty0 + ti / ntx; tx = tx0 + ti % ntx;
        const int x0 = max(tx * 8, b.px0), x1 = min(tx * 8 + 7, b.px1), y0 = max(ty * 8, b.py0), y1 = min(ty * 8 + 7, b.py1);
        const long long cx0 = static_cast<long long>(x0) * 256 + 128, cx1 = static_cast<long long>(x1) * 256 + 128;
        const long long cy0 = static_cast<long long>(y0) * 256 + 128, cy1 = static_cast<long long>(y1) * 256 + 128;
        bool out = false;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const long long emax = b.ea[i] * (b.ea[i] > 0 ? cx1 : cx0) + b.eb[i] * (b.eb[i] > 0 ? cy1 : cy0) + b.ec[i];
          out = out || (emax < 0);
        }
        keep = !out;
      }
      unsigned km = __ballot_sync(0xffffffffu, keep);
      while (km) {
        const int sl = __ffs(km) - 1;
        km &= km - 1;
        const int stx = __shfl_sync(0xffffffffu, tx, sl), sty = __shfl_sync(0xffffffffu, ty, sl);
        const int x0 = max(stx * 8, b.px0), x1 = min(stx * 8 + 7, b.px1), y0 = max(sty * 8, b.py0), y1 = min(sty * 8 + 7, b.py1);
        // a lane owns pixel (lane & 7, lane >> 3) of the tile and the one four rows below: the edge values of the first are
        // evaluated (three 64-bit multiply-adds), those of the second follow by adding 4 * 256 * eb (same exact integers)
        {
          const int px = stx * 8 + (lane & 7), py = sty * 8 + (lane >> 3);
          const long long cx = static_cast<long long>(px) * 256 + 128, cy = static_cast<long long>(py) * 256 + 128;
          long long E[3];
#pragma unroll
          for (int i = 0; i < 3; ++i) E[i] = b.ea[i] * cx + b.eb[i] * cy + b.ec[i];
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            const int qy = py + 4 * half;
            bool in = px >= x0 && px <= x1 && qy >= y0 && qy <= y1;
#pragma unroll
            for (int i = 0; i < 3; ++i) in = in && (E[i] > 0 || (E[i] == 0 && ((b.tie >> i) & 1)));
            if (in) rtri_cover(b, static_cast<float>(E[0]), static_cast<float>(E[1]), static_cast<float>(E[2]), px, qy, S, vis, simple);
#pragma unroll
            for (int i = 0; i < 3; ++i) E[i] += b.eb[i] * 1024;
          }
        }
      }
    }
  }
  __syncwarp();      // the stash rows are reused by the next sub-triangle of this warp
}

__global__ void __launch_bounds__(128, 5) raster_kernel(const RasterParams p) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  const int view = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x & 31;
  __shared__ __align__(16) uint32_t s_stash[128][kRTriWords];
  __shared__ __align__(16) uint32_t s_second[128][kRTriWords];      // the rare second sub-triangle of a near-clipped face waits here
  uint32_t (*stash)[kRTriWords] = s_stash + (threadIdx.x & ~31);
  unsigned long long* vis = p.vis + (static_cast<size_t>(b) * p.nviews + view) * p.S * p.S;
  RTri t;
  t.valid = 0;
  bool second = false;
  if (f < p.F) {
    // faces are visited in a permuted order (7919 is coprime to the face count of any (n+1)^2*2 grid used here) so that
    // the runs of large triangles (frustum ring rows) spread over all warps; primitive ids stay the face indices
    const int fi = static_cast<int>((static_cast<long long>(f) * 7919) % p.F);
    const ViewRef vr = p.views[b * p.nviews + view];
    const float* mvp = p.mvp + b * 16;
    WVtx in[3], poly[4];
#pragma unroll
    for (int k = 0; k < 3; ++k) load_vertex(vr.verts, vr.faces[fi * 3 + k], mvp, in[k]);
    const int n = clip_near(in, poly);
    if (n == 4) {
      WVtx q[3] = {poly[0], poly[2], poly[3]};
      rtri_make(q, p.S, static_cast<uint32_t>(fi) * 2u + 1u, t);
      if (t.valid) {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&t);
#pragma unroll
        for (int i = 0; i < kRTriWords; ++i) s_second[threadIdx.x][i] = src[i];
        second = true;
        t.valid = 0;
      }
    }
    if (n >= 3) rtri_make(poly, p.S, static_cast<uint32_t>(fi) * 2u, t);
  }
  rtri_raster(t, p.S, vis, lane, p.simple, stash);
  if (__any_sync(0xffffffffu, second)) {      // atomicMin commutes: the order of the two sub-triangles is irrelevant
    t.valid = 0;
    if (second) {
      uint32_t* dst = reinterpret_cast<uint32_t*>(&t);
#pragma unroll
      for (int i = 0; i < kRTriWords; ++i) dst[i] = s_second[threadIdx.x][i];
    }
    rtri_raster(t, p.S, vis, lane, p.simple, stash);
  }
}

// ----------------------------------------------------------------------------------------------------------------------
// deferred shading + aggregation.csh across source views (in draw order) + read-back resolve (flip, divide, linearise)
// ----------------------------------------------------------------------------------------------------------------------
struct ResolveParams {
  const ViewRef* views;
  const float* mvp;
  const unsigned long long* vis;
  int nviews, S, T;
  float nf_f, far_f, fn_f;    // near*far, far, far-near of the renderer planes (python floats cast like numpy does)
  float* color;               // [B][S][S][3]   (image row 0 = top)
  float* depth;               // [B][S][S]
  float* mask_color;          // [B][S][S]  0/1
  float* mask_depth;          // [B][S][S]
  float4* frag_c;             // [B][nviews][S*S] shaded fragment colour + weight of every source view (shade_kernel)
  float* frag_d;              // [B][nviews][S*S] its window depth (1 where nothing was drawn)
};

__device__ __forceinline__ float shade_weight(const float* pos, const float* nrm, const float* cam, float edge, float pad, float ero) {
  const float dir[3] = {cam[0] - pos[0], cam[1] - pos[1], cam[2] - pos[2]};
  const float dl = sqrtf(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
  const float nl = sqrtf(nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2]);
  const float dt = (dir[0] * nrm[0] + dir[1] * nrm[1] + dir[2] * nrm[2]) / (dl * nl);
  float w = dt < 0.f ? 0.f : (dt > 1.f ? 1.f : dt);
  w = acosf(w);
  w = fmaxf(-w * 20.f, -50.f);
  w = expf(w);
  w = fmaxf(w, 1e-4f);
  if (!(ero < 0.999f)) w *= 1e-8f;
  if (pad > 0.001f || edge > 0.999f) w = 1e-16f;
  return fmaxf(w, 1e-16f);
}

// Pass 1 (one thread per (pixel, source view, sample): every covered fragment is shaded independently, so the dependent
// gathers key -> face -> vertices -> texel of different views overlap instead of running one after the other per pixel):
// fragment colour / weight and window depth exactly as aggregation.fsh produces them.
__global__ void __launch_bounds__(128) shade_kernel(const ResolveParams p) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int i = blockIdx.y, b = blockIdx.z;
  if (pix >= p.S * p.S) return;
  const int px = pix % p.S, py = pix / p.S;       // framebuffer coordinates (row 0 = bottom)
  const float* mvp = p.mvp + b * 16;
  const size_t slot = (static_cast<size_t>(b) * p.nviews + i) * p.S * p.S + pix;
  const unsigned long long key = p.vis[slot];
  float c[4] = {0.f, 0.f, 0.f, 0.f};
  float depth = 1.0f;
  if (key != ~0ull) {
    depth = __uint_as_float(static_cast<uint32_t>(key >> 32));
    const uint32_t prim = static_cast<uint32_t>(key & 0xFFFFFFFFull);
    const uint32_t f = prim >> 1, sub = prim & 1u;
    const ViewRef vr = p.views[b * p.nviews + i];
    WVtx in[3], poly[4];
#pragma unroll
    for (int k = 0; k < 3; ++k) load_vertex(vr.verts, vr.faces[f * 3 + k], mvp, in[k]);
    clip_near(in, poly);
    WVtx tv[3];
    tv[0] = poly[0];
    tv[1] = sub ? poly[2] : poly[1];
    tv[2] = sub ? poly[3] : poly[2];
    TriSetup t;
    tri_setup(tv, p.S, t);
    float l0, l1, l2;
    if (t.area > 0 && tri_eval(t, px, py, l0, l1, l2)) {     // front face: shade; back face keeps (0,0,0,0)
      const float b0 = l0 * t.iw[0], b1 = l1 * t.iw[1], b2 = l2 * t.iw[2];
      const float bs = (b0 + b1) + b2;
      const float c0 = b0 / bs, c1 = b1 / bs, c2 = b2 / bs;
      float pos[3], nrm[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        pos[k] = (c0 * tv[0].pos[k] + c1 * tv[1].pos[k]) + c2 * tv[2].pos[k];
        nrm[k] = (c0 * tv[0].nrm[k] + c1 * tv[1].nrm[k]) + c2 * tv[2].nrm[k];
      }
      const float uu = (c0 * tv[0].uv[0] + c1 * tv[1].uv[0]) + c2 * tv[2].uv[0];
      const float vv = (c0 * tv[0].uv[1] + c1 * tv[1].uv[1]) + c2 * tv[2].uv[1];
      const float edge = (c0 * tv[0].edge + c1 * tv[1].edge) + c2 * tv[2].edge;
      const float pad = (c0 * tv[0].pad + c1 * tv[1].pad) + c2 * tv[2].pad;
      const float ero = (c0 * tv[0].ero + c1 * tv[1].ero) + c2 * tv[2].ero;
      int tx = static_cast<int>(floorf(uu * static_cast<float>(p.T))), ty = static_cast<int>(floorf(vv * static_cast<float>(p.T)));
      tx = min(max(tx, 0), p.T - 1); ty = min(max(ty, 0), p.T - 1);
      const float* tc = vr.tex + (static_cast<size_t>(ty) * p.T + tx) * 3;
      c[0] = tc[0]; c[1] = tc[1]; c[2] = tc[2];
      c[3] = shade_weight(pos, nrm, vr.cam, edge, pad, ero);
    }
  }
  p.frag_c[slot] = make_float4(c[0], c[1], c[2], c[3]);
  p.frag_d[slot] = depth;
}

// Pass 2 (one thread per pixel): aggregation.csh across the source views IN DRAW ORDER + read-back resolve.
__global__ void __launch_bounds__(128) resolve_kernel(const ResolveParams p) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (pix >= p.S * p.S) return;
  const int px = pix % p.S, py = pix / p.S;
  float ac[4] = {0.f, 0.f, 0.f, 0.f}, ad[2] = {0.f, 0.f}, am[2] = {0.f, 0.f};
  for (int i = 0; i < p.nviews; ++i) {
    const size_t slot = (static_cast<size_t>(b) * p.nviews + i) * p.S * p.S + pix;
    const float4 c4 = p.frag_c[slot];
    const float c[4] = {c4.x, c4.y, c4.z, c4.w};
    const float depth = p.frag_d[slot];
    // aggregation.csh:18-43
    const float wc = c[3];
    const float wd = c[3] > 1e-14f ? 1.0f : (c[3] > 0.0f ? 1e-8f : 0.0f);
    const float mc = c[3] > 1e-6f ? 1.0f : 0.0f;
    const float md = c[3] > 1e-14f ? 1.0f : 0.0f;
    if (fabsf(ad[1] - 1e-8f) < 1e-8f && fabsf(wd - 1e-8f) < 1e-8f) {
      if (depth * 1e-8f > ad[0]) {
        ad[0] = depth * 1e-8f; ad[1] = 1e-8f;
        ac[0] = c[0] * wc; ac[1] = c[1] * wc; ac[2] = c[2] * wc; ac[3] = wc;
      }
    } else {
      ad[0] += depth * wd; ad[1] += wd;
      ac[0] += c[0] * wc; ac[1] += c[1] * wc; ac[2] += c[2] * wc; ac[3] += wc;
    }
    am[0] += md; am[1] += mc;
  }
  // read-back (moderngl_renderer.py:318-331): flip rows, divide by weights, linearise the z-buffer value
  const size_t o = (static_cast<size_t>(b) * p.S + (p.S - 1 - py)) * p.S + px;
  const float den = fmaxf(ac[3], 1e-24f);
  p.color[o * 3 + 0] = ac[3] > 0.f ? ac[0] / den : 0.f;
  p.color[o * 3 + 1] = ac[3] > 0.f ? ac[1] / den : 0.f;
  p.color[o * 3 + 2] = ac[3] > 0.f ? ac[2] / den : 0.f;
  const float zb = ad[1] > 0.f ? ad[0] / fmaxf(ad[1], 1e-24f) : 0.f;
  // numpy: near*far / (far - depth*(far-near)) with python-float planes on a float32 array -> float32 ops
  p.depth[o] = p.nf_f / (p.far_f - zb * p.fn_f);
  p.mask_color[o] = am[1] > 0.5f ? 1.f : 0.f;
  p.mask_depth[o] = am[0] > 0.5f ? 1.f : 0.f;
}

// SimpleRenderer read-back (moderngl_renderer.py:128-146 + shaders/simple.fsh) of ONE mesh per sample: colour = raw texture
// colour, alpha = 0 on back faces and where the interpolated edge flag exceeds 0.999, depth = linearised z-buffer value
// (cleared to 1 -> `far` where nothing was drawn), mask = alpha > 0.5; rows flipped like np.flip(pixels, axis=0).
__global__ void __launch_bounds__(128) simple_resolve_kernel(const ResolveParams p) {
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (pix >= p.S * p.S) return;
  const int px = pix % p.S, py = pix / p.S;
  const float* mvp = p.mvp + b * 16;
  const unsigned long long key = p.vis[static_cast<size_t>(b) * p.S * p.S + pix];
  float c[4] = {0.f, 0.f, 0.f, 0.f};
  float depth = 1.0f;
  if (key != ~0ull) {
    depth = __uint_as_float(static_cast<uint32_t>(key >> 32));
    const uint32_t prim = static_cast<uint32_t>(key & 0xFFFFFFFFull);
    const uint32_t f = prim >> 1, sub = prim & 1u;
    const ViewRef vr = p.views[b];
    WVtx in[3], poly[4];
#pragma unroll
    for (int k = 0; k < 3; ++k) load_vertex(vr.verts, vr.faces[f * 3 + k], mvp, in[k]);
    clip_near(in, poly);
    WVtx tv[3];
    tv[0] = poly[0];
    tv[1] = sub ? poly[2] : poly[1];
    tv[2] = sub ? poly[3] : poly[2];
    TriSetup t;
    tri_setup(tv, p.S, t);
    float l0, l1, l2;
    if (t.area > 0 && tri_eval(t, px, py, l0, l1, l2)) {
      const float b0 = l0 * t.iw[0], b1 = l1 * t.iw[1], b2 = l2 * t.iw[2];
      const float bs = (b0 + b1) + b2;
      const float c0 = b0 / bs, c1 = b1 / bs, c2 = b2 / bs;
      const float uu = (c0 * tv[0].uv[0] + c1 * tv[1].uv[0]) + c2 * tv[2].uv[0];
      const float vv = (c0 * tv[0].uv[1] + c1 * tv[1].uv[1]) + c2 * tv[2].uv[1];
      const float edge = (c0 * tv[0].edge + c1 * tv[1].edge) + c2 * tv[2].edge;
      int tx = static_cast<int>(floorf(uu * static_cast<float>(p.T))), ty = static_cast<int>(floorf(vv * static_cast<float>(p.T)));
      tx = min(max(tx, 0), p.T - 1); ty = min(max(ty, 0), p.T - 1);
      const float* tc = vr.tex + (static_cast<size_t>(ty) * p.T + tx) * 3;
      c[0] = tc[0]; c[1] = tc[1]; c[2] = tc[2];
      c[3] = edge > 0.999f ? 0.f : 1.f;
    }
  }
  const size_t o = (static_cast<size_t>(b) * p.S + (p.S - 1 - py)) * p.S + px;
  p.color[o * 3 + 0] = c[0]; p.color[o * 3 + 1] = c[1]; p.color[o * 3 + 2] = c[2];
  p.depth[o] = p.nf_f / (p.far_f - depth * p.fn_f);
  p.mask_color[o] = c[3] > 0.5f ? 1.f : 0.f;
}

// forward_backward_warp, between the two renders (utils.py:385-387): the resolved 8-bit colour becomes the float32 texture of
// the second mesh (color1 = LANCZOS(to8b(color)) / 255.0, cast by color_texture.write), depth1 = depth[off::ssaa, off::ssaa].
__global__ void fbw_mid_kernel(const unsigned char* __restrict__ col8, const float* __restrict__ depth, int n, int S, int ssaa,
                               float* __restrict__ tex, size_t tex_stride, float* __restrict__ d1) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= n * n) return;
  const int y = idx / n, x = idx % n;
  const int off = (ssaa - 1) / 2;
  const unsigned char* c8 = col8 + (static_cast<size_t>(b) * n * n + idx) * 3;
  float* t = tex + b * tex_stride + static_cast<size_t>(idx) * 3;
  for (int c = 0; c < 3; ++c) t[c] = static_cast<float>(static_cast<double>(c8[c]) / 255.0);
  d1[static_cast<size_t>(b) * n * n + idx] = depth[static_cast<size_t>(b) * S * S + static_cast<size_t>(y * ssaa + off) * S + (x * ssaa + off)];
}

// ----------------------------------------------------------------------------------------------------------------------
// mesh construction (depth_to_mesh, cal_normal=True), one thread per grid vertex / cell.  pad = 1: the grid is padded by one
// 'edge' ring ((n+2)^2 vertices; padding='frustum' or numeric); pad = 0: padding=None, n^2 vertices.
// ----------------------------------------------------------------------------------------------------------------------
struct MeshParams {
  const float* rgbd;          // [B][4][n][n] model space [-1,1]   (lin_depth_in == nullptr)
  const float* lin_depth_in;  // [B][n][n] already linearised depth (numpy-facing depth_to_mesh), or nullptr
  int B, n;                   // n = image size (128); grid is (n + 2*pad)^2
  int pad;                    // 1: one ring of 'edge' padding (padding='frustum' / numeric), 0: padding=None
  const float* tex_in;        // optional [B][n][n][3] colour texture already in [0,1] (lin_depth_in path)
  float near_f, far_f;        // linearize_depth planes (float32 casts)
  float fn_f, nf_f;           // (far-near), near*far as float32
  double focal, step;         // 0.5/tan(fov/2), plane/n (frustum) or (padding*plane)/n
  int frustum;                // 1: padding='frustum' (ring pulled to z = -0.1); 0: numeric padding
  double lin0, lin_step;      // np.linspace(0.5/n, 1-0.5/n, n): start, step
  double lin_last;
  float atol_f, rtol_f;
  int no_disc;                // 1: atol and rtol both None -> mask_discontinuity is skipped entirely (utils.py:227)
  int erode_k;                // 2*erode_rgb+1 (0 = no erosion)
  const float* inv_mv;        // [B][16] row-major float32 inverse(modelview)
  // scratch / outputs
  double* pts;                // [B][(n+2)^2][3] camera-space points (padded, frustum applied)
  double* nrm;                // [B][(n+2)^2][3]
  float* dep;                 // [B][(n+2)^2]  padded linear depth (float32)
  int* disc;                  // [B][(n+2)^2]  discontinuity flags
  float* verts;               // [B][(n+2)^2][9]
  uint32_t* faces;            // [B][2*(n+1)^2][3]
  float* tex;                 // [B][n][n][3]
  size_t verts_stride, faces_stride, tex_stride;   // per-sample strides (elements) of the destination view slot
};

__device__ __forceinline__ double lin_uv(const MeshParams& p, int i) {
  return i == p.n - 1 ? p.lin_last : static_cast<double>(i) * p.lin_step + p.lin0;
}
__device__ __forceinline__ float lin_depth(const MeshParams& p, int b, int r, int c) {
  if (p.lin_depth_in != nullptr) return p.lin_depth_in[(static_cast<size_t>(b) * p.n + r) * p.n + c];
  // rgbd*0.5+0.5 (float32), clip(1e-6, 1-1e-6), near*far/(far-(far-near)*d)   (sample.py:83, utils.py:53-55)
  const float raw = p.rgbd[((static_cast<size_t>(b) * 4 + 3) * p.n + r) * p.n + c];
  float d = raw * 0.5f + 0.5f;
  d = fminf(fmaxf(d, 1e-6f), static_cast<float>(1.0 - 1e-6));
  return p.nf_f / (p.far_f - p.fn_f * d);
}
__device__ __forceinline__ void cam_point(const MeshParams& p, int b, int r, int c, double (&o)[3]) {
  // unproject (utils.py:104-110): rays[::-1] * depth
  const double u = lin_uv(p, c), v = lin_uv(p, p.n - 1 - r);
  const double z = static_cast<double>(lin_depth(p, b, r, c));
  o[0] = (u - 0.5) / p.focal * z;
  o[1] = (v - 0.5) / p.focal * z;
  o[2] = -1.0 * z;
}

// stage 1: padded points (+frustum ring), padded depth, normals, texture
__global__ void mesh_points_kernel(const MeshParams p) {
  const int m = p.n + 2 * p.pad;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= m * m) return;
  const int R = idx / m, C = idx % m;
  const int r = min(max(R - p.pad, 0), p.n - 1), c = min(max(C - p.pad, 0), p.n - 1);     // 'edge' padding
  double pt[3];
  cam_point(p, b, r, c, pt);
  const float dz = lin_depth(p, b, r, c);
  // Sobel-smoothed normal of the unpadded grid (cal_depth_normal, utils.py:263-274)
  double ex[3] = {0, 0, 0}, ey[3] = {0, 0, 0};
  {
    const int wts[3] = {1, 2, 1};
    for (int k = -1; k <= 1; ++k) {
      const int rr = min(max(r + k, 0), p.n - 1), cc = min(max(c + k, 0), p.n - 1);
      double a[3], bq[3];
      cam_point(p, b, rr, min(c + 1, p.n - 1), a); cam_point(p, b, rr, max(c - 1, 0), bq);
      for (int j = 0; j < 3; ++j) ex[j] += wts[k + 1] * (a[j] - bq[j]);
      cam_point(p, b, max(r - 1, 0), cc, a); cam_point(p, b, min(r + 1, p.n - 1), cc, bq);
      for (int j = 0; j < 3; ++j) ey[j] += wts[k + 1] * (a[j] - bq[j]);
    }
    for (int j = 0; j < 3; ++j) { ex[j] /= 4; ey[j] /= 4; }
  }
  double nv[3] = {ex[1] * ey[2] - ex[2] * ey[1], ex[2] * ey[0] - ex[0] * ey[2], ex[0] * ey[1] - ex[1] * ey[0]};
  const double nl = sqrt(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
  for (int j = 0; j < 3; ++j) nv[j] /= nl;
  // frustum ring (utils.py:190-199), in the reference's statement order
  const double dzd = static_cast<double>(dz);
  if (p.pad) {
    if (R == 0) pt[1] += p.step * dzd;
    if (R == m - 1) pt[1] -= p.step * dzd;
    if (C == 0) pt[0] -= p.step * dzd;
    if (C == m - 1) pt[0] += p.step * dzd;
  }
  if (p.pad && p.frustum) {
    if (R == 0) { const double s = -0.1 / pt[2]; pt[0] *= s; pt[1] *= s; pt[2] *= s; }
    if (R == m - 1) { const double s = -0.1 / pt[2]; pt[0] *= s; pt[1] *= s; pt[2] *= s; }
    if (C == 0) { const double s = -0.1 / pt[2]; pt[0] *= s; pt[1] *= s; pt[2] *= s; }
    if (C == m - 1) { const double s = -0.1 / pt[2]; pt[0] *= s; pt[1] *= s; pt[2] *= s; }
  }
  const size_t o = static_cast<size_t>(b) * m * m + idx;
  for (int j = 0; j < 3; ++j) { p.pts[o * 3 + j] = pt[j]; p.nrm[o * 3 + j] = nv[j]; }
  p.dep[o] = dz;
  p.disc[o] = 0;
  if (R >= p.pad && R < p.n + p.pad && C >= p.pad && C < p.n + p.pad) {
    float* t = p.tex + b * p.tex_stride + (static_cast<size_t>(r) * p.n + c) * 3;
    if (p.rgbd != nullptr) {
      for (int j = 0; j < 3; ++j) t[j] = p.rgbd[((static_cast<size_t>(b) * 4 + j) * p.n + r) * p.n + c] * 0.5f + 0.5f;
    } else if (p.tex_in != nullptr) {
      for (int j = 0; j < 3; ++j) t[j] = p.tex_in[((static_cast<size_t>(b) * p.n + r) * p.n + c) * 3 + j];
    }
  }
}

// stage 2: per grid cell — diagonal choice, two faces, discontinuity marking (utils.py:113-141, 213-218)
__global__ void mesh_faces_kernel(const MeshParams p) {
  const int m = p.n + 2 * p.pad, q = m - 1;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= q * q) return;
  const int R = idx / q, C = idx % q;
  const uint32_t tl = R * m + C, tr = tl + 1, bl = tl + m, br = bl + 1;
  const double* P = p.pts + static_cast<size_t>(b) * m * m * 3;
  auto dist = [&](uint32_t a, uint32_t c2) {
    const double dx = P[a * 3] - P[c2 * 3], dy = P[a * 3 + 1] - P[c2 * 3 + 1], dz = P[a * 3 + 2] - P[c2 * 3 + 2];
    return sqrt(dx * dx + dy * dy + dz * dz);
  };
  const bool main_diag = dist(tl, br) < dist(tr, bl);
  uint32_t f[2][3] = {{tr, tl, main_diag ? br : bl}, {bl, br, main_diag ? tl : tr}};
  uint32_t* F = p.faces + b * p.faces_stride + static_cast<size_t>(idx) * 6;
  const float* D = p.dep + static_cast<size_t>(b) * m * m;
  int* disc = p.disc + static_cast<size_t>(b) * m * m;
  for (int t = 0; t < 2; ++t) {
    float dmax = -INFINITY, dmin = INFINITY, imax = -INFINITY, imin = INFINITY;
    for (int k = 0; k < 3; ++k) {
      F[t * 3 + k] = f[t][k];
      const float d = D[f[t][k]];
      const float inv = 1.0f / d;
      dmax = fmaxf(dmax, d); dmin = fminf(dmin, d); imax = fmaxf(imax, inv); imin = fminf(imin, inv);
    }
    if (!p.no_disc && (dmax - dmin) > p.atol_f && (imax - imin) > p.rtol_f)
      for (int k = 0; k < 3; ++k) atomicOr(disc + f[t][k], 1);
  }
}

// stage 3: erosion flags, world transform, float32 vertex buffer (utils.py:232-258, moderngl_renderer.py:284-289)
__global__ void mesh_verts_kernel(const MeshParams p) {
  const int m = p.n + 2 * p.pad;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= m * m) return;
  const int R = idx / m, C = idx % m;
  const size_t base = static_cast<size_t>(b) * m * m;
  const int* disc = p.disc + base;
  int ero = 0;
  if (p.erode_k > 0) {
    const int h = p.erode_k / 2;
    for (int dy = -h; dy <= h && !ero; ++dy)
      for (int dx = -h; dx <= h; ++dx) {
        const int rr = R + dy, cc = C + dx;
        if (rr >= 0 && rr < m && cc >= 0 && cc < m && disc[rr * m + cc]) { ero = 1; break; }
      }
  }
  const int ring = (p.pad && (R == 0 || R == m - 1 || C == 0 || C == m - 1)) ? 1 : 0;
  const int flag = disc[idx] + 2 * ring + 4 * ero;
  const float* M = p.inv_mv + b * 16;
  const double* pt = p.pts + (base + idx) * 3;
  const double* nv = p.nrm + (base + idx) * 3;
  float* o = p.verts + b * p.verts_stride + static_cast<size_t>(idx) * 9;
  for (int r = 0; r < 3; ++r) {
    const double w = ((static_cast<double>(M[r * 4]) * pt[0] + static_cast<double>(M[r * 4 + 1]) * pt[1]) +
                      static_cast<double>(M[r * 4 + 2]) * pt[2]) + static_cast<double>(M[r * 4 + 3]);
    o[r] = static_cast<float>(w);
    const double nn = (static_cast<double>(M[r * 4]) * nv[0] + static_cast<double>(M[r * 4 + 1]) * nv[1]) +
                      static_cast<double>(M[r * 4 + 2]) * nv[2];
    o[3 + r] = static_cast<float>(nn);
  }
  const int r0 = min(max(R - p.pad, 0), p.n - 1), c0 = min(max(C - p.pad, 0), p.n - 1);
  o[6] = static_cast<float>(lin_uv(p, c0));
  o[7] = static_cast<float>(lin_uv(p, r0));
  o[8] = static_cast<float>(flag);
}

// ----------------------------------------------------------------------------------------------------------------------
// aggregate_conditions post-filters (utils.py:449-469)
// ----------------------------------------------------------------------------------------------------------------------
struct PostParams {
  const float* color;        // [B][S][S][3]
  const float* depth;        // [B][S][S]
  const float* mask_color;   // [B][S][S]
  const float* mask_depth;
  int B, S, n, ssaa;
  const int* coef;           // [n][ksize] Pillow 8-bit LANCZOS coefficients (22 fractional bits)
  const int* bounds;         // [n][2] (xmin, count)
  int ksize;
  float near_f, far_f;       // project_depth planes
  float inv_near_f, denom_f; // 1/near, (1/near - 1/far) as float32
  float atol_f, rtol_f;
  int erode_k;               // 2*erode_rgb-1
  unsigned char* tmp8;       // [B][S][n][3]  horizontal pass
  unsigned char* col8;       // [B][n][n][3]
  float* dproj;              // [B][n][n] projected depth
  unsigned char* m0;         // [B][n][n] mask after votes & depth edge
  unsigned char* mr0;        // [B][n][n] mask_rgb votes
  float* out;                // [B][7][n][n]: color(3) depth mask mask_rgb depth_convex
};

__device__ __forceinline__ unsigned char to8b(float x) {
  // (np.clip(x, 0, 1) * 255).astype(np.uint8) on the float32 colour image: float32 multiply, truncation (utils.py:34-35)
  const float v = fminf(fmaxf(x, 0.0f), 1.0f) * 255.0f;
  return static_cast<unsigned char>(static_cast<int>(v));
}
__device__ __forceinline__ unsigned char clip8(int v) {
  v >>= 22;
  return static_cast<unsigned char>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Pillow ImagingResampleHorizontal_8bpc: [S rows][S] -> [S rows][n]
__global__ void lanczos_h_kernel(const PostParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= p.S * p.n) return;
  const int y = idx / p.n, xx = idx % p.n;
  const int xmin = p.bounds[xx * 2], cnt = p.bounds[xx * 2 + 1];
  const int* k = p.coef + xx * p.ksize;
  int ss[3] = {1 << 21, 1 << 21, 1 << 21};
  const float* row = p.color + ((static_cast<size_t>(b) * p.S + y) * p.S) * 3;
  for (int x = 0; x < cnt; ++x)
    for (int c = 0; c < 3; ++c) ss[c] += static_cast<int>(to8b(row[(xmin + x) * 3 + c])) * k[x];
  unsigned char* o = p.tmp8 + ((static_cast<size_t>(b) * p.S + y) * p.n + xx) * 3;
  for (int c = 0; c < 3; ++c) o[c] = clip8(ss[c]);
}
// vertical pass: [S][n] -> [n][n]
__global__ void lanczos_v_kernel(const PostParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= p.n * p.n) return;
  const int yy = idx / p.n, x = idx % p.n;
  const int ymin = p.bounds[yy * 2], cnt = p.bounds[yy * 2 + 1];
  const int* k = p.coef + yy * p.ksize;
  int ss[3] = {1 << 21, 1 << 21, 1 << 21};
  for (int y = 0; y < cnt; ++y) {
    const unsigned char* s = p.tmp8 + ((static_cast<size_t>(b) * p.S + ymin + y) * p.n + x) * 3;
    for (int c = 0; c < 3; ++c) ss[c] += static_cast<int>(s[c]) * k[y];
  }
  unsigned char* o = p.col8 + (static_cast<size_t>(b) * p.n * p.n + idx) * 3;
  for (int c = 0; c < 3; ++c) o[c] = clip8(ss[c]);
}

// depth point-sample + project_depth, 7-of-9 mask votes
__global__ void post_sample_kernel(const PostParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= p.n * p.n) return;
  const int y = idx / p.n, x = idx % p.n;
  const int off = (p.ssaa - 1) / 2;
  const size_t sb = static_cast<size_t>(b) * p.S * p.S;
  float d = p.depth[sb + static_cast<size_t>(y * p.ssaa + off) * p.S + (x * p.ssaa + off)];
  d = fminf(fmaxf(d, p.near_f), p.far_f);
  d = (p.inv_near_f - 1.0f / d) / p.denom_f;
  p.dproj[static_cast<size_t>(b) * p.n * p.n + idx] = d;
  float sd = 0.f, sc = 0.f;
  for (int j = 0; j < p.ssaa; ++j)
    for (int i = 0; i < p.ssaa; ++i) {
      const size_t o = sb + static_cast<size_t>(y * p.ssaa + j) * p.S + (x * p.ssaa + i);
      sd += p.mask_depth[o]; sc += p.mask_color[o];
    }
  const float thr = 0.75f * static_cast<float>(p.ssaa * p.ssaa);
  p.m0[static_cast<size_t>(b) * p.n * p.n + idx] = sd > thr;
  p.mr0[static_cast<size_t>(b) * p.n * p.n + idx] = sc > thr;
}

__device__ __forceinline__ bool depth_differs(float a, float bq, float atol, float rtol) {
  a = fmaxf(a, 1e-6f); bq = fmaxf(bq, 1e-6f);
  return fabsf(a - bq) > atol && fabsf(1.0f / a - 1.0f / bq) > rtol;
}
// depth_edge (utils.py:311-332): keep pixels with fewer than 3 differing 8-neighbours; mask &= edge (in place)
__global__ void post_edge_kernel(const PostParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= p.n * p.n) return;
  const int y = idx / p.n, x = idx % p.n;
  const float* D = p.dproj + static_cast<size_t>(b) * p.n * p.n;
  const float d = D[idx];
  int hits = 0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      if (dx == 0 && dy == 0) continue;
      const int yy = y + dy, xx = x + dx;
      if (yy < 0 || yy >= p.n || xx < 0 || xx >= p.n) continue;
      hits += depth_differs(d, D[yy * p.n + xx], p.atol_f, p.rtol_f) ? 1 : 0;
    }
  unsigned char* m = p.m0 + static_cast<size_t>(b) * p.n * p.n;
  // written to a second plane to keep the stencil race-free: reuse the upper bits
  m[idx] = (m[idx] & 1) | (((m[idx] & 1) && hits < 3) ? 2 : 0);
}
// Free-view frames (inference/render.py:74-84): centre point sample of the linear depth -> project_depth -> colour map.
// idx = uint8((clip(1 - d, 0, 1) * 255)) in float32 exactly as numpy evaluates colorize_depth(d, min=0, max=1) on a float32
// array; `lut` is the 256-entry uint8 RGB table the host derived from cv2.COLORMAP_INFERNO through the same numpy steps.
__global__ void depth_colormap_kernel(const float* __restrict__ depth, int S, int n, int ssaa, float near_f, float far_f,
                                      float inv_near_f, float denom_f, const unsigned char* __restrict__ lut,
                                      unsigned char* __restrict__ out) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= n * n) return;
  const int y = idx / n, x = idx % n;
  const int off = ssaa / 2;
  float d = depth[static_cast<size_t>(b) * S * S + static_cast<size_t>(y * ssaa + off) * S + (x * ssaa + off)];
  d = fminf(fmaxf(d, near_f), far_f);
  d = (inv_near_f - 1.0f / d) / denom_f;
  float v = 1.0f - d;
  v = fminf(fmaxf(v, 0.0f), 1.0f) * 255.0f;
  const int k = static_cast<int>(v);
  unsigned char* o = out + (static_cast<size_t>(b) * n * n + idx) * 3;
  o[0] = lut[k * 3 + 0]; o[1] = lut[k * 3 + 1]; o[2] = lut[k * 3 + 2];
}

// erosion of mask for mask_rgb, final products (utils.py:464-469)
__global__ void post_final_kernel(const PostParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (idx >= p.n * p.n) return;
  const int y = idx / p.n, x = idx % p.n;
  const unsigned char* m = p.m0 + static_cast<size_t>(b) * p.n * p.n;
  const bool mask = (m[idx] & 2) != 0;
  bool er = true;
  const int h = p.erode_k / 2;
  for (int dy = -h; dy <= h && er; ++dy)
    for (int dx = -h; dx <= h; ++dx) {
      const int yy = y + dy, xx = x + dx;
      if (yy < 0 || yy >= p.n || xx < 0 || xx >= p.n) continue;      // cv2 default border: ignored by erosion
      if (!(m[yy * p.n + xx] & 2)) { er = false; break; }
    }
  const bool mrgb = p.mr0[static_cast<size_t>(b) * p.n * p.n + idx] && er;
  const size_t plane = static_cast<size_t>(p.n) * p.n;
  float* o = p.out + static_cast<size_t>(b) * 7 * plane;
  const unsigned char* c8 = p.col8 + (static_cast<size_t>(b) * plane + idx) * 3;
  for (int c = 0; c < 3; ++c) o[c * plane + idx] = mrgb ? static_cast<float>(static_cast<double>(c8[c]) / 255.0) : 0.f;
  const float d = p.dproj[static_cast<size_t>(b) * plane + idx];
  o[3 * plane + idx] = mask ? d : 0.f;
  o[4 * plane + idx] = mask ? 1.f : 0.f;
  o[5 * plane + idx] = mrgb ? 1.f : 0.f;
  o[6 * plane + idx] = d;
}

// ----------------------------------------------------------------------------------------------------------------------
// host object
// ----------------------------------------------------------------------------------------------------------------------
static void mat4_mul(const double* a, const double* b, double* o) {
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += a[r * 4 + k] * b[k * 4 + c];
      o[r * 4 + c] = s;
    }
}
static void mat4_inverse(const float* m, float* out) {
  // general 4x4 inverse in double (Gauss-Jordan), result rounded to float32 (glm::inverse works in float32)
  double a[4][8];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) { a[r][c] = m[r * 4 + c]; a[r][4 + c] = r == c ? 1.0 : 0.0; }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int r = c + 1; r < 4; ++r) if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
    if (std::fabs(a[piv][c]) < 1e-30) throw Error(kErrInvalidArgument, "modelview matrix is singular");
    if (piv != c) for (int k = 0; k < 8; ++k) std::swap(a[piv][k], a[c][k]);
    const double d = a[c][c];
    for (int k = 0; k < 8; ++k) a[c][k] /= d;
    for (int r = 0; r < 4; ++r)
      if (r != c) { const double f = a[r][c]; for (int k = 0; k < 8; ++k) a[r][k] -= f * a[c][k]; }
  }
  for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) out[r * 4 + c] = static_cast<float>(a[r][4 + c]);
}

class Warp {
 public:
  Warp(int image_size, int render_size, int max_views, int batch, double near, double far, int device)
      : n_(image_size), S_(render_size), maxv_(max_views), B_(batch), near_(near), far_(far), device_(device) {
    IVID_REQUIRE(image_size >= 8 && render_size % image_size == 0, "render_size must be a multiple of image_size");
    IVID_REQUIRE(batch >= 1 && max_views >= 1, "batch and max_views must be positive");
    IVID_CHECK_CUDA(cudaSetDevice(device));
    const int m = n_ + 2;
    V_ = m * m; F_ = 2 * (m - 1) * (m - 1);
    const size_t slots = static_cast<size_t>(B_) * maxv_;
    IVID_CHECK_CUDA(cudaMalloc(&verts_, slots * V_ * 9 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&faces_, slots * F_ * 3 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&tex_, slots * n_ * n_ * 3 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&views_dev_, slots * sizeof(ViewRef)));
    IVID_CHECK_CUDA(cudaMalloc(&vis_, slots * S_ * S_ * 8));
    IVID_CHECK_CUDA(cudaMalloc(&frag_c_, slots * S_ * S_ * sizeof(float4)));
    IVID_CHECK_CUDA(cudaMalloc(&frag_d_, slots * S_ * S_ * 4));
    IVID_CHECK_CUDA(cudaMalloc(&mvp_dev_, B_ * 16 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&inv_dev_, B_ * 16 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&pts_, static_cast<size_t>(B_) * V_ * 3 * 8));
    IVID_CHECK_CUDA(cudaMalloc(&nrm_, static_cast<size_t>(B_) * V_ * 3 * 8));
    IVID_CHECK_CUDA(cudaMalloc(&dep_, static_cast<size_t>(B_) * V_ * 4));
    IVID_CHECK_CUDA(cudaMalloc(&disc_, static_cast<size_t>(B_) * V_ * 4));
    const size_t px = static_cast<size_t>(B_) * S_ * S_;
    IVID_CHECK_CUDA(cudaMalloc(&raw_color_, px * 3 * 4));
    IVID_CHECK_CUDA(cudaMalloc(&raw_depth_, px * 4));
    IVID_CHECK_CUDA(cudaMalloc(&raw_mc_, px * 4));
    IVID_CHECK_CUDA(cudaMalloc(&raw_md_, px * 4));
    IVID_CHECK_CUDA(cudaMalloc(&tmp8_, static_cast<size_t>(B_) * S_ * n_ * 3));
    IVID_CHECK_CUDA(cudaMalloc(&col8_, static_cast<size_t>(B_) * n_ * n_ * 3));
    IVID_CHECK_CUDA(cudaMalloc(&dproj_, static_cast<size_t>(B_) * n_ * n_ * 4));
    IVID_CHECK_CUDA(cudaMalloc(&m0_, static_cast<size_t>(B_) * n_ * n_));
    IVID_CHECK_CUDA(cudaMalloc(&mr0_, static_cast<size_t>(B_) * n_ * n_));
    cams_.assign(slots * 3, 0.f);
    build_lanczos();
  }
  ~Warp() {
    for (void* p : {static_cast<void*>(verts_), static_cast<void*>(faces_), static_cast<void*>(tex_), static_cast<void*>(views_dev_),
                    static_cast<void*>(vis_), static_cast<void*>(frag_c_), static_cast<void*>(frag_d_), static_cast<void*>(mvp_dev_), static_cast<void*>(inv_dev_), static_cast<void*>(pts_),
                    static_cast<void*>(nrm_), static_cast<void*>(dep_), static_cast<void*>(disc_), static_cast<void*>(raw_color_),
                    static_cast<void*>(raw_depth_), static_cast<void*>(raw_mc_), static_cast<void*>(raw_md_), static_cast<void*>(tmp8_),
                    static_cast<void*>(col8_), static_cast<void*>(dproj_), static_cast<void*>(m0_), static_cast<void*>(mr0_),
                    static_cast<void*>(coef_dev_), static_cast<void*>(bounds_dev_), static_cast<void*>(lut_dev_)})
      if (p) cudaFree(p);
  }
  int image_size() const { return n_; }
  int render_size() const { return S_; }
  int batch() const { return B_; }
  int num_views() const { return nviews_; }
  int V() const { return V_; }
  int F() const { return F_; }
  void reset() { nviews_ = 0; }

  float* verts_slot(int b, int v) { return verts_ + (static_cast<size_t>(b) * maxv_ + v) * V_ * 9; }
  uint32_t* faces_slot(int b, int v) { return faces_ + (static_cast<size_t>(b) * maxv_ + v) * F_ * 3; }
  float* tex_slot(int b, int v) { return tex_ + (static_cast<size_t>(b) * maxv_ + v) * n_ * n_ * 3; }

  // sample.py:126-138 for every sample of the batch: colors.append(rgb), meshes.append(depth_to_mesh(...))
  // numpy-facing depth_to_mesh: linear depth in, vertex buffer + faces out (the last view slot is used as scratch).
  // wp.padding: 0 = 'frustum', > 0 = that many pixels, < 0 = None (no ring: n^2 vertices, 2*(n-1)^2 faces).
  void mesh_from_depth(const float* lin_depth_host, const float* mv_host, const ivid_warp_params_t& wp, float* verts_host,
                       uint32_t* faces_host, cudaStream_t st) {
    IVID_REQUIRE(B_ == 1, "mesh_from_depth works on single-sample renderers");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    float* d_in = nullptr;
    IVID_CHECK_CUDA(cudaMalloc(&d_in, static_cast<size_t>(n_) * n_ * 4));
    IVID_CHECK_CUDA(cudaMemcpy(d_in, lin_depth_host, static_cast<size_t>(n_) * n_ * 4, cudaMemcpyHostToDevice));
    const int pad = wp.padding < 0.0 ? 0 : 1;
    const int m = n_ + 2 * pad;
    try {
      build_mesh(maxv_ - 1, nullptr, d_in, nullptr, mv_host, true, wp, st);
    } catch (...) { cudaFree(d_in); throw; }
    IVID_CHECK_CUDA(cudaMemcpy(verts_host, verts_slot(0, maxv_ - 1), static_cast<size_t>(m) * m * 9 * 4, cudaMemcpyDeviceToHost));
    IVID_CHECK_CUDA(cudaMemcpy(faces_host, faces_slot(0, maxv_ - 1), static_cast<size_t>(2) * (m - 1) * (m - 1) * 3 * 4, cudaMemcpyDeviceToHost));
    cudaFree(d_in);
  }
  void add_view(const float* rgbd_dev, const float* mv_host, bool shared, const ivid_warp_params_t& wp, cudaStream_t st) {
    IVID_REQUIRE(nviews_ < maxv_, "more source views than max_views");
    IVID_REQUIRE(wp.padding >= 0.0, "add_view: source views of the aggregation renderer are padded meshes");
    build_mesh(nviews_, rgbd_dev, nullptr, nullptr, mv_host, shared, wp, st);
    ++nviews_;
    views_dirty_ = true;
  }
  // depth_to_mesh for every sample of the batch into view slot `slot` (utils.py:144-260); the depth comes either from the
  // model-space RGBD (rgbd_dev, sampling loop) or from an already linearised depth image (lin_depth_dev [+ tex_in_dev]).
  void build_mesh(int slot, const float* rgbd_dev, const float* lin_depth_dev, const float* tex_in_dev, const float* mv_host,
                  bool shared, const ivid_warp_params_t& wp, cudaStream_t st) {
    IVID_REQUIRE(slot >= 0 && slot < maxv_, "view slot out of range");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    std::vector<float> inv(B_ * 16);
    for (int b = 0; b < B_; ++b) {
      const float* mv = mv_host + (shared ? 0 : b * 16);
      mat4_inverse(mv, inv.data() + b * 16);
      float* cam = cams_.data() + (static_cast<size_t>(b) * maxv_ + slot) * 3;
      cam[0] = inv[b * 16 + 3]; cam[1] = inv[b * 16 + 7]; cam[2] = inv[b * 16 + 11];     // inverse(modelview)[3] (column 3)
    }
    IVID_CHECK_CUDA(cudaMemcpyAsync(inv_dev_, inv.data(), inv.size() * 4, cudaMemcpyHostToDevice, st));
    MeshParams p;
    p.rgbd = rgbd_dev; p.lin_depth_in = lin_depth_dev; p.tex_in = tex_in_dev; p.B = B_; p.n = n_;
    p.pad = wp.padding < 0.0 ? 0 : 1;
    p.near_f = static_cast<float>(wp.near); p.far_f = static_cast<float>(wp.far);
    p.fn_f = static_cast<float>(wp.far - wp.near);
    p.nf_f = static_cast<float>(wp.near * wp.far);
    const double fov = wp.fov_deg * (M_PI / 180.0);      // np.deg2rad
    p.focal = 0.5 / std::tan(0.5 * fov);
    p.frustum = wp.padding > 0.0 ? 0 : 1;
    p.step = p.frustum ? (2 * std::tan(0.5 * fov)) / n_ : (wp.padding * (2 * std::tan(0.5 * fov))) / n_;   // utils.py:190,201
    p.lin0 = 0.5 / n_; p.lin_last = 1 - 0.5 / n_;
    p.lin_step = (p.lin_last - p.lin0) / (n_ - 1);
    // a negative tolerance stands for Python's None: both None -> no discontinuity test at all; exactly one None -> that one
    // is 0 (utils.py:227-229)
    p.no_disc = (wp.atol < 0.0 && wp.rtol < 0.0) ? 1 : 0;
    p.atol_f = static_cast<float>(wp.atol < 0.0 ? 0.0 : wp.atol); p.rtol_f = static_cast<float>(wp.rtol < 0.0 ? 0.0 : wp.rtol);
    p.erode_k = wp.erode_rgb > 0 ? 2 * wp.erode_rgb + 1 : 0;
    p.inv_mv = inv_dev_;
    p.pts = pts_; p.nrm = nrm_; p.dep = dep_; p.disc = disc_;
    p.verts = verts_slot(0, slot); p.faces = faces_slot(0, slot); p.tex = tex_slot(0, slot);
    p.verts_stride = static_cast<size_t>(maxv_) * V_ * 9; p.faces_stride = static_cast<size_t>(maxv_) * F_ * 3;
    p.tex_stride = static_cast<size_t>(maxv_) * n_ * n_ * 3;
    const int m = n_ + 2 * p.pad;
    dim3 gv((m * m + 127) / 128, B_), gf(((m - 1) * (m - 1) + 127) / 128, B_);
    mesh_points_kernel<<<gv, 128, 0, st>>>(p);
    mesh_faces_kernel<<<gf, 128, 0, st>>>(p);
    mesh_verts_kernel<<<gv, 128, 0, st>>>(p);
    IVID_CHECK_CUDA(cudaGetLastError());
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));     // inv is a host temporary
  }

  void set_mesh(int b, int v, const float* verts_host, const uint32_t* faces_host, const float* color_host, const float* mv_host) {
    IVID_REQUIRE(b >= 0 && b < B_ && v >= 0 && v < maxv_, "set_mesh: slot out of range");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    IVID_CHECK_CUDA(cudaMemcpy(verts_slot(b, v), verts_host, static_cast<size_t>(V_) * 9 * 4, cudaMemcpyHostToDevice));
    IVID_CHECK_CUDA(cudaMemcpy(faces_slot(b, v), faces_host, static_cast<size_t>(F_) * 3 * 4, cudaMemcpyHostToDevice));
    IVID_CHECK_CUDA(cudaMemcpy(tex_slot(b, v), color_host, static_cast<size_t>(n_) * n_ * 3 * 4, cudaMemcpyHostToDevice));
    float inv[16];
    mat4_inverse(mv_host, inv);
    float* cam = cams_.data() + (static_cast<size_t>(b) * maxv_ + v) * 3;
    cam[0] = inv[3]; cam[1] = inv[7]; cam[2] = inv[11];
    nviews_ = std::max(nviews_, v + 1);
    views_dirty_ = true;
  }
  // raw upload of a grid mesh with explicit sizes (SimpleRenderer meshes may be unpadded)
  void upload_mesh(int b, int v, const float* verts_host, int nverts, const uint32_t* faces_host, int nfaces, const float* color_host) {
    IVID_REQUIRE(b >= 0 && b < B_ && v >= 0 && v < maxv_ && nverts <= V_ && nfaces <= F_, "upload_mesh: out of range");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    IVID_CHECK_CUDA(cudaMemcpy(verts_slot(b, v), verts_host, static_cast<size_t>(nverts) * 9 * 4, cudaMemcpyHostToDevice));
    IVID_CHECK_CUDA(cudaMemcpy(faces_slot(b, v), faces_host, static_cast<size_t>(nfaces) * 3 * 4, cudaMemcpyHostToDevice));
    IVID_CHECK_CUDA(cudaMemcpy(tex_slot(b, v), color_host, static_cast<size_t>(n_) * n_ * 3 * 4, cudaMemcpyHostToDevice));
  }
  void download_raw(float* color, float* depth, float* mask, cudaStream_t st) {
    const size_t px = static_cast<size_t>(B_) * S_ * S_;
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
    if (color) IVID_CHECK_CUDA(cudaMemcpy(color, raw_color_, px * 12, cudaMemcpyDeviceToHost));
    if (depth) IVID_CHECK_CUDA(cudaMemcpy(depth, raw_depth_, px * 4, cudaMemcpyDeviceToHost));
    if (mask) IVID_CHECK_CUDA(cudaMemcpy(mask, raw_mc_, px * 4, cudaMemcpyDeviceToHost));
  }
  void get_mesh(int b, int v, float* verts_host, uint32_t* faces_host, float* color_host) {
    IVID_REQUIRE(b >= 0 && b < B_ && v >= 0 && v < nviews_, "get_mesh: slot out of range");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    IVID_CHECK_CUDA(cudaDeviceSynchronize());
    if (verts_host) IVID_CHECK_CUDA(cudaMemcpy(verts_host, verts_slot(b, v), static_cast<size_t>(V_) * 9 * 4, cudaMemcpyDeviceToHost));
    if (faces_host) IVID_CHECK_CUDA(cudaMemcpy(faces_host, faces_slot(b, v), static_cast<size_t>(F_) * 3 * 4, cudaMemcpyDeviceToHost));
    if (color_host) IVID_CHECK_CUDA(cudaMemcpy(color_host, tex_slot(b, v), static_cast<size_t>(n_) * n_ * 3 * 4, cudaMemcpyDeviceToHost));
  }

  // AggregationRenderer.render(meshes, colors, modelview, fov, is_autoregressive=True) for one target per sample
  void render(const float* target_mv_host, bool shared, double fov_deg, cudaStream_t st) {
    IVID_REQUIRE(nviews_ >= 1, "render: no source views");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    upload_views(st);
    upload_mvp(target_mv_host, shared, fov_deg, st);
    // visibility buffers are stored [B][nviews][S*S] contiguously for the live view count
    IVID_CHECK_CUDA(cudaMemsetAsync(vis_, 0xFF, static_cast<size_t>(B_) * nviews_ * S_ * S_ * 8, st));
    RasterParams rp;
    rp.views = views_dev_; rp.mvp = mvp_dev_; rp.vis = vis_; rp.nviews = nviews_; rp.F = F_; rp.S = S_; rp.simple = 0;
    dim3 gr((F_ + 127) / 128, nviews_, B_);
    raster_kernel<<<gr, 128, 0, st>>>(rp);
    ResolveParams sp;
    sp.views = views_dev_; sp.mvp = mvp_dev_; sp.vis = vis_; sp.nviews = nviews_; sp.S = S_; sp.T = n_;
    sp.nf_f = static_cast<float>(near_ * far_); sp.far_f = static_cast<float>(far_); sp.fn_f = static_cast<float>(far_ - near_);
    sp.color = raw_color_; sp.depth = raw_depth_; sp.mask_color = raw_mc_; sp.mask_depth = raw_md_;
    sp.frag_c = frag_c_; sp.frag_d = frag_d_;
    dim3 gsh((S_ * S_ + 127) / 128, nviews_, B_);
    shade_kernel<<<gsh, 128, 0, st>>>(sp);
    dim3 gs((S_ * S_ + 127) / 128, B_);
    resolve_kernel<<<gs, 128, 0, st>>>(sp);
    IVID_CHECK_CUDA(cudaGetLastError());
  }
  // P*MV of the target view(s): glm::perspective(radians(fov), 1, near, far) in float32, product in double -> float32
  void upload_mvp(const float* target_mv_host, bool shared, double fov_deg, cudaStream_t st) {
    const float t = std::tan(static_cast<float>(fov_deg * (M_PI / 180.0)) / 2.0f);
    const float nf = static_cast<float>(near_), ff = static_cast<float>(far_);
    double P[16] = {0};
    P[0] = static_cast<double>(1.0f / (1.0f * t));
    P[5] = static_cast<double>(1.0f / t);
    P[10] = static_cast<double>(-(ff + nf) / (ff - nf));
    P[11] = static_cast<double>(-(2.0f * ff * nf) / (ff - nf));
    P[14] = -1.0;
    std::vector<float> mvp(B_ * 16);
    for (int b = 0; b < B_; ++b) {
      double mv[16], o[16];
      for (int i = 0; i < 16; ++i) mv[i] = target_mv_host[(shared ? 0 : b * 16) + i];
      mat4_mul(P, mv, o);
      for (int i = 0; i < 16; ++i) mvp[b * 16 + i] = static_cast<float>(o[i]);
    }
    IVID_CHECK_CUDA(cudaMemcpyAsync(mvp_dev_, mvp.data(), mvp.size() * 4, cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  }

  // SimpleRenderer.render(mesh, color, modelview, fov) (moderngl_renderer.py:94-146) of the mesh in view slot `slot` of every
  // sample (faces of an n + 2*pad grid) -> raw_color_ / raw_depth_ / raw_mc_ (mask = alpha > 0.5) at render size.
  void render_simple(int slot, int pad, const float* target_mv_host, bool shared, double fov_deg, cudaStream_t st) {
    IVID_REQUIRE(slot >= 0 && slot < maxv_, "render_simple: view slot out of range");
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    std::vector<ViewRef> refs(static_cast<size_t>(B_));
    for (int b = 0; b < B_; ++b) {
      ViewRef& r = refs[b];
      r.verts = verts_slot(b, slot); r.faces = faces_slot(b, slot); r.tex = tex_slot(b, slot);
      r.cam[0] = r.cam[1] = r.cam[2] = 0.f;
    }
    IVID_CHECK_CUDA(cudaMemcpyAsync(views_dev_, refs.data(), refs.size() * sizeof(ViewRef), cudaMemcpyHostToDevice, st));
    views_dirty_ = true;       // the aggregation renderer's table was overwritten
    upload_mvp(target_mv_host, shared, fov_deg, st);
    IVID_CHECK_CUDA(cudaMemsetAsync(vis_, 0xFF, static_cast<size_t>(B_) * S_ * S_ * 8, st));
    const int m = n_ + 2 * pad;
    RasterParams rp;
    rp.views = views_dev_; rp.mvp = mvp_dev_; rp.vis = vis_; rp.nviews = 1; rp.F = 2 * (m - 1) * (m - 1); rp.S = S_; rp.simple = 1;
    dim3 gr((rp.F + 127) / 128, 1, B_);
    raster_kernel<<<gr, 128, 0, st>>>(rp);
    ResolveParams sp;
    sp.views = views_dev_; sp.mvp = mvp_dev_; sp.vis = vis_; sp.nviews = 1; sp.S = S_; sp.T = n_;
    sp.nf_f = static_cast<float>(near_ * far_); sp.far_f = static_cast<float>(far_); sp.fn_f = static_cast<float>(far_ - near_);
    sp.color = raw_color_; sp.depth = raw_depth_; sp.mask_color = raw_mc_; sp.mask_depth = raw_md_;
    dim3 gs((S_ * S_ + 127) / 128, B_);
    simple_resolve_kernel<<<gs, 128, 0, st>>>(sp);
    IVID_CHECK_CUDA(cudaGetLastError());
  }

  // forward_backward_warp (utils.py:335-417) for every sample of the batch: view-0 RGBD -> mesh (wp.padding) -> rendered at
  // view 1 -> resolved (8-bit LANCZOS colour, point-sampled depth) -> re-meshed without padding, with the discontinuity
  // test -> rendered back at view 0 -> resolve, project_depth, 7-of-9 mask vote, depth_edge, products.
  //   lin_depth0_dev [B][n][n] linearised view-0 depth, color0_dev [B][n][n][3] in [0,1]; out_dev [B][7][n][n] =
  //   color(3) depth mask mask mask-less-projected-depth (same layout as aggregate_conditions; rows 4 and 5 are both `mask`).
  void forward_backward(const float* lin_depth0_dev, const float* color0_dev, const float* mv1_host, const float* mv0_host, bool shared,
                        const ivid_warp_params_t& wp, float* out_dev, cudaStream_t st) {
    IVID_REQUIRE(maxv_ >= 2, "forward_backward_warp needs two view slots");
    IVID_REQUIRE((S_ / n_) % 2 == 1 || S_ == n_, "forward_backward_warp: odd super-sampling factor");
    ivid_warp_params_t w0 = wp;
    w0.atol = -1.0; w0.rtol = -1.0; w0.erode_rgb = 0;                 // mesh0: atol = rtol = None (utils.py:378-379)
    build_mesh(0, nullptr, lin_depth0_dev, color0_dev, mv0_host, shared, w0, st);
    render_simple(0, wp.padding < 0.0 ? 0 : 1, mv1_host, shared, wp.fov_deg, st);
    PostParams pp = post_params(raw_color_, raw_depth_, raw_mc_, raw_mc_, wp, nullptr);
    dim3 gh((S_ * n_ + 127) / 128, B_), gn((n_ * n_ + 127) / 128, B_);
    lanczos_h_kernel<<<gh, 128, 0, st>>>(pp);
    lanczos_v_kernel<<<gn, 128, 0, st>>>(pp);
    fbw_mid_kernel<<<gn, 128, 0, st>>>(col8_, raw_depth_, n_, S_, S_ / n_, tex_slot(0, 1), static_cast<size_t>(maxv_) * n_ * n_ * 3, dproj_);
    IVID_CHECK_CUDA(cudaGetLastError());
    ivid_warp_params_t w1 = wp;
    w1.padding = -1.0; w1.erode_rgb = 0;                              // mesh1: padding=None, atol / rtol as given
    build_mesh(1, nullptr, dproj_, nullptr, mv1_host, shared, w1, st);
    render_simple(1, 0, mv0_host, shared, wp.fov_deg, st);
    ivid_warp_params_t wpost = wp;
    wpost.erode_rgb = 1;                                              // no erosion: mask_rgb == mask
    post(raw_color_, raw_depth_, raw_mc_, raw_mc_, wpost, out_dev, st);
    nviews_ = 0;
  }

  // inference/render.py:74-84 on the last raw render: 8-bit LANCZOS colour + colour-mapped projected depth, both uint8
  // [B][n][n][3] on the host (two 48 KB copies per frame instead of the 640^2 float images)
  void resolve_frame(double pnear, double pfar, const unsigned char* lut_host, unsigned char* color8_host, unsigned char* depth8_host,
                     cudaStream_t st) {
    IVID_CHECK_CUDA(cudaSetDevice(device_));
    ivid_warp_params_t wp{};
    wp.near = pnear; wp.far = pfar; wp.erode_rgb = 1;
    PostParams pp = post_params(raw_color_, raw_depth_, raw_mc_, raw_md_, wp, nullptr);
    dim3 gh((S_ * n_ + 127) / 128, B_), gn((n_ * n_ + 127) / 128, B_);
    lanczos_h_kernel<<<gh, 128, 0, st>>>(pp);
    lanczos_v_kernel<<<gn, 128, 0, st>>>(pp);
    if (lut_dev_ == nullptr) IVID_CHECK_CUDA(cudaMalloc(&lut_dev_, 768));
    IVID_CHECK_CUDA(cudaMemcpyAsync(lut_dev_, lut_host, 768, cudaMemcpyHostToDevice, st));
    unsigned char* d8 = tmp8_;      // the horizontal-pass scratch is free again after the vertical pass
    depth_colormap_kernel<<<gn, 128, 0, st>>>(raw_depth_, S_, n_, S_ / n_, pp.near_f, pp.far_f, pp.inv_near_f, pp.denom_f, lut_dev_, d8);
    IVID_CHECK_CUDA(cudaGetLastError());
    const size_t bytes = static_cast<size_t>(B_) * n_ * n_ * 3;
    IVID_CHECK_CUDA(cudaMemcpyAsync(color8_host, col8_, bytes, cudaMemcpyDeviceToHost, st));
    IVID_CHECK_CUDA(cudaMemcpyAsync(depth8_host, d8, bytes, cudaMemcpyDeviceToHost, st));
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  }

  void copy_raw(float* color, float* depth, float* mc, float* md, cudaStream_t st) {
    const size_t px = static_cast<size_t>(B_) * S_ * S_;
    if (color) IVID_CHECK_CUDA(cudaMemcpyAsync(color, raw_color_, px * 12, cudaMemcpyDeviceToDevice, st));
    if (depth) IVID_CHECK_CUDA(cudaMemcpyAsync(depth, raw_depth_, px * 4, cudaMemcpyDeviceToDevice, st));
    if (mc) IVID_CHECK_CUDA(cudaMemcpyAsync(mc, raw_mc_, px * 4, cudaMemcpyDeviceToDevice, st));
    if (md) IVID_CHECK_CUDA(cudaMemcpyAsync(md, raw_md_, px * 4, cudaMemcpyDeviceToDevice, st));
  }

  // aggregate_conditions(renderer, meshes, colors, modelview, fov, near, far, atol, rtol, erode_rgb)
  void aggregate(const float* target_mv_host, bool shared, const ivid_warp_params_t& wp, float* out_dev, cudaStream_t st) {
    render(target_mv_host, shared, wp.fov_deg, st);
    post(raw_color_, raw_depth_, raw_mc_, raw_md_, wp, out_dev, st);
  }
  PostParams post_params(const float* color, const float* depth, const float* mc, const float* md, const ivid_warp_params_t& wp,
                         float* out_dev) {
    PostParams p;
    p.color = color; p.depth = depth; p.mask_color = mc; p.mask_depth = md;
    p.B = B_; p.S = S_; p.n = n_; p.ssaa = S_ / n_;
    p.coef = coef_dev_; p.bounds = bounds_dev_; p.ksize = ksize_;
    p.near_f = static_cast<float>(wp.near); p.far_f = static_cast<float>(wp.far);
    p.inv_near_f = static_cast<float>(1.0 / wp.near);
    p.denom_f = static_cast<float>(1.0 / wp.near - 1.0 / wp.far);
    p.atol_f = static_cast<float>(wp.atol < 0.0 ? 0.0 : wp.atol); p.rtol_f = static_cast<float>(wp.rtol < 0.0 ? 0.0 : wp.rtol);
    p.erode_k = 2 * wp.erode_rgb - 1;
    p.tmp8 = tmp8_; p.col8 = col8_; p.dproj = dproj_; p.m0 = m0_; p.mr0 = mr0_; p.out = out_dev;
    return p;
  }
  void post(const float* color, const float* depth, const float* mc, const float* md, const ivid_warp_params_t& wp, float* out_dev,
            cudaStream_t st) {
    IVID_REQUIRE(wp.erode_rgb >= 1, "aggregate_conditions: erode_rgb must be >= 1");
    PostParams p = post_params(color, depth, mc, md, wp, out_dev);
    dim3 gh((S_ * n_ + 127) / 128, B_), gn((n_ * n_ + 127) / 128, B_);
    lanczos_h_kernel<<<gh, 128, 0, st>>>(p);
    lanczos_v_kernel<<<gn, 128, 0, st>>>(p);
    post_sample_kernel<<<gn, 128, 0, st>>>(p);
    post_edge_kernel<<<gn, 128, 0, st>>>(p);
    post_final_kernel<<<gn, 128, 0, st>>>(p);
    IVID_CHECK_CUDA(cudaGetLastError());
  }

 private:
  void upload_views(cudaStream_t st) {
    // ViewRef table laid out [B][nviews] for the live view count
    std::vector<ViewRef> refs(static_cast<size_t>(B_) * nviews_);
    for (int b = 0; b < B_; ++b)
      for (int v = 0; v < nviews_; ++v) {
        ViewRef& r = refs[static_cast<size_t>(b) * nviews_ + v];
        r.verts = verts_slot(b, v); r.faces = faces_slot(b, v); r.tex = tex_slot(b, v);
        const float* cam = cams_.data() + (static_cast<size_t>(b) * maxv_ + v) * 3;
        r.cam[0] = cam[0]; r.cam[1] = cam[1]; r.cam[2] = cam[2];
      }
    IVID_CHECK_CUDA(cudaMemcpyAsync(views_dev_, refs.data(), refs.size() * sizeof(ViewRef), cudaMemcpyHostToDevice, st));
    IVID_CHECK_CUDA(cudaStreamSynchronize(st));
    views_dirty_ = false;
  }
  // Pillow precompute_coeffs + normalize_coeffs_8bpc for LANCZOS (support 3), S -> n (PIL 'Image.resize(..., LANCZOS)',
  // reference utils.py:454); coefficients in 22-bit fixed point exactly as libImaging/Resample.c computes them.
  void build_lanczos() {
    const double scale = static_cast<double>(S_) / n_;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 3.0 * filterscale;
    ksize_ = static_cast<int>(std::ceil(support)) * 2 + 1;
    std::vector<int> coef(static_cast<size_t>(n_) * ksize_, 0), bounds(static_cast<size_t>(n_) * 2);
    auto sinc = [](double x) { return x == 0.0 ? 1.0 : std::sin(x * M_PI) / (x * M_PI); };
    auto lanczos = [&](double x) { return (-3.0 <= x && x < 3.0) ? sinc(x) * sinc(x / 3) : 0.0; };
    std::vector<double> k(ksize_);
    for (int xx = 0; xx < n_; ++xx) {
      const double center = (xx + 0.5) * scale;
      const double ss = 1.0 / filterscale;
      int xmin = static_cast<int>(center - support + 0.5);
      if (xmin < 0) xmin = 0;
      int xmax = static_cast<int>(center + support + 0.5);
      if (xmax > S_) xmax = S_;
      xmax -= xmin;
      double ww = 0.0;
      for (int x = 0; x < xmax; ++x) { k[x] = lanczos((x + xmin - center + 0.5) * ss); ww += k[x]; }
      for (int x = 0; x < xmax; ++x) {
        if (ww != 0.0) k[x] /= ww;
        coef[static_cast<size_t>(xx) * ksize_ + x] = k[x] < 0 ? static_cast<int>(-0.5 + k[x] * (1 << 22)) : static_cast<int>(0.5 + k[x] * (1 << 22));
      }
      bounds[xx * 2] = xmin; bounds[xx * 2 + 1] = xmax;
    }
    IVID_CHECK_CUDA(cudaMalloc(&coef_dev_, coef.size() * 4));
    IVID_CHECK_CUDA(cudaMalloc(&bounds_dev_, bounds.size() * 4));
    IVID_CHECK_CUDA(cudaMemcpy(coef_dev_, coef.data(), coef.size() * 4, cudaMemcpyHostToDevice));
    IVID_CHECK_CUDA(cudaMemcpy(bounds_dev_, bounds.data(), bounds.size() * 4, cudaMemcpyHostToDevice));
  }

  int n_, S_, maxv_, B_;
  double near_, far_;         // renderer planes as the python floats the reference passes (0.01, 200.0)
  int device_;
  int V_ = 0, F_ = 0, nviews_ = 0, ksize_ = 0;
  bool views_dirty_ = true;
  float* verts_ = nullptr; uint32_t* faces_ = nullptr; float* tex_ = nullptr; ViewRef* views_dev_ = nullptr;
  unsigned long long* vis_ = nullptr; float4* frag_c_ = nullptr; float* frag_d_ = nullptr; float* mvp_dev_ = nullptr; float* inv_dev_ = nullptr;
  double* pts_ = nullptr; double* nrm_ = nullptr; float* dep_ = nullptr; int* disc_ = nullptr;
  float *raw_color_ = nullptr, *raw_depth_ = nullptr, *raw_mc_ = nullptr, *raw_md_ = nullptr;
  unsigned char *tmp8_ = nullptr, *col8_ = nullptr, *m0_ = nullptr, *mr0_ = nullptr;
  float* dproj_ = nullptr;
  int *coef_dev_ = nullptr, *bounds_dev_ = nullptr;
  unsigned char* lut_dev_ = nullptr;
  std::vector<float> cams_;
};

}  // namespace ivid

// ----------------------------------------------------------------------------------------------------------------------
// C ABI
// ----------------------------------------------------------------------------------------------------------------------
using namespace ivid;
struct ivid_warp { std::unique_ptr<Warp> impl; };
namespace ivid { void set_last_error(const std::string& msg); }   // api.cu

template <class Fn>
static int warp_guard(Fn&& f) {
  try { f(); return IVID_OK; }
  catch (const Error& e) { set_last_error(e.what()); return e.code; }
  catch (const std::exception& e) { set_last_error(e.what()); return IVID_ERR_STATE; }
}

extern "C" {
int ivid_warp_create(int image_size, int render_size, int max_views, int batch, double near, double far, int device,
                     ivid_warp_t** out) {
  return warp_guard([&] {
    IVID_REQUIRE(out != nullptr, "out must not be NULL");
    auto h = std::make_unique<ivid_warp>();
    h->impl = std::make_unique<Warp>(image_size, render_size, max_views, batch, near, far, device);
    *out = h.release();
  });
}
int ivid_warp_destroy(ivid_warp_t* w) { return warp_guard([&] { delete w; }); }
int ivid_warp_reset(ivid_warp_t* w) { return warp_guard([&] { IVID_REQUIRE(w, "handle"); w->impl->reset(); }); }
int ivid_warp_num_views(const ivid_warp_t* w, int* n) { return warp_guard([&] { IVID_REQUIRE(w && n, "args"); *n = w->impl->num_views(); }); }
int ivid_warp_add_view(ivid_warp_t* w, const float* rgbd_dev, const float* modelviews_host, int shared_modelview,
                       const ivid_warp_params_t* params, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && rgbd_dev && modelviews_host && params, "add_view: NULL argument");
    w->impl->add_view(rgbd_dev, modelviews_host, shared_modelview != 0, *params, static_cast<cudaStream_t>(stream));
  });
}
int ivid_warp_set_mesh(ivid_warp_t* w, int sample, int view, const float* verts_host, const uint32_t* faces_host,
                       const float* color_host, const float* modelview_host) {
  return warp_guard([&] {
    IVID_REQUIRE(w && verts_host && faces_host && color_host && modelview_host, "set_mesh: NULL argument");
    w->impl->set_mesh(sample, view, verts_host, faces_host, color_host, modelview_host);
  });
}
int ivid_warp_get_mesh(ivid_warp_t* w, int sample, int view, float* verts_host, uint32_t* faces_host, float* color_host) {
  return warp_guard([&] { IVID_REQUIRE(w, "handle"); w->impl->get_mesh(sample, view, verts_host, faces_host, color_host); });
}
int ivid_warp_mesh_from_depth(ivid_warp_t* w, const float* lin_depth_host, const float* modelview_host,
                              const ivid_warp_params_t* params, float* verts_host, uint32_t* faces_host, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && lin_depth_host && modelview_host && params && verts_host && faces_host, "mesh_from_depth: NULL argument");
    w->impl->mesh_from_depth(lin_depth_host, modelview_host, *params, verts_host, faces_host, static_cast<cudaStream_t>(stream));
  });
}
int ivid_warp_render(ivid_warp_t* w, const float* target_mv_host, int shared_modelview, double fov_deg, float* color_dev,
                     float* depth_dev, float* mask_color_dev, float* mask_depth_dev, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && target_mv_host, "render: NULL argument");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    w->impl->render(target_mv_host, shared_modelview != 0, fov_deg, st);
    w->impl->copy_raw(color_dev, depth_dev, mask_color_dev, mask_depth_dev, st);
  });
}
int ivid_warp_aggregate(ivid_warp_t* w, const float* target_mv_host, int shared_modelview, const ivid_warp_params_t* params,
                        float* cond_dev, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && target_mv_host && params && cond_dev, "aggregate: NULL argument");
    w->impl->aggregate(target_mv_host, shared_modelview != 0, *params, cond_dev, static_cast<cudaStream_t>(stream));
  });
}
int ivid_warp_resolve_frame(ivid_warp_t* w, double project_near, double project_far, const uint8_t* lut_host, uint8_t* color8_host,
                            uint8_t* depth8_host, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && lut_host && color8_host && depth8_host, "resolve_frame: NULL argument");
    w->impl->resolve_frame(project_near, project_far, lut_host, color8_host, depth8_host, static_cast<cudaStream_t>(stream));
  });
}
int ivid_warp_render_simple(ivid_warp_t* w, const float* verts_host, int nverts, const uint32_t* faces_host, int nfaces,
                            const float* color_host, const float* target_mv_host, double fov_deg, float* color_out_host,
                            float* depth_out_host, float* mask_out_host, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && verts_host && faces_host && color_host && target_mv_host, "render_simple: NULL argument");
    Warp& W = *w->impl;
    IVID_REQUIRE(W.batch() == 1, "render_simple works on single-sample renderers");
    const int n = W.image_size();
    const int pad = nverts == (n + 2) * (n + 2) ? 1 : 0;
    const int m = n + 2 * pad;
    IVID_REQUIRE(nverts == m * m && nfaces == 2 * (m - 1) * (m - 1), "render_simple: the mesh must be an n x n or (n+2) x (n+2) grid mesh");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    W.upload_mesh(0, 0, verts_host, nverts, faces_host, nfaces, color_host);
    W.render_simple(0, pad, target_mv_host, true, fov_deg, st);
    W.download_raw(color_out_host, depth_out_host, mask_out_host, st);
  });
}
int ivid_warp_forward_backward(ivid_warp_t* w, const float* lin_depth0_host, const float* color0_host, const float* mv1_host,
                               const float* mv0_host, int shared_modelview, const ivid_warp_params_t* params, float* out_host,
                               void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && lin_depth0_host && color0_host && mv1_host && mv0_host && params && out_host, "forward_backward: NULL argument");
    Warp& W = *w->impl;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t px = static_cast<size_t>(W.batch()) * W.image_size() * W.image_size();
    float *d_lin = nullptr, *d_col = nullptr, *d_out = nullptr;
    IVID_CHECK_CUDA(cudaMalloc(&d_lin, px * 4));
    IVID_CHECK_CUDA(cudaMalloc(&d_col, px * 12));
    IVID_CHECK_CUDA(cudaMalloc(&d_out, px * 28));
    try {
      IVID_CHECK_CUDA(cudaMemcpyAsync(d_lin, lin_depth0_host, px * 4, cudaMemcpyHostToDevice, st));
      IVID_CHECK_CUDA(cudaMemcpyAsync(d_col, color0_host, px * 12, cudaMemcpyHostToDevice, st));
      W.forward_backward(d_lin, d_col, mv1_host, mv0_host, shared_modelview != 0, *params, d_out, st);
      IVID_CHECK_CUDA(cudaMemcpyAsync(out_host, d_out, px * 28, cudaMemcpyDeviceToHost, st));
      IVID_CHECK_CUDA(cudaStreamSynchronize(st));
    } catch (...) { cudaFree(d_lin); cudaFree(d_col); cudaFree(d_out); throw; }
    cudaFree(d_lin); cudaFree(d_col); cudaFree(d_out);
  });
}
int ivid_warp_postfilter(ivid_warp_t* w, const float* color_dev, const float* depth_dev, const float* mask_color_dev,
                         const float* mask_depth_dev, const ivid_warp_params_t* params, float* cond_dev, void* stream) {
  return warp_guard([&] {
    IVID_REQUIRE(w && color_dev && depth_dev && mask_color_dev && mask_depth_dev && params && cond_dev, "postfilter: NULL argument");
    w->impl->post(color_dev, depth_dev, mask_color_dev, mask_depth_dev, *params, cond_dev, static_cast<cudaStream_t>(stream));
  });
}
}  // extern "C"
