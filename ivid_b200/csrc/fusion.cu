// TSDF fusion of RGBD views into a dense voxel grid and surface-nets extraction of a coloured triangle mesh.
// The rule (validity, grid, integration, extraction, numbering) is defined once in oracle/fusion_ref.py; these kernels
// follow it operation for operation in fp32, and this translation unit is compiled with -fmad=false so every product and
// sum rounds as numpy's does.  Both stages are deterministic without atomics: integration is one thread per voxel over the
// views in index order; extraction numbers vertices and faces through exclusive scans of per-cell and per-voxel counts.
#include <cub/device/device_scan.cuh>

#include <cmath>
#include <cstring>
#include <string>

#include "../../include/ivid_b200.h"
#include "host_util.h"

namespace ivid {
void set_last_error(const std::string& msg);   // api.cu

namespace {

constexpr int kViewsPerLaunch = 32;   // camera rows carried in the kernel's parameter block (32 * 12 floats = 1.5 KB)

struct IntegrateParams {
  const float* depth;      // [V][n][n] linear depth
  const uint8_t* valid;    // [V][n][n] 0 / 1
  const float* color;      // [V][n][n][3]
  int n;
  float nf, focal, tv;     // float(n), 0.5 / tan(fov / 2), trunc * voxel
  float ox, oy, oz, voxel;
  int dx, dy, dz;
  int v0, nv;              // views [v0, v0 + nv) of this launch
  int first;               // 1: the accumulators start at zero instead of being read back
  float mv[kViewsPerLaunch][12];   // rows 0..2 of each row-major modelview
  float* tsum;             // [dz][dy][dx]  sum of tsdf
  float* w;                // [dz][dy][dx]  number of tsdf samples
  float* csum;             // [dz][dy][dx][3] sum of colour
  float* cw;               // [dz][dy][dx]  number of colour samples
};

// One thread per voxel, views in index order (oracle/fusion_ref.py:integrate).
__global__ void __launch_bounds__(256) tsdf_integrate_kernel(const IntegrateParams p) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int nvox = p.dx * p.dy * p.dz;
  if (idx >= nvox) return;
  const int i = idx % p.dx, j = (idx / p.dx) % p.dy, k = idx / (p.dx * p.dy);
  const float x = p.ox + (static_cast<float>(i) + 0.5f) * p.voxel;
  const float y = p.oy + (static_cast<float>(j) + 0.5f) * p.voxel;
  const float z = p.oz + (static_cast<float>(k) + 0.5f) * p.voxel;
  float ts = 0.f, w = 0.f, cr = 0.f, cg = 0.f, cb = 0.f, cw = 0.f;
  if (!p.first) {
    ts = p.tsum[idx]; w = p.w[idx]; cw = p.cw[idx];
    cr = p.csum[static_cast<size_t>(idx) * 3]; cg = p.csum[static_cast<size_t>(idx) * 3 + 1]; cb = p.csum[static_cast<size_t>(idx) * 3 + 2];
  }
  const size_t plane = static_cast<size_t>(p.n) * p.n;
  for (int v = 0; v < p.nv; ++v) {
    const float* M = p.mv[v];
    const float cz = ((M[8] * x + M[9] * y) + M[10] * z) + M[11];
    if (cz >= 0.f) continue;
    const float cx = ((M[0] * x + M[1] * y) + M[2] * z) + M[3];
    const float cy = ((M[4] * x + M[5] * y) + M[6] * z) + M[7];
    const float dist = -cz;
    const float col = floorf(((cx / dist) * p.focal + 0.5f) * p.nf);
    const float rowv = floorf(((cy / dist) * p.focal + 0.5f) * p.nf);
    if (!(col >= 0.f && col < p.nf && rowv >= 0.f && rowv < p.nf)) continue;
    const size_t pix = static_cast<size_t>(p.v0 + v) * plane + static_cast<size_t>(p.n - 1 - static_cast<int>(rowv)) * p.n +
                       static_cast<int>(col);
    if (!p.valid[pix]) continue;
    const float sdf = p.depth[pix] - dist;
    if (sdf < -p.tv) continue;
    ts += fminf(1.f, sdf / p.tv);
    w += 1.f;
    if (fabsf(sdf) <= p.tv) {
      cr += p.color[pix * 3]; cg += p.color[pix * 3 + 1]; cb += p.color[pix * 3 + 2];
      cw += 1.f;
    }
  }
  p.tsum[idx] = ts; p.w[idx] = w; p.cw[idx] = cw;
  p.csum[static_cast<size_t>(idx) * 3] = cr; p.csum[static_cast<size_t>(idx) * 3 + 1] = cg; p.csum[static_cast<size_t>(idx) * 3 + 2] = cb;
}

// ------------------------------------------------------------------------------------------------------------------------
// surface nets
// ------------------------------------------------------------------------------------------------------------------------
struct ExtractParams {
  const float* tsum;
  const float* w;
  const float* csum;
  const float* cw;
  int dx, dy, dz;
  float ox, oy, oz, voxel;
  int* active;             // [cells + 1] 0 / 1, then scanned into vidx
  const int* vidx;         // [cells + 1] exclusive scan of active
  long long* quads;        // [voxels + 1] quads emitted by the voxel's +x, +y, +z edges
  const long long* qoff;   // [voxels + 1] exclusive scan of quads
  float* verts;            // [N][3]
  uint8_t* colors;         // [N][3]
  long long* faces;        // [2 * quads][3]
};

// tsdf of voxel v; false where no view wrote it
__device__ __forceinline__ bool voxel_tsdf(const ExtractParams& p, long long v, float& t) {
  const float w = p.w[v];
  if (!(w > 0.f)) return false;
  t = p.tsum[v] / w;
  return true;
}

__device__ __forceinline__ long long vox(const ExtractParams& p, int i, int j, int k) {
  return (static_cast<long long>(k) * p.dy + j) * p.dx + i;
}

// corner q of cell (i,j,k) is voxel (i + (q & 1), j + (q >> 1 & 1), k + (q >> 2))
__device__ __forceinline__ bool cell_corners(const ExtractParams& p, int i, int j, int k, float (&T)[8]) {
#pragma unroll
  for (int q = 0; q < 8; ++q)
    if (!voxel_tsdf(p, vox(p, i + (q & 1), j + ((q >> 1) & 1), k + (q >> 2)), T[q])) return false;
  return true;
}

__global__ void __launch_bounds__(256) cell_active_kernel(const ExtractParams p) {
  const int cx = p.dx - 1, cy = p.dy - 1, cz = p.dz - 1;
  const int ncell = cx * cy * cz;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > ncell) return;
  int act = 0;
  if (c < ncell) {
    float T[8];
    if (cell_corners(p, c % cx, (c / cx) % cy, c / (cx * cy), T)) {
      int nin = 0;
#pragma unroll
      for (int q = 0; q < 8; ++q) nin += T[q] < 0.f ? 1 : 0;
      act = (nin != 0 && nin != 8) ? 1 : 0;
    }
  }
  p.active[c] = act;
}

// Is cell (i,j,k) inside the cell grid and active?
__device__ __forceinline__ bool cell_on(const ExtractParams& p, int i, int j, int k) {
  if (i < 0 || j < 0 || k < 0 || i >= p.dx - 1 || j >= p.dy - 1 || k >= p.dz - 1) return false;
  return p.active[(static_cast<long long>(k) * (p.dy - 1) + j) * (p.dx - 1) + i] != 0;
}
__device__ __forceinline__ int cell_id(const ExtractParams& p, int i, int j, int k) {
  return p.vidx[(static_cast<long long>(k) * (p.dy - 1) + j) * (p.dx - 1) + i];
}

// The quad of voxel (i,j,k)'s edge along `axis`: 0 = none, +1 = its inside end is (i,j,k) (outward normal along +axis),
// -1 = its inside end is the neighbour.  The four cells around the edge, in the order c00, c10, c11, c01 over the two other
// axes u = axis+1, v = axis+2 (mod 3), go to cells[][3].
__device__ __forceinline__ int edge_quad(const ExtractParams& p, int i, int j, int k, int axis, int (&cells)[4][3]) {
  const int a[3] = {i, j, k};
  const int u = (axis + 1) % 3, v = (axis + 2) % 3;
  const int du[4] = {-1, 0, 0, -1}, dv[4] = {-1, -1, 0, 0};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    int c[3] = {a[0], a[1], a[2]};
    c[u] += du[q]; c[v] += dv[q];
    if (!cell_on(p, c[0], c[1], c[2])) return 0;
    cells[q][0] = c[0]; cells[q][1] = c[1]; cells[q][2] = c[2];
  }
  // all four cells are active, so both ends of the edge carry weight
  int b[3] = {i, j, k};
  b[axis] += 1;
  float ta, tb;
  voxel_tsdf(p, vox(p, i, j, k), ta);
  voxel_tsdf(p, vox(p, b[0], b[1], b[2]), tb);
  const bool ia = ta < 0.f, ib = tb < 0.f;
  if (ia == ib) return 0;
  return ia ? 1 : -1;
}

__global__ void __launch_bounds__(256) edge_count_kernel(const ExtractParams p) {
  const int nvox = p.dx * p.dy * p.dz;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v > nvox) return;
  long long q = 0;
  if (v < nvox) {
    const int i = v % p.dx, j = (v / p.dx) % p.dy, k = v / (p.dx * p.dy);
    int cells[4][3];
#pragma unroll
    for (int axis = 0; axis < 3; ++axis) q += edge_quad(p, i, j, k, axis, cells) != 0 ? 1 : 0;
  }
  p.quads[v] = q;
}

__device__ __forceinline__ uint8_t to_u8(float c) {
  return static_cast<uint8_t>(floorf(fminf(fmaxf(c, 0.f), 1.f) * 255.f + 0.5f));
}

// Vertex of every active cell: the mean of the zero crossings on its sign-changing edges, in the fixed edge order of
// oracle/fusion_ref.py:EDGES (x edges, then y, then z; the first corner of each edge is its lower end).
__global__ void __launch_bounds__(256) vertex_kernel(const ExtractParams p) {
  const int cx = p.dx - 1, cy = p.dy - 1, cz = p.dz - 1;
  const int ncell = cx * cy * cz;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= ncell || !p.active[c]) return;
  const int i = c % cx, j = (c / cx) % cy, k = c / (cx * cy);
  float T[8];
  cell_corners(p, i, j, k, T);
  constexpr int kEdges[12][2] = {{0, 1}, {2, 3}, {4, 5}, {6, 7}, {0, 2}, {1, 3}, {4, 6}, {5, 7}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
  float s[3] = {0.f, 0.f, 0.f}, cnt = 0.f;
#pragma unroll
  for (int e = 0; e < 12; ++e) {
    const int qa = kEdges[e][0], qb = kEdges[e][1], axis = e / 4;
    const float ta = T[qa], tb = T[qb];
    if ((ta < 0.f) == (tb < 0.f)) continue;
    const float t = ta / (ta - tb);
#pragma unroll
    for (int d = 0; d < 3; ++d) s[d] += d == axis ? t : static_cast<float>((qa >> d) & 1);
    cnt += 1.f;
  }
  const long long o = cell_id(p, i, j, k);
  const float org[3] = {p.ox, p.oy, p.oz};
  const int ci[3] = {i, j, k};
#pragma unroll
  for (int d = 0; d < 3; ++d) p.verts[o * 3 + d] = org[d] + ((static_cast<float>(ci[d]) + 0.5f) + s[d] / cnt) * p.voxel;
  float rgb[3] = {0.f, 0.f, 0.f}, nc = 0.f;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const long long v = vox(p, i + (q & 1), j + ((q >> 1) & 1), k + (q >> 2));
    const float cw = p.cw[v];
    if (!(cw > 0.f)) continue;
#pragma unroll
    for (int d = 0; d < 3; ++d) rgb[d] += p.csum[v * 3 + d] / cw;
    nc += 1.f;
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) p.colors[o * 3 + d] = nc > 0.f ? to_u8(rgb[d] / nc) : 0;
}

// Two triangles per quad, quads in edge order (voxel linear order, then axis x, y, z), wound so that the right-hand normal
// points from the inside end of the edge to its outside end.
__global__ void __launch_bounds__(256) face_kernel(const ExtractParams p) {
  const int nvox = p.dx * p.dy * p.dz;
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvox || p.quads[v] == 0) return;
  const int i = v % p.dx, j = (v / p.dx) % p.dy, k = v / (p.dx * p.dy);
  long long f = p.qoff[v] * 2;
#pragma unroll
  for (int axis = 0; axis < 3; ++axis) {
    int cells[4][3];
    const int dir = edge_quad(p, i, j, k, axis, cells);
    if (dir == 0) continue;
    long long id[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) id[q] = cell_id(p, cells[q][0], cells[q][1], cells[q][2]);
    long long* F = p.faces + f * 3;
    if (dir > 0) {
      F[0] = id[0]; F[1] = id[1]; F[2] = id[2]; F[3] = id[0]; F[4] = id[2]; F[5] = id[3];
    } else {
      F[0] = id[0]; F[1] = id[2]; F[2] = id[1]; F[3] = id[0]; F[4] = id[3]; F[5] = id[2];
    }
    f += 2;
  }
}

void check_grid(const ivid_fusion_grid_t* g) {
  IVID_REQUIRE(g != nullptr, "fusion: grid must not be NULL");
  IVID_REQUIRE(g->dims[0] >= 2 && g->dims[1] >= 2 && g->dims[2] >= 2, "fusion: every grid dimension must be >= 2");
  IVID_REQUIRE(std::isfinite(g->voxel) && g->voxel > 0.f, "fusion: voxel size must be positive");
  IVID_REQUIRE(std::isfinite(g->origin[0]) && std::isfinite(g->origin[1]) && std::isfinite(g->origin[2]), "fusion: origin must be finite");
  const long long nvox = static_cast<long long>(g->dims[0]) * g->dims[1] * g->dims[2];
  // linear voxel indices are int32 (one past the end included)
  IVID_REQUIRE(nvox < 2147483647LL, "fusion: the grid has more voxels than a 32-bit index can address");
}

// stream-ordered scratch, released on every exit path
struct Scratch {
  cudaStream_t st;
  void* ptr = nullptr;
  Scratch(size_t bytes, cudaStream_t s) : st(s) { IVID_CHECK_CUDA(cudaMallocAsync(&ptr, bytes, s)); }
  ~Scratch() { if (ptr) cudaFreeAsync(ptr, st); }
  template <class T> T* as() const { return static_cast<T*>(ptr); }
};

void integrate(const float* depth, const uint8_t* valid, const float* color, const float* mv_host, int V, int n, float focal,
               const ivid_fusion_grid_t& g, float trunc, float* tsum, float* w, float* csum, float* cw, cudaStream_t st) {
  IntegrateParams p;
  p.depth = depth; p.valid = valid; p.color = color;
  p.n = n; p.nf = static_cast<float>(n); p.focal = focal;
  p.tv = trunc * g.voxel;
  p.ox = g.origin[0]; p.oy = g.origin[1]; p.oz = g.origin[2]; p.voxel = g.voxel;
  p.dx = g.dims[0]; p.dy = g.dims[1]; p.dz = g.dims[2];
  p.tsum = tsum; p.w = w; p.csum = csum; p.cw = cw;
  const int nvox = p.dx * p.dy * p.dz;
  const int blocks = (nvox + 255) / 256;
  for (int v0 = 0; v0 < V; v0 += kViewsPerLaunch) {
    p.v0 = v0; p.nv = V - v0 < kViewsPerLaunch ? V - v0 : kViewsPerLaunch; p.first = v0 == 0;
    for (int v = 0; v < p.nv; ++v) std::memcpy(p.mv[v], mv_host + static_cast<size_t>(v0 + v) * 16, 12 * sizeof(float));
    tsdf_integrate_kernel<<<blocks, 256, 0, st>>>(p);
    IVID_CHECK_CUDA(cudaGetLastError());
  }
}

void extract(const ivid_fusion_grid_t& g, const float* tsum, const float* w, const float* csum, const float* cw, long long max_v,
             long long max_f, float* verts, uint8_t* colors, long long* faces, long long* nv_out, long long* nf_out, cudaStream_t st) {
  ExtractParams p;
  p.tsum = tsum; p.w = w; p.csum = csum; p.cw = cw;
  p.dx = g.dims[0]; p.dy = g.dims[1]; p.dz = g.dims[2];
  p.ox = g.origin[0]; p.oy = g.origin[1]; p.oz = g.origin[2]; p.voxel = g.voxel;
  const int nvox = p.dx * p.dy * p.dz;
  const int ncell = (p.dx - 1) * (p.dy - 1) * (p.dz - 1);
  size_t tmp_a = 0, tmp_b = 0;
  IVID_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_a, static_cast<int*>(nullptr), static_cast<int*>(nullptr), ncell + 1, st));
  IVID_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tmp_b, static_cast<long long*>(nullptr), static_cast<long long*>(nullptr), nvox + 1, st));
  Scratch active(sizeof(int) * (static_cast<size_t>(ncell) + 1), st), vidx(sizeof(int) * (static_cast<size_t>(ncell) + 1), st);
  Scratch quads(sizeof(long long) * (static_cast<size_t>(nvox) + 1), st), qoff(sizeof(long long) * (static_cast<size_t>(nvox) + 1), st);
  Scratch tmp(tmp_a > tmp_b ? tmp_a : tmp_b, st);
  p.active = active.as<int>(); p.vidx = vidx.as<int>(); p.quads = quads.as<long long>(); p.qoff = qoff.as<long long>();
  p.verts = verts; p.colors = colors; p.faces = faces;
  cell_active_kernel<<<ncell / 256 + 1, 256, 0, st>>>(p);
  IVID_CHECK_CUDA(cudaGetLastError());
  IVID_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.ptr, tmp_a, active.as<int>(), vidx.as<int>(), ncell + 1, st));
  edge_count_kernel<<<nvox / 256 + 1, 256, 0, st>>>(p);
  IVID_CHECK_CUDA(cudaGetLastError());
  IVID_CHECK_CUDA(cub::DeviceScan::ExclusiveSum(tmp.ptr, tmp_b, quads.as<long long>(), qoff.as<long long>(), nvox + 1, st));
  int nv = 0;
  long long nq = 0;
  IVID_CHECK_CUDA(cudaMemcpyAsync(&nv, vidx.as<int>() + ncell, sizeof(int), cudaMemcpyDeviceToHost, st));
  IVID_CHECK_CUDA(cudaMemcpyAsync(&nq, qoff.as<long long>() + nvox, sizeof(long long), cudaMemcpyDeviceToHost, st));
  IVID_CHECK_CUDA(cudaStreamSynchronize(st));
  *nv_out = nv;
  *nf_out = 2 * nq;
  if (verts == nullptr && colors == nullptr && faces == nullptr) return;
  IVID_REQUIRE(verts != nullptr && colors != nullptr && faces != nullptr, "fusion_extract: pass all three outputs or none");
  IVID_REQUIRE(nv <= max_v && 2 * nq <= max_f, "fusion_extract: the output buffers are smaller than the mesh");
  if (nv > 0) {
    vertex_kernel<<<(ncell + 255) / 256, 256, 0, st>>>(p);
    face_kernel<<<(nvox + 255) / 256, 256, 0, st>>>(p);
    IVID_CHECK_CUDA(cudaGetLastError());
  }
}

template <class Fn>
int guard(Fn&& f) {
  try { f(); return IVID_OK; }
  catch (const Error& e) { set_last_error(e.what()); return e.code; }
  catch (const std::exception& e) { set_last_error(e.what()); return IVID_ERR_STATE; }
}

}  // namespace
}  // namespace ivid

using namespace ivid;

extern "C" {
int ivid_fusion_integrate(const float* depth_dev, const uint8_t* valid_dev, const float* color_dev, const float* modelviews_host,
                          int num_views, int image_size, float focal, const ivid_fusion_grid_t* grid, float trunc,
                          float* tsdf_sum_dev, float* weight_dev, float* color_sum_dev, float* color_weight_dev, void* stream) {
  return guard([&] {
    IVID_REQUIRE(depth_dev && valid_dev && color_dev && modelviews_host && tsdf_sum_dev && weight_dev && color_sum_dev && color_weight_dev,
                 "fusion_integrate: NULL argument");
    IVID_REQUIRE(num_views >= 1, "fusion_integrate: at least one view");
    IVID_REQUIRE(image_size >= 1, "fusion_integrate: image_size must be positive");
    IVID_REQUIRE(std::isfinite(focal) && focal > 0.f, "fusion_integrate: focal must be positive");
    IVID_REQUIRE(std::isfinite(trunc) && trunc > 0.f, "fusion_integrate: trunc must be positive");
    check_grid(grid);
    IVID_REQUIRE(std::isfinite(trunc * grid->voxel), "fusion_integrate: trunc * voxel overflows");
    integrate(depth_dev, valid_dev, color_dev, modelviews_host, num_views, image_size, focal, *grid, trunc, tsdf_sum_dev, weight_dev,
              color_sum_dev, color_weight_dev, static_cast<cudaStream_t>(stream));
  });
}

int ivid_fusion_extract(const ivid_fusion_grid_t* grid, const float* tsdf_sum_dev, const float* weight_dev, const float* color_sum_dev,
                        const float* color_weight_dev, int64_t max_vertices, int64_t max_faces, float* vertices_dev,
                        uint8_t* colors_dev, int64_t* faces_dev, int64_t* num_vertices, int64_t* num_faces, void* stream) {
  return guard([&] {
    IVID_REQUIRE(tsdf_sum_dev && weight_dev && color_sum_dev && color_weight_dev && num_vertices && num_faces,
                 "fusion_extract: NULL argument");
    check_grid(grid);
    long long nv = 0, nf = 0;
    extract(*grid, tsdf_sum_dev, weight_dev, color_sum_dev, color_weight_dev, max_vertices, max_faces, vertices_dev, colors_dev,
            reinterpret_cast<long long*>(faces_dev), &nv, &nf, static_cast<cudaStream_t>(stream));
    *num_vertices = nv;
    *num_faces = nf;
  });
}
}  // extern "C"
