// Mesh extraction, tools/mesh_generator.py + tools/visualizer.py of the original project: query grid of the occupancy sweep and
// its epilogue, marching cubes on a caller-provided grid, scene-space vertices, area-weighted vertex normals, edge-connected
// triangle clusters, small-cluster removal and the per-vertex label rays.  Conventions: DESIGN.md, "Mesh extraction".
#include <cmath>
#include <cstring>

#include <cub/cub.cuh>

#include "common.cuh"
#include "ray_ops.cuh"

namespace dmnerf {

// ---- marching-cubes case table --------------------------------------------------------------------------------------------
// Generated at compile time from the face rule (no hand-typed table).  Corner c of a cell has bit a = its offset along axis a;
// local edge e = 4 * axis + r, r = the bits of the two other axes (lower axis in bit 0).  Every face is walked on its own:
// the edges of the face whose end points differ in inside-ness are paired into segments, the inside corners of an ambiguous
// face (two diagonal inside corners) each keep their own segment, and every segment is directed so that the surface normal
// points toward the inside corners (increasing value).  A face shared by two cells yields the same segments, opposite
// directions: the surface is crack-free and consistently oriented.  The segments close into loops, taken in order of their
// smallest local edge and walked from it; each loop is a triangle fan from its first vertex whose chords all cross the cell's
// interior.  oracle/marching_cubes.py restates the rule cell by cell without a table.
constexpr int MC_MAX_TRI = 5;
struct McTable {
  uint8_t ntri[256];
  int8_t e[256][3 * MC_MAX_TRI];
};

namespace mcgen {
struct V3 { int x, y, z; };
__host__ __device__ constexpr int edge_lo(int e) {
  return (e & 1) << (e / 4 == 0 ? 1 : 0) | ((e >> 1) & 1) << (e / 4 == 2 ? 1 : 2);
}
constexpr int edge_hi(int e) { return edge_lo(e) | (1 << (e / 4)); }
constexpr V3 pos2(int c) { return {2 * (c & 1), 2 * ((c >> 1) & 1), 2 * ((c >> 2) & 1)}; }
constexpr V3 mid2(int e) {
  const V3 a = pos2(edge_lo(e)), b = pos2(edge_hi(e));
  return {(a.x + b.x) / 2, (a.y + b.y) / 2, (a.z + b.z) / 2};
}
constexpr V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
constexpr int dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
constexpr bool share_face(int e1, int e2) {
  for (int a = 0; a < 3; ++a)
    if (e1 / 4 != a && e2 / 4 != a && ((edge_lo(e1) >> a) & 1) == ((edge_lo(e2) >> a) & 1)) return true;
  return false;
}

constexpr McTable make_table() {
  McTable t{};
  for (int cs = 0; cs < 256; ++cs) {
    auto in = [cs](int c) { return (cs >> c) & 1; };
    int nxt[12] = {-1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1, -1};
    for (int a = 0; a < 3; ++a)
      for (int s = 0; s < 2; ++s) {
        int cr[4] = {0, 0, 0, 0}, nc = 0;
        for (int e = 0; e < 12; ++e)
          if (e / 4 != a && ((edge_lo(e) >> a) & 1) == s && in(edge_lo(e)) != in(edge_hi(e))) cr[nc++] = e;
        V3 nf = {0, 0, 0};
        (a == 0 ? nf.x : a == 1 ? nf.y : nf.z) = s ? 1 : -1;
        int s0[2] = {0, 0}, s1[2] = {0, 0}, ns = 0;
        V3 tw[2] = {};
        if (nc == 2) {
          // toward the centroid of the face's inside corners, from the segment's midpoint
          V3 sum = {0, 0, 0};
          int nin = 0;
          for (int c = 0; c < 8; ++c)
            if (((c >> a) & 1) == s && in(c)) { const V3 p = pos2(c); sum = {sum.x + p.x, sum.y + p.y, sum.z + p.z}; ++nin; }
          const V3 m0 = mid2(cr[0]), m1 = mid2(cr[1]);
          s0[0] = cr[0]; s1[0] = cr[1];
          tw[0] = {2 * sum.x - nin * (m0.x + m1.x), 2 * sum.y - nin * (m0.y + m1.y), 2 * sum.z - nin * (m0.z + m1.z)};
          ns = 1;
        } else if (nc == 4) {
          for (int c = 0; c < 8; ++c) {
            if (((c >> a) & 1) != s || !in(c)) continue;
            int mine[2] = {0, 0}, k = 0;
            for (int q = 0; q < 4; ++q)
              if (edge_lo(cr[q]) == c || edge_hi(cr[q]) == c) mine[k++] = cr[q];
            const V3 p = pos2(c), m0 = mid2(mine[0]), m1 = mid2(mine[1]);
            s0[ns] = mine[0]; s1[ns] = mine[1];
            tw[ns] = {2 * p.x - m0.x - m1.x, 2 * p.y - m0.y - m1.y, 2 * p.z - m0.z - m1.z};
            ++ns;
          }
        } else if (nc != 0) {
          throw "marching-cubes table: odd number of crossings on a face";
        }
        for (int q = 0; q < ns; ++q) {
          int e0 = s0[q], e1 = s1[q];
          const V3 m0 = mid2(e0), m1 = mid2(e1);
          if (dot({m1.x - m0.x, m1.y - m0.y, m1.z - m0.z}, cross(nf, tw[q])) > 0) { const int x = e0; e0 = e1; e1 = x; }
          if (nxt[e0] != -1) throw "marching-cubes table: two segments leave one edge";
          nxt[e0] = e1;
        }
      }
    bool seen[12] = {};
    int n = 0;
    for (int e = 0; e < 12; ++e) {
      if (nxt[e] < 0 || seen[e]) continue;
      int loop[12] = {}, len = 0;
      for (int x = e; !seen[x]; x = nxt[x]) { seen[x] = true; loop[len++] = x; }
      // fan apex: the first loop vertex whose chords all cross the cell's interior.  A chord between two edges of one face (a loop
      // holding both segments of an ambiguous face) would be shared with the fan of the neighbouring cell.
      int k0 = -1;
      for (int k = 0; k < len && k0 < 0; ++k) {
        bool ok = true;
        for (int j = 0; j < len; ++j)
          if (j != k && j != (k + 1) % len && j != (k + len - 1) % len && share_face(loop[k], loop[j])) ok = false;
        if (ok) k0 = k;
      }
      if (k0 < 0) throw "marching-cubes table: no fan apex with interior chords";
      for (int i = 1; i + 1 < len; ++i) {
        if (n >= MC_MAX_TRI) throw "marching-cubes table: more triangles than MC_MAX_TRI";
        t.e[cs][3 * n] = (int8_t)loop[k0];
        t.e[cs][3 * n + 1] = (int8_t)loop[(k0 + i) % len];
        t.e[cs][3 * n + 2] = (int8_t)loop[(k0 + i + 1) % len];
        ++n;
      }
    }
    t.ntri[cs] = (uint8_t)n;
  }
  return t;
}
constexpr McTable kTable = make_table();
}  // namespace mcgen

__constant__ McTable c_mc = mcgen::kTable;

static inline unsigned blocks(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

// ---- query grid and occupancy -------------------------------------------------------------------------------------------
struct GridXform {
  float r[12];     // rows of [R | t], float32 like the original's torch.from_numpy(transform).float()
  float s[3];      // extents / 2 (float32)
  float step;      // torch.linspace(-1, 1, dim) step
  int dim;
};

// torch.linspace(-1, 1, dim) on the CPU in float32: start + step * i below the half, end - step * (dim - 1 - i) above it, each a
// single rounding (fused multiply-add)
__device__ __forceinline__ float linspace_m11(int i, const GridXform& g) {
  return i < g.dim / 2 ? __fmaf_rn(g.step, (float)i, -1.0f) : __fmaf_rn(-g.step, (float)(g.dim - 1 - i), 1.0f);
}

// visualizer.make_3D_grid / grid_within_bound + mesh_generator.py:28-29, in the original's fp32 operation order:
// q = (R q_scaled summed left to right) + t, then (x, y, z) -> (x, -z, y)
__device__ __forceinline__ void sweep_point(const GridXform& g, int64_t p, float out[3]) {
  const int64_t d = g.dim;
  const float q[3] = {__fmul_rn(linspace_m11((int)(p / (d * d)), g), g.s[0]), __fmul_rn(linspace_m11((int)((p / d) % d), g), g.s[1]),
                      __fmul_rn(linspace_m11((int)(p % d), g), g.s[2])};
  float w[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* row = g.r + 4 * r;
    w[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(row[0], q[0]), __fmul_rn(row[1], q[1])), __fmul_rn(row[2], q[2])), row[3]);
  }
  out[0] = w[0];
  out[1] = -w[2];
  out[2] = w[1];
}

__global__ void grid_points_kernel(GridXform g, int64_t begin, int64_t count, float* __restrict__ pts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float w[3];
  sweep_point(g, begin + i, w);
  pts[3 * i] = w[0];
  pts[3 * i + 1] = w[1];
  pts[3 * i + 2] = w[2];
}

static GridXform make_xform(const double* T16, const double* ext3, int dim) {
  GridXform g;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) g.r[4 * r + c] = (float)T16[4 * r + c];
  for (int a = 0; a < 3; ++a) g.s[a] = (float)(ext3[a] / 2.0);
  g.step = 2.0f / (float)(dim - 1);
  g.dim = dim;
  return g;
}

int launch_grid_points(const double* T16, const double* ext3, int dim, int64_t begin, int64_t count, float* pts, cudaStream_t st) {
  DMN_CHECK(dim >= 2 && dim <= 2048, "grid_points: dim %d out of range [2, 2048]", dim);
  DMN_CHECK(begin >= 0 && count >= 0 && begin + count <= (int64_t)dim * dim * dim, "grid_points: range outside the grid");
  if (count == 0) return 0;
  grid_points_kernel<<<blocks(count, 256), 256, 0, st>>>(make_xform(T16, ext3, dim), begin, count, pts);
  DMN_LAUNCH_OK();
  return 0;
}

// mesh_generator.py:51-62: occ = 1 - exp(-relu(sigma) * voxel), sigma = channel 3 of the network output [n, c]
__device__ __forceinline__ float occupancy_of(float a, float voxel) {
  const float r = a > 0.f ? a : (a != a ? a : 0.f);           // torch.relu keeps NaN
  return __fsub_rn(1.0f, expf(__fmul_rn(-r, voxel)));
}

__global__ void occupancy_kernel(const float* __restrict__ raw, int64_t n, int c, float voxel, float* __restrict__ occ) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  occ[i] = occupancy_of(raw[i * c + 3], voxel);
}

int launch_occupancy(const float* raw, int64_t n, int c, float voxel, float* occ, cudaStream_t st) {
  if (n == 0) return 0;
  occupancy_kernel<<<blocks(n, 256), 256, 0, st>>>(raw, n, c, voxel, occ);
  DMN_LAUNCH_OK();
  return 0;
}

// The same occupancy with an object selection: the point's label is argmax_sigmoid of its c - 4 instance logits (the rule of
// the selected composites), occ = 0 where that label is not kept; labels (optional) receives the label of every point.
__global__ void occupancy_objects_kernel(const float* __restrict__ raw, int64_t n, int c, float voxel, const ObjMask keep,
                                         float* __restrict__ occ, int16_t* __restrict__ labels) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* ri = raw + i * c;
  const int label = argmax_sigmoid(ri + 4, c - 4);
  occ[i] = obj_kept(keep, label) ? occupancy_of(ri[3], voxel) : 0.0f;
  if (labels) labels[i] = (int16_t)label;
}

int launch_occupancy_objects(const float* raw, int64_t n, int c, float voxel, const ObjMask& keep, float* occ, int16_t* labels,
                             cudaStream_t st) {
  if (n == 0) return 0;
  occupancy_objects_kernel<<<blocks(n, 256), 256, 0, st>>>(raw, n, c, voxel, keep, occ, labels);
  DMN_LAUNCH_OK();
  return 0;
}

// ---- marching cubes -------------------------------------------------------------------------------------------------------
// One thread per grid point p: the crossing flags of its three +axis edges (bit a) and, when p is the lowest corner of a cell,
// that cell's case index (bit c = corner c is inside) and triangle count.
__global__ void mc_classify_kernel(const float* __restrict__ g, int nx, int ny, int nz, float level, uint8_t* __restrict__ eflags,
                                   int32_t* __restrict__ vcnt, uint8_t* __restrict__ cases, int32_t* __restrict__ tcnt,
                                   int32_t* __restrict__ nan_seen) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t sy = nz, sx = (int64_t)ny * nz;
  if (p >= sx * nx) return;
  const int k = (int)(p % nz), j = (int)((p / nz) % ny), i = (int)(p / sx);
  const float v = g[p];
  if (v != v) *nan_seen = 1;
  const bool in0 = v > level;
  int f = 0;
  if (i + 1 < nx) f |= (int)(in0 != (g[p + sx] > level));
  if (j + 1 < ny) f |= (int)(in0 != (g[p + sy] > level)) << 1;
  if (k + 1 < nz) f |= (int)(in0 != (g[p + 1] > level)) << 2;
  eflags[p] = (uint8_t)f;
  vcnt[p] = __popc(f);
  int cs = 0;
  if (i + 1 < nx && j + 1 < ny && k + 1 < nz) {
#pragma unroll
    for (int c = 0; c < 8; ++c) cs |= (int)(g[p + (c & 1) * sx + ((c >> 1) & 1) * sy + ((c >> 2) & 1)] > level) << c;
  }
  cases[p] = (uint8_t)cs;
  tcnt[p] = c_mc.ntri[cs];
}

__global__ void mc_totals_kernel(const int32_t* vscan, const int32_t* vcnt, const int32_t* tscan, const int32_t* tcnt, int64_t n,
                                 const int32_t* nan_seen, int64_t* out) {
  out[0] = (int64_t)vscan[n - 1] + vcnt[n - 1];
  out[1] = (int64_t)tscan[n - 1] + tcnt[n - 1];
  out[2] = *nan_seen;
}

// vertex of edge (p, a): p + t e_a in index units, t = (level - v0) / (v1 - v0), v0 at the lower end (one rounding per operation)
__global__ void mc_vertex_kernel(const float* __restrict__ g, int nx, int ny, int nz, float level, const uint8_t* __restrict__ eflags,
                                 const int32_t* __restrict__ vscan, float* __restrict__ verts) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t sy = nz, sx = (int64_t)ny * nz;
  if (p >= sx * nx) return;
  const int f = eflags[p];
  if (!f) return;
  const float pos[3] = {(float)(p / sx), (float)((p / nz) % ny), (float)(p % nz)};
  const int64_t stride[3] = {sx, sy, 1};
  const float v0 = g[p];
  int64_t out = vscan[p];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (!((f >> a) & 1)) continue;
    const float t = __fdiv_rn(__fsub_rn(level, v0), __fsub_rn(g[p + stride[a]], v0));
    float* o = verts + 3 * out;
    o[0] = pos[0]; o[1] = pos[1]; o[2] = pos[2];
    o[a] = __fadd_rn(pos[a], t);
    ++out;
  }
}

__global__ void mc_triangle_kernel(int nx, int ny, int nz, const uint8_t* __restrict__ cases, const int32_t* __restrict__ tscan,
                                   const uint8_t* __restrict__ eflags, const int32_t* __restrict__ vscan, int32_t* __restrict__ tris) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t sy = nz, sx = (int64_t)ny * nz;
  if (p >= sx * nx) return;
  const int cs = cases[p];
  const int nt = c_mc.ntri[cs];
  if (!nt) return;
  int32_t* o = tris + 3 * (int64_t)tscan[p];
  for (int q = 0; q < 3 * nt; ++q) {
    const int e = c_mc.e[cs][q], a = e >> 2, lo = mcgen::edge_lo(e);
    const int64_t pe = p + (lo & 1) * sx + ((lo >> 1) & 1) * sy + ((lo >> 2) & 1);
    o[q] = vscan[pe] + __popc(eflags[pe] & ((1 << a) - 1));
  }
}

template <class F>
static int cub_temp(MeshState& s, F&& run) {
  size_t bytes = 0;
  DMN_CUDA(run(nullptr, bytes));
  uint8_t* tmp = nullptr;
  if (s.temp.get(bytes, &tmp)) return 2;
  DMN_CUDA(run(tmp, bytes));
  return 0;
}

static int exclusive_sum(MeshState& s, const int32_t* in, int32_t* out, int64_t n, cudaStream_t st) {
  return cub_temp(s, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int)n, st); });
}

static int read_back(MeshState& s, int64_t* host, int n, cudaStream_t st) {
  int64_t* d = nullptr;
  if (s.totals.get(4, &d)) return 2;
  DMN_CUDA(cudaMemcpyAsync(host, d, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int mc_count(MeshState& s, const float* grid, int nx, int ny, int nz, float level, int64_t* counts, cudaStream_t st) {
  DMN_CHECK(nx >= 2 && ny >= 2 && nz >= 2, "mc_count: grid %dx%dx%d is smaller than one cell", nx, ny, nz);
  const int64_t n = (int64_t)nx * ny * nz;
  DMN_CHECK(n * MC_MAX_TRI < INT32_MAX, "mc_count: grid of %lld points exceeds the 32-bit vertex / triangle numbering", (long long)n);
  DMN_CHECK(!(level != level), "mc_count: level is NaN");
  s.grid = nullptr;
  uint8_t *ef, *cs;
  int32_t *vc, *vs, *tc, *ts;
  int64_t* tot;
  if (s.eflags.get(n, &ef) || s.cases.get(n, &cs) || s.vcnt.get(n, &vc) || s.vscan.get(n, &vs) || s.tcnt.get(n, &tc) ||
      s.tscan.get(n, &ts) || s.totals.get(4, &tot))
    return 2;
  int32_t* nan_seen = reinterpret_cast<int32_t*>(tot + 3);
  DMN_CUDA(cudaMemsetAsync(nan_seen, 0, sizeof(int32_t), st));
  mc_classify_kernel<<<blocks(n, 256), 256, 0, st>>>(grid, nx, ny, nz, level, ef, vc, cs, tc, nan_seen);
  DMN_LAUNCH_OK();
  if (exclusive_sum(s, vc, vs, n, st) || exclusive_sum(s, tc, ts, n, st)) return 2;
  mc_totals_kernel<<<1, 1, 0, st>>>(vs, vc, ts, tc, n, nan_seen, tot);
  DMN_LAUNCH_OK();
  int64_t h[3];
  if (read_back(s, h, 3, st)) return 2;
  DMN_CHECK(h[2] == 0, "mc_count: the grid holds NaN values");
  s.grid = grid; s.nx = nx; s.ny = ny; s.nz = nz; s.level = level;
  s.nv = h[0]; s.nt = h[1];
  counts[0] = h[0];
  counts[1] = h[1];
  return 0;
}

int mc_emit(MeshState& s, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris, cudaStream_t st) {
  DMN_CHECK(s.grid == grid && s.nx == nx && s.ny == ny && s.nz == nz && s.level == level,
            "mc_emit: call dmnerf_mesh_mc_count on the same grid and level first");
  DMN_CHECK((s.nv == 0 || verts) && (s.nt == 0 || tris), "mc_emit: NULL output");
  const int64_t n = (int64_t)nx * ny * nz;
  uint8_t *ef, *cs;
  int32_t *vs, *ts;
  if (s.eflags.get(n, &ef) || s.cases.get(n, &cs) || s.vscan.get(n, &vs) || s.tscan.get(n, &ts)) return 2;   // as mc_count left them
  if (s.nv) {
    mc_vertex_kernel<<<blocks(n, 256), 256, 0, st>>>(grid, nx, ny, nz, level, ef, vs, verts);
    DMN_LAUNCH_OK();
  }
  if (s.nt) {
    mc_triangle_kernel<<<blocks(n, 256), 256, 0, st>>>(nx, ny, nz, cs, ts, ef, vs, tris);
    DMN_LAUNCH_OK();
  }
  return 0;
}

// ---- scene-space vertices (mesh_generator.py:70-86, trimesh in float64) ------------------------------------------------------
// v / (dim - 1) in float32 (the original divides skimage's float32 vertices), then in float64: (q - 0.5) * 2 * extents / 2,
// then R x + t; rounded once to float32.
__global__ void to_scene_kernel(const float* __restrict__ v, int64_t n, float div, double3 half, double4 r0, double4 r1, double4 r2,
                                float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = ((double)__fdiv_rn(v[3 * i], div) - 0.5) * 2.0 * half.x;
  const double y = ((double)__fdiv_rn(v[3 * i + 1], div) - 0.5) * 2.0 * half.y;
  const double z = ((double)__fdiv_rn(v[3 * i + 2], div) - 0.5) * 2.0 * half.z;
  out[3 * i] = (float)(r0.x * x + r0.y * y + r0.z * z + r0.w);
  out[3 * i + 1] = (float)(r1.x * x + r1.y * y + r1.z * z + r1.w);
  out[3 * i + 2] = (float)(r2.x * x + r2.y * y + r2.z * z + r2.w);
}

int launch_to_scene(const float* v, int64_t n, const double* T16, const double* ext3, int dim, float* out, cudaStream_t st) {
  DMN_CHECK(dim >= 2, "mesh_to_scene: dim must be >= 2");
  if (n == 0) return 0;
  const double3 half = make_double3(ext3[0] / 2.0, ext3[1] / 2.0, ext3[2] / 2.0);
  const double* T = T16;
  to_scene_kernel<<<blocks(n, 256), 256, 0, st>>>(v, n, (float)(dim - 1), half, make_double4(T[0], T[1], T[2], T[3]),
                                                  make_double4(T[4], T[5], T[6], T[7]), make_double4(T[8], T[9], T[10], T[11]), out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---- vertex normals: sum of the unnormalised face cross products of the incident triangles, in triangle order, float64 -----
static int bits_for(int64_t n) {
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < n) ++b;
  return b;
}

__global__ void iota_tri_kernel(int64_t n3, int32_t* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < n3) out[q] = (int32_t)(q / 3);
}

__device__ __forceinline__ int64_t lower_bound(const int32_t* a, int64_t n, int32_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void normals_kernel(const float* __restrict__ v, const int32_t* __restrict__ tris, int64_t nv, const int32_t* __restrict__ vkey,
                               const int32_t* __restrict__ tri_of, int64_t n3, float* __restrict__ normals) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv) return;
  const int64_t lo = lower_bound(vkey, n3, (int32_t)i), hi = lower_bound(vkey, n3, (int32_t)(i + 1));
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (int64_t q = lo; q < hi; ++q) {
    const int32_t* t = tris + 3 * (int64_t)tri_of[q];
    const float* a = v + 3 * (int64_t)t[0];
    const float* b = v + 3 * (int64_t)t[1];
    const float* c = v + 3 * (int64_t)t[2];
    const double ux = (double)b[0] - a[0], uy = (double)b[1] - a[1], uz = (double)b[2] - a[2];
    const double wx = (double)c[0] - a[0], wy = (double)c[1] - a[1], wz = (double)c[2] - a[2];
    sx += uy * wz - uz * wy;
    sy += uz * wx - ux * wz;
    sz += ux * wy - uy * wx;
  }
  const double len = sqrt(sx * sx + sy * sy + sz * sz);
  const double inv = len > 0.0 ? 1.0 / len : 0.0;                // a vertex without area keeps a zero normal
  normals[3 * i] = (float)(sx * inv);
  normals[3 * i + 1] = (float)(sy * inv);
  normals[3 * i + 2] = (float)(sz * inv);
}

int mesh_normals(MeshState& s, const float* v, int64_t nv, const int32_t* tris, int64_t nt, float* normals, cudaStream_t st) {
  DMN_CHECK(nv >= 0 && nt >= 0 && nv < INT32_MAX && 3 * nt < INT32_MAX, "mesh_normals: bad sizes");
  if (nv == 0) return 0;
  const int64_t n3 = 3 * nt;
  int32_t *kout, *vin, *vout;
  if (s.keys_out.get(n3, &kout) || s.vals_in.get(n3, &vin) || s.vals_out.get(n3, &vout)) return 2;
  if (n3) {
    iota_tri_kernel<<<blocks(n3, 256), 256, 0, st>>>(n3, vin);
    DMN_LAUNCH_OK();
    const int eb = bits_for(nv);
    // stable radix sort by vertex: every vertex's incident triangles in increasing triangle order (deterministic sums)
    if (cub_temp(s, [&](void* tmp, size_t& bytes) {
          return cub::DeviceRadixSort::SortPairs(tmp, bytes, tris, kout, vin, vout, (int)n3, 0, eb, st);
        }))
      return 2;
  }
  normals_kernel<<<blocks(nv, 128), 128, 0, st>>>(v, tris, nv, kout, vout, n3, normals);
  DMN_LAUNCH_OK();
  return 0;
}

// ---- edge-connected triangle clusters (open3d cluster_connected_triangles): union-find over triangles sharing an edge -------
__global__ void edge_keys_kernel(const int32_t* __restrict__ tris, int64_t nt, int64_t nv, uint64_t* __restrict__ keys,
                                 int32_t* __restrict__ vals) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= 3 * nt) return;
  const int64_t t = q / 3;
  const int m = (int)(q % 3);
  const uint64_t a = (uint32_t)tris[3 * t + m], b = (uint32_t)tris[3 * t + (m + 1) % 3];
  keys[q] = (a < b ? a : b) * (uint64_t)nv + (a < b ? b : a);
  vals[q] = (int32_t)t;
}

__global__ void iota_kernel(int64_t n, int32_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int32_t)i;
}

// parent[x] <= x always (a root is hooked under the smaller root), so every root is the smallest triangle of its cluster
__device__ int32_t uf_find(volatile int32_t* parent, int32_t x) {
  while (true) {
    const int32_t p = parent[x];
    if (p == x) return x;
    const int32_t gp = parent[p];
    if (gp != p) parent[x] = gp;                                      // path halving
    x = p;
  }
}

__global__ void union_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, int64_t n3, int32_t* parent) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q == 0 || q >= n3 || keys[q] != keys[q - 1]) return;
  int32_t a = vals[q - 1], b = vals[q];
  while (true) {
    a = uf_find(parent, a);
    b = uf_find(parent, b);
    if (a == b) return;
    if (a < b) { const int32_t x = a; a = b; b = x; }
    if (atomicCAS(parent + a, a, b) == a) return;
  }
}

__global__ void roots_kernel(int64_t nt, int32_t* parent, int32_t* __restrict__ cluster, int32_t* __restrict__ size) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nt) return;
  const int32_t r = uf_find(parent, (int32_t)t);
  cluster[t] = r;
  atomicAdd(size + r, 1);
}

__global__ void cluster_size_kernel(int64_t nt, const int32_t* __restrict__ cluster, const int32_t* __restrict__ size,
                                    int32_t* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nt) out[t] = size[cluster[t]];
}

int mesh_clusters(MeshState& s, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size,
                  cudaStream_t st) {
  DMN_CHECK(nt >= 0 && nv >= 0 && 3 * nt < INT32_MAX && nv < INT32_MAX, "mesh_clusters: bad sizes");
  if (nt == 0) return 0;
  const int64_t n3 = 3 * nt;
  uint64_t *kin, *kout;
  int32_t *vin, *vout, *parent, *size;
  if (s.keys_in.get(n3, &kin) || s.keys_out.get(n3, &kout) || s.vals_in.get(n3, &vin) || s.vals_out.get(n3, &vout) ||
      s.parent.get(nt, &parent) || s.size.get(nt, &size))
    return 2;
  edge_keys_kernel<<<blocks(n3, 256), 256, 0, st>>>(tris, nt, nv, kin, vin);
  DMN_LAUNCH_OK();
  const int eb = bits_for(nv * nv);
  if (cub_temp(s, [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, kin, kout, vin, vout, (int)n3, 0, eb, st);
      }))
    return 2;
  iota_kernel<<<blocks(nt, 256), 256, 0, st>>>(nt, parent);
  DMN_LAUNCH_OK();
  union_kernel<<<blocks(n3, 256), 256, 0, st>>>(kout, vout, n3, parent);
  DMN_LAUNCH_OK();
  DMN_CUDA(cudaMemsetAsync(size, 0, nt * sizeof(int32_t), st));
  roots_kernel<<<blocks(nt, 256), 256, 0, st>>>(nt, parent, cluster, size);
  DMN_LAUNCH_OK();
  cluster_size_kernel<<<blocks(nt, 256), 256, 0, st>>>(nt, cluster, size, cluster_size);
  DMN_LAUNCH_OK();
  return 0;
}

// ---- cleanup (clean_mesh: remove_triangles_by_mask + remove_unreferenced_vertices), order-preserving compaction ------------
__global__ void keep_kernel(const int32_t* __restrict__ csize, int64_t nt, int min_cluster, int32_t* __restrict__ keep) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nt) keep[t] = csize[t] >= min_cluster ? 1 : 0;
}

__global__ void mark_vertices_kernel(const int32_t* __restrict__ tris, const int32_t* __restrict__ keep, int64_t nt, int32_t* vref) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q < 3 * nt && keep[q / 3]) vref[tris[q]] = 1;
}

__global__ void compact_tris_kernel(const int32_t* __restrict__ tris, const int32_t* __restrict__ keep, const int32_t* __restrict__ tpos,
                                    const int32_t* __restrict__ vpos, int64_t nt, int32_t* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= 3 * nt || !keep[q / 3]) return;
  out[3 * (int64_t)tpos[q / 3] + q % 3] = vpos[tris[q]];
}

__global__ void compact_verts_kernel(const float* __restrict__ v, const float* __restrict__ nrm, const int32_t* __restrict__ vref,
                                     const int32_t* __restrict__ vpos, int64_t nv, float* __restrict__ ov, float* __restrict__ on) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nv || !vref[i]) return;
  const int64_t o = vpos[i];
  for (int c = 0; c < 3; ++c) {
    ov[3 * o + c] = v[3 * i + c];
    if (on) on[3 * o + c] = nrm[3 * i + c];
  }
}

__global__ void clean_totals_kernel(const int32_t* vref, const int32_t* vpos, int64_t nv, const int32_t* keep, const int32_t* tpos,
                                    int64_t nt, int64_t* out) {
  out[0] = nv ? (int64_t)vpos[nv - 1] + vref[nv - 1] : 0;
  out[1] = nt ? (int64_t)tpos[nt - 1] + keep[nt - 1] : 0;
}

int mesh_clean(MeshState& s, const float* v, const float* nrm, int64_t nv, const int32_t* tris, int64_t nt, const int32_t* csize,
               int min_cluster, float* out_v, float* out_n, int32_t* out_t, int64_t* counts, cudaStream_t st) {
  DMN_CHECK(nt >= 0 && nv >= 0 && 3 * nt < INT32_MAX && nv < INT32_MAX, "mesh_clean: bad sizes");
  counts[0] = counts[1] = 0;
  if (nt == 0 && nv == 0) return 0;
  int32_t *keep, *tpos, *vref, *vpos;
  int64_t* tot;
  if (s.vcnt.get(nt + 1, &keep) || s.vscan.get(nt + 1, &tpos) || s.tcnt.get(nv + 1, &vref) || s.tscan.get(nv + 1, &vpos) ||
      s.totals.get(4, &tot))
    return 2;
  s.grid = nullptr;                             // the marching-cubes scans share these buffers
  if (nt) {
    keep_kernel<<<blocks(nt, 256), 256, 0, st>>>(csize, nt, min_cluster, keep);
    DMN_LAUNCH_OK();
    if (exclusive_sum(s, keep, tpos, nt, st)) return 2;
  }
  if (nv) {
    DMN_CUDA(cudaMemsetAsync(vref, 0, nv * sizeof(int32_t), st));
    if (nt) {
      mark_vertices_kernel<<<blocks(3 * nt, 256), 256, 0, st>>>(tris, keep, nt, vref);
      DMN_LAUNCH_OK();
    }
    if (exclusive_sum(s, vref, vpos, nv, st)) return 2;
    compact_verts_kernel<<<blocks(nv, 256), 256, 0, st>>>(v, nrm, vref, vpos, nv, out_v, out_n);
    DMN_LAUNCH_OK();
  }
  if (nt) {
    compact_tris_kernel<<<blocks(3 * nt, 256), 256, 0, st>>>(tris, keep, tpos, vpos, nt, out_t);
    DMN_LAUNCH_OK();
  }
  clean_totals_kernel<<<1, 1, 0, st>>>(vref, vpos, nv, keep, tpos, nt, tot);
  DMN_LAUNCH_OK();
  return read_back(s, counts, 2, st);
}

// ---- label rays (mesh_generator.py:106-113) and argmax -------------------------------------------------------------------
// rays_d = -normal and the vertex, both with axes (0, 2, 1) and y negated; rays_o = v - rays_d * 0.03 * near (fp32, in that order)
__global__ void label_rays_kernel(const float* __restrict__ v, const float* __restrict__ nrm, int64_t n, float near_z,
                                  float* __restrict__ ro, float* __restrict__ rd) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float d[3] = {-nrm[3 * i], nrm[3 * i + 2], -nrm[3 * i + 1]};
  const float p[3] = {v[3 * i], -v[3 * i + 2], v[3 * i + 1]};
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    rd[3 * i + c] = d[c];
    ro[3 * i + c] = __fsub_rn(p[c], __fmul_rn(__fmul_rn(d[c], 0.03f), near_z));
  }
}

int launch_label_rays(const float* v, const float* nrm, int64_t n, float near_z, float* ro, float* rd, cudaStream_t st) {
  if (n == 0) return 0;
  label_rays_kernel<<<blocks(n, 256), 256, 0, st>>>(v, nrm, n, near_z, ro, rd);
  DMN_LAUNCH_OK();
  return 0;
}

// torch.argmax(x, -1): first maximum; a NaN counts as the maximum
__global__ void argmax_rows_kernel(const float* __restrict__ x, int64_t n, int c, int64_t* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* r = x + i * c;
  float best = r[0];
  int bi = 0;
  for (int k = 1; k < c && best == best; ++k) {
    const float y = r[k];
    if (y > best || y != y) { best = y; bi = k; }
  }
  out[i] = bi;
}

int launch_argmax_rows(const float* x, int64_t n, int c, int64_t* out, cudaStream_t st) {
  if (n == 0) return 0;
  argmax_rows_kernel<<<blocks(n, 256), 256, 0, st>>>(x, n, c, out);
  DMN_LAUNCH_OK();
  return 0;
}

// ---- meshing an edited scene (DESIGN.md, "Meshing an edited scene") ---------------------------------------------------------
// Every fp64 expression below is written with one rounding per operation (no contraction), so that a numpy restatement
// (oracle/edit_sweep_oracle.py) takes the same decisions.

// The grid's index map of objects.grid_affine: p = A idx + b with A = S R diag(h), b = S (t - R e), h = extents / (dim - 1),
// e = extents / 2 and S the axis swap (x, y, z) -> (x, -z, y); inv = diag(1 / h) R^-1 S^T, R^-1 = adj(R) / det(R).
static void grid_index_map(const double* T, const double* ext, int dim, double inv[9], double b[3]) {
  const double R[3][3] = {{T[0], T[1], T[2]}, {T[4], T[5], T[6]}, {T[8], T[9], T[10]}};
  double adj[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const int i1 = (j + 1) % 3, i2 = (j + 2) % 3, j1 = (i + 1) % 3, j2 = (i + 2) % 3;
      adj[i][j] = R[i1][j1] * R[i2][j2] - R[i1][j2] * R[i2][j1];       // cofactor (j, i)
    }
  const double det = (R[0][0] * adj[0][0] + R[0][1] * adj[1][0]) + R[0][2] * adj[2][0];
  double w[3];
  for (int r = 0; r < 3; ++r)
    w[r] = T[4 * r + 3] - ((R[r][0] * (ext[0] / 2.0) + R[r][1] * (ext[1] / 2.0)) + R[r][2] * (ext[2] / 2.0));
  b[0] = w[0]; b[1] = -w[2]; b[2] = w[1];
  for (int a = 0; a < 3; ++a) {
    const double scale = (double)(dim - 1) / ext[a];
    const double ri[3] = {adj[a][0] / det, adj[a][1] / det, adj[a][2] / det};
    // column c of S^T: S^T e_0 = e_0, S^T e_1 = -e_2, S^T e_2 = e_1
    inv[3 * a] = scale * ri[0];
    inv[3 * a + 1] = scale * -ri[2];
    inv[3 * a + 2] = scale * ri[1];
  }
}

int edit_move_from_abi(const dmnerf_edit_move& d, const double* T16, const double* ext3, int dim, int ins_num, EditMove& m,
                       const char* who, int i) {
  memset(&m, 0, sizeof(m));
  DMN_CHECK(d.label >= 0 && d.label <= ins_num, "%s: move %d: label %d outside [0, %d]", who, i, d.label, ins_num);
  for (int k = 0; k < 12; ++k) DMN_CHECK(std::isfinite(d.trans[k]), "%s: move %d: the transformation is not finite", who, i);
  const double* t = d.trans;
  const double det = t[0] * (t[5] * t[10] - t[6] * t[9]) - t[1] * (t[4] * t[10] - t[6] * t[8]) + t[2] * (t[4] * t[9] - t[5] * t[8]);
  DMN_CHECK(det > 0.0, "%s: move %d: the transformation has det %g <= 0 (a reflection or a degenerate matrix)", who, i, det);
  const int* bx = d.box;
  const bool empty = bx[0] == 1 && bx[1] == 0 && bx[2] == 1 && bx[3] == 0 && bx[4] == 1 && bx[5] == 0;
  if (!empty)
    for (int a = 0; a < 3; ++a)
      DMN_CHECK(bx[2 * a] >= 0 && bx[2 * a] <= bx[2 * a + 1] && bx[2 * a + 1] <= dim - 1,
                "%s: move %d: box [%d, %d] x [%d, %d] x [%d, %d] is inverted or outside the grid [0, %d]", who, i, bx[0], bx[1], bx[2],
                bx[3], bx[4], bx[5], dim - 1);
  if (piece_region(d.piece, d.label, m.piece, who, i)) return 1;
  memcpy(m.trans, d.trans, sizeof(m.trans));
  grid_index_map(T16, ext3, dim, m.inv, m.b);
  for (int a = 0; a < 3; ++a) { m.lo[a] = bx[2 * a]; m.hi[a] = bx[2 * a + 1]; }
  m.label = d.label;
  m.rest_drop = d.rest_drop ? 1 : 0;
  m.empty = empty ? 1 : 0;
  return 0;
}

// One thread per grid point of the slab: its target t = trans p (fp64, rounded once to fp32) and whether the nearest grid index
// of t, rint(A^-1 (t - b)), lies in the box (an fp32 sweep point maps to its own index, also on the grid's faces).
__global__ void edit_target_kernel(const GridXform g, const EditMove m, int64_t begin, int64_t count, float* __restrict__ tgt,
                                   int32_t* __restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float p[3];
  sweep_point(g, begin + i, p);
  float t[3];
  double dt[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* r = m.trans + 4 * a;
    const double v = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], (double)p[0]), __dmul_rn(r[1], (double)p[1])),
                                         __dmul_rn(r[2], (double)p[2])), r[3]);
    t[a] = __double2float_rn(v);
    dt[a] = __dsub_rn((double)t[a], m.b[a]);
  }
  bool in = !m.empty;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double* row = m.inv + 3 * a;
    const double u = __dadd_rn(__dadd_rn(__dmul_rn(row[0], dt[0]), __dmul_rn(row[1], dt[1])), __dmul_rn(row[2], dt[2]));
    const double i = rint(u);                                     // the nearest grid index, half to even
    in = in && i >= m.lo[a] && i <= m.hi[a];
  }
  tgt[3 * i] = t[0];
  tgt[3 * i + 1] = t[1];
  tgt[3 * i + 2] = t[2];
  flag[i] = in ? 1 : 0;
}

// order-keeping compaction of the boxed targets (pos: exclusive scan of flag)
__global__ void edit_compact_kernel(const float* __restrict__ tgt, const int32_t* __restrict__ flag, const int32_t* __restrict__ pos,
                                    int64_t count, float* __restrict__ pts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count || !flag[i]) return;
  const int64_t o = pos[i];
  pts[3 * o] = tgt[3 * i];
  pts[3 * o + 1] = tgt[3 * i + 1];
  pts[3 * o + 2] = tgt[3 * i + 2];
}

__global__ void edit_count_kernel(const int32_t* flag, const int32_t* pos, int64_t count, int64_t* out) {
  out[0] = (int64_t)pos[count - 1] + flag[count - 1];
}

// One thread per grid point of the slab: take the target's (occ, label), or vacate the point.
__global__ void edit_apply_kernel(const GridXform g, const EditMove m, int64_t begin, int64_t count, const int32_t* __restrict__ flag,
                                  const int32_t* __restrict__ pos, const float* __restrict__ tgt, const float* __restrict__ raw, int c,
                                  float voxel, float level, float* __restrict__ occ, int16_t* __restrict__ labels) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int64_t p = begin + i;
  const float o = occ[p];
  const int l = labels[p];
  const bool has_piece = m.piece.bits != nullptr;
  if (flag[i]) {
    const float* r = raw + (int64_t)pos[i] * c;
    const int lt = argmax_sigmoid(r + 4, c - 4);
    const float ot = occupancy_of(r[3], voxel);
    if (lt == m.label && (ot > level || o <= level) &&
        (!has_piece || !region_drops(m.piece, m.label, tgt[3 * i], tgt[3 * i + 1], tgt[3 * i + 2]))) {
      occ[p] = ot;
      labels[p] = (int16_t)m.label;
      return;
    }
  }
  if (l == m.label && o > level) {
    bool in_piece = true;
    if (has_piece) {
      float q[3];
      sweep_point(g, p, q);
      in_piece = !region_drops(m.piece, m.label, q[0], q[1], q[2]);
    }
    if (in_piece || m.rest_drop) occ[p] = 0.0f;
  }
}

int edit_targets(MeshState& s, const double* T16, const double* ext3, int dim, const EditMove& m, int64_t begin, int64_t count,
                 float* pts, int64_t* n_eval, cudaStream_t st) {
  *n_eval = 0;
  DMN_CHECK(count >= 1 && count < INT32_MAX, "edit_targets: slab of %lld points outside [1, 2^31)", (long long)count);
  float* tgt;
  int32_t *flag, *pos;
  int64_t* tot;
  if (s.edit_t.get((size_t)count * 3, &tgt) || s.edit_flag.get((size_t)count, &flag) || s.edit_pos.get((size_t)count, &pos) ||
      s.totals.get(4, &tot))
    return 2;
  const GridXform g = make_xform(T16, ext3, dim);
  edit_target_kernel<<<blocks(count, 256), 256, 0, st>>>(g, m, begin, count, tgt, flag);
  DMN_LAUNCH_OK();
  if (exclusive_sum(s, flag, pos, count, st)) return 2;
  edit_count_kernel<<<1, 1, 0, st>>>(flag, pos, count, tot);
  DMN_LAUNCH_OK();
  int64_t n = 0;
  if (read_back(s, &n, 1, st)) return 2;
  if (n) {
    edit_compact_kernel<<<blocks(count, 256), 256, 0, st>>>(tgt, flag, pos, count, pts);
    DMN_LAUNCH_OK();
  }
  *n_eval = n;
  return 0;
}

int edit_apply(MeshState& s, const double* T16, const double* ext3, int dim, const EditMove& m, int64_t begin, int64_t count,
               const float* raw, int c, float voxel, float level, float* occ, int16_t* labels, cudaStream_t st) {
  float* tgt;
  int32_t *flag, *pos;
  if (s.edit_t.get((size_t)count * 3, &tgt) || s.edit_flag.get((size_t)count, &flag) || s.edit_pos.get((size_t)count, &pos))
    return 2;                                                     // as edit_targets left them
  edit_apply_kernel<<<blocks(count, 256), 256, 0, st>>>(make_xform(T16, ext3, dim), m, begin, count, flag, pos, tgt, raw, c, voxel,
                                                        level, occ, labels);
  DMN_LAUNCH_OK();
  return 0;
}

// The label of the nearest solid grid point closer than 2 to an index-space vertex: the 4^3 block floor(v) - 1 .. floor(v) + 2
// holds every grid point closer than 2; it is walked in ascending linear index and only a strictly smaller squared distance
// replaces the best, so an exact tie goes to the lowest index.
__global__ void vertex_labels_kernel(const float* __restrict__ v, int64_t n, const float* __restrict__ occ,
                                     const int16_t* __restrict__ labels, int dim, float level, int16_t* __restrict__ out) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const float x[3] = {v[3 * q], v[3 * q + 1], v[3 * q + 2]};
  int lo[3], hi[3];
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ok = ok && x[a] > -2.0f && x[a] < (float)(dim + 1);           // also false for NaN
    const int f = ok ? (int)floorf(x[a]) : 0;
    lo[a] = max(f - 1, 0);
    hi[a] = min(f + 2, dim - 1);
  }
  int best = -1;
  double bd = 4.0;
  if (ok) {
    for (int i = lo[0]; i <= hi[0]; ++i) {
      const double dx = __dsub_rn((double)x[0], (double)i);
      for (int j = lo[1]; j <= hi[1]; ++j) {
        const double dy = __dsub_rn((double)x[1], (double)j);
        const double dxy = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        for (int k = lo[2]; k <= hi[2]; ++k) {
          const double dz = __dsub_rn((double)x[2], (double)k);
          const double d2 = __dadd_rn(dxy, __dmul_rn(dz, dz));
          const int64_t p = ((int64_t)i * dim + j) * dim + k;
          if (d2 < bd && occ[p] > level) { bd = d2; best = labels[p]; }
        }
      }
    }
  }
  out[q] = (int16_t)best;
}

int launch_vertex_labels(const float* v, int64_t n, const float* occ, const int16_t* labels, int dim, float level, int16_t* out,
                         cudaStream_t st) {
  DMN_CHECK(n >= 0, "mesh_vertex_labels: negative vertex count");
  DMN_CHECK(dim >= 2 && dim <= 2048, "mesh_vertex_labels: dim %d out of range [2, 2048]", dim);
  DMN_CHECK(std::isfinite(level), "mesh_vertex_labels: level is not finite");
  DMN_CHECK(occ && labels && (n == 0 || (v && out)), "mesh_vertex_labels: NULL argument");
  if (n == 0) return 0;
  vertex_labels_kernel<<<blocks(n, 256), 256, 0, st>>>(v, n, occ, labels, dim, level, out);
  DMN_LAUNCH_OK();
  return 0;
}

}  // namespace dmnerf
