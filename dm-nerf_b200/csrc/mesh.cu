// Mesh extraction, tools/mesh_generator.py + tools/visualizer.py of the original project: query grid of the occupancy sweep and
// its epilogue, marching cubes on a caller-provided grid, scene-space vertices, area-weighted vertex normals, edge-connected
// triangle clusters, small-cluster removal and the per-vertex label rays.  Conventions: DESIGN.md, "Mesh extraction".
#include <cub/cub.cuh>

#include "common.cuh"

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

// ---- device buffers of the mesh entry points (grow-only, owned by the context) ---------------------------------------------
struct MeshState {
  enum { EFLAGS, CASES, VCNT, VSCAN, TCNT, TSCAN, TEMP, TOTALS, KEYS_IN, KEYS_OUT, VALS_IN, VALS_OUT, PARENT, SIZE, N_BUF };
  void* p[N_BUF] = {};
  size_t cap[N_BUF] = {};
  // what the last marching-cubes count pass classified (mc_emit must see the same grid)
  const float* grid = nullptr;
  int nx = 0, ny = 0, nz = 0;
  float level = 0.f;
  int64_t nv = -1, nt = -1;
  template <class T>
  int get(int i, size_t n, T** out) {
    const size_t bytes = n * sizeof(T) + 16;
    if (bytes > cap[i]) {
      if (p[i]) DMN_CUDA(cudaFree(p[i]));
      p[i] = nullptr; cap[i] = 0;
      DMN_CUDA(cudaMalloc(&p[i], bytes + bytes / 4));
      cap[i] = bytes + bytes / 4;
    }
    *out = static_cast<T*>(p[i]);
    return 0;
  }
};

void mesh_state_free(MeshState* s) {
  if (!s) return;
  for (void* q : s->p) if (q) cudaFree(q);
  delete s;
}

static MeshState* state(MeshState** s) {
  if (!*s) *s = new MeshState();
  return *s;
}

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
__global__ void grid_points_kernel(GridXform g, int64_t begin, int64_t count, float* __restrict__ pts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int64_t p = begin + i, d = g.dim;
  const float q[3] = {__fmul_rn(linspace_m11((int)(p / (d * d)), g), g.s[0]), __fmul_rn(linspace_m11((int)((p / d) % d), g), g.s[1]),
                      __fmul_rn(linspace_m11((int)(p % d), g), g.s[2])};
  float w[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const float* row = g.r + 4 * r;
    w[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(row[0], q[0]), __fmul_rn(row[1], q[1])), __fmul_rn(row[2], q[2])), row[3]);
  }
  pts[3 * i] = w[0];
  pts[3 * i + 1] = -w[2];
  pts[3 * i + 2] = w[1];
}

int launch_grid_points(const double* T16, const double* ext3, int dim, int64_t begin, int64_t count, float* pts, cudaStream_t st) {
  DMN_CHECK(dim >= 2 && dim <= 2048, "grid_points: dim %d out of range [2, 2048]", dim);
  DMN_CHECK(begin >= 0 && count >= 0 && begin + count <= (int64_t)dim * dim * dim, "grid_points: range outside the grid");
  if (count == 0) return 0;
  GridXform g;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) g.r[4 * r + c] = (float)T16[4 * r + c];
  for (int a = 0; a < 3; ++a) g.s[a] = (float)(ext3[a] / 2.0);
  g.step = 2.0f / (float)(dim - 1);
  g.dim = dim;
  grid_points_kernel<<<blocks(count, 256), 256, 0, st>>>(g, begin, count, pts);
  DMN_LAUNCH_OK();
  return 0;
}

// mesh_generator.py:51-62: occ = 1 - exp(-relu(sigma) * voxel), sigma = channel 3 of the network output [n, c]
__global__ void occupancy_kernel(const float* __restrict__ raw, int64_t n, int c, float voxel, float* __restrict__ occ) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float a = raw[i * c + 3];
  const float r = a > 0.f ? a : (a != a ? a : 0.f);           // torch.relu keeps NaN
  occ[i] = __fsub_rn(1.0f, expf(__fmul_rn(-r, voxel)));
}

int launch_occupancy(const float* raw, int64_t n, int c, float voxel, float* occ, cudaStream_t st) {
  if (n == 0) return 0;
  occupancy_kernel<<<blocks(n, 256), 256, 0, st>>>(raw, n, c, voxel, occ);
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
static int cub_temp(MeshState* s, F&& run) {
  size_t bytes = 0;
  DMN_CUDA(run(nullptr, bytes));
  uint8_t* tmp = nullptr;
  if (s->get(MeshState::TEMP, bytes, &tmp)) return 2;
  DMN_CUDA(run(tmp, bytes));
  return 0;
}

static int exclusive_sum(MeshState* s, const int32_t* in, int32_t* out, int64_t n, cudaStream_t st) {
  return cub_temp(s, [&](void* tmp, size_t& bytes) { return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int)n, st); });
}

static int read_back(MeshState* s, int64_t* host, int n, cudaStream_t st) {
  int64_t* d = nullptr;
  if (s->get(MeshState::TOTALS, 4, &d)) return 2;
  DMN_CUDA(cudaMemcpyAsync(host, d, n * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  DMN_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int mc_count(MeshState** sp, const float* grid, int nx, int ny, int nz, float level, int64_t* counts, cudaStream_t st) {
  DMN_CHECK(nx >= 2 && ny >= 2 && nz >= 2, "mc_count: grid %dx%dx%d is smaller than one cell", nx, ny, nz);
  const int64_t n = (int64_t)nx * ny * nz;
  DMN_CHECK(n * MC_MAX_TRI < INT32_MAX, "mc_count: grid of %lld points exceeds the 32-bit vertex / triangle numbering", (long long)n);
  DMN_CHECK(!(level != level), "mc_count: level is NaN");
  MeshState* s = state(sp);
  s->grid = nullptr;
  uint8_t *ef, *cs;
  int32_t *vc, *vs, *tc, *ts;
  int64_t* tot;
  if (s->get(MeshState::EFLAGS, n, &ef) || s->get(MeshState::CASES, n, &cs) || s->get(MeshState::VCNT, n, &vc) ||
      s->get(MeshState::VSCAN, n, &vs) || s->get(MeshState::TCNT, n, &tc) || s->get(MeshState::TSCAN, n, &ts) ||
      s->get(MeshState::TOTALS, 4, &tot))
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
  s->grid = grid; s->nx = nx; s->ny = ny; s->nz = nz; s->level = level;
  s->nv = h[0]; s->nt = h[1];
  counts[0] = h[0];
  counts[1] = h[1];
  return 0;
}

int mc_emit(MeshState* s, const float* grid, int nx, int ny, int nz, float level, float* verts, int32_t* tris, cudaStream_t st) {
  DMN_CHECK(s && s->grid == grid && s->nx == nx && s->ny == ny && s->nz == nz && s->level == level,
            "mc_emit: call dmnerf_mesh_mc_count on the same grid and level first");
  DMN_CHECK((s->nv == 0 || verts) && (s->nt == 0 || tris), "mc_emit: NULL output");
  const int64_t n = (int64_t)nx * ny * nz;
  auto* ef = static_cast<const uint8_t*>(s->p[MeshState::EFLAGS]);
  auto* cs = static_cast<const uint8_t*>(s->p[MeshState::CASES]);
  auto* vs = static_cast<const int32_t*>(s->p[MeshState::VSCAN]);
  auto* ts = static_cast<const int32_t*>(s->p[MeshState::TSCAN]);
  if (s->nv) {
    mc_vertex_kernel<<<blocks(n, 256), 256, 0, st>>>(grid, nx, ny, nz, level, ef, vs, verts);
    DMN_LAUNCH_OK();
  }
  if (s->nt) {
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

int mesh_normals(MeshState** sp, const float* v, int64_t nv, const int32_t* tris, int64_t nt, float* normals, cudaStream_t st) {
  DMN_CHECK(nv >= 0 && nt >= 0 && nv < INT32_MAX && 3 * nt < INT32_MAX, "mesh_normals: bad sizes");
  if (nv == 0) return 0;
  MeshState* s = state(sp);
  const int64_t n3 = 3 * nt;
  int32_t *kout, *vin, *vout;
  if (s->get(MeshState::KEYS_OUT, n3, &kout) || s->get(MeshState::VALS_IN, n3, &vin) || s->get(MeshState::VALS_OUT, n3, &vout)) return 2;
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

int mesh_clusters(MeshState** sp, const int32_t* tris, int64_t nt, int64_t nv, int32_t* cluster, int32_t* cluster_size,
                  cudaStream_t st) {
  DMN_CHECK(nt >= 0 && nv >= 0 && 3 * nt < INT32_MAX && nv < INT32_MAX, "mesh_clusters: bad sizes");
  if (nt == 0) return 0;
  MeshState* s = state(sp);
  const int64_t n3 = 3 * nt;
  uint64_t *kin, *kout;
  int32_t *vin, *vout, *parent, *size;
  if (s->get(MeshState::KEYS_IN, n3, &kin) || s->get(MeshState::KEYS_OUT, n3, &kout) || s->get(MeshState::VALS_IN, n3, &vin) ||
      s->get(MeshState::VALS_OUT, n3, &vout) || s->get(MeshState::PARENT, nt, &parent) || s->get(MeshState::SIZE, nt, &size))
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

int mesh_clean(MeshState** sp, const float* v, const float* nrm, int64_t nv, const int32_t* tris, int64_t nt, const int32_t* csize,
               int min_cluster, float* out_v, float* out_n, int32_t* out_t, int64_t* counts, cudaStream_t st) {
  DMN_CHECK(nt >= 0 && nv >= 0 && 3 * nt < INT32_MAX && nv < INT32_MAX, "mesh_clean: bad sizes");
  MeshState* s = state(sp);
  counts[0] = counts[1] = 0;
  if (nt == 0 && nv == 0) return 0;
  int32_t *keep, *tpos, *vref, *vpos;
  int64_t* tot;
  if (s->get(MeshState::VCNT, nt + 1, &keep) || s->get(MeshState::VSCAN, nt + 1, &tpos) || s->get(MeshState::TCNT, nv + 1, &vref) ||
      s->get(MeshState::TSCAN, nv + 1, &vpos) || s->get(MeshState::TOTALS, 4, &tot))
    return 2;
  s->grid = nullptr;                            // the marching-cubes scans share these buffers
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

}  // namespace dmnerf
