// Per-ray device primitives shared by the stand-alone stage kernels and the fused render kernels:
// warp-scan transmittance composite, inverse-CDF sampling, rank sort, positional encoding.
// One warp owns one ray; `lane` is threadIdx.x & 31.  All arithmetic is fp32 with the accurate
// libdevice sinf/cosf/expf (no fast-math): sin/cos arguments reach 2^9 * |x| ~ 1e4.
#pragma once
#include "common.cuh"

namespace dmnerf {

constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// The per-sample object label: torch.argmax(torch.sigmoid(v[0:n])), first maximum wins (manipulator.py:19-25, 45-53).  The one
// label rule of the library: the exchanger, the object-selected composites and the selected occupancy sweep all call this, so
// ties from fp32 saturation of the sigmoid resolve the same way everywhere.  `start`: the channel the walk begins at, wrapping
// around (the fused kernel staggers it across the lanes of a warp to spread shared-memory banks); the result does not depend on
// it for NaN-free logits: the largest sigmoid wins, the lowest channel among equal ones.
__device__ __forceinline__ int argmax_sigmoid(const float* __restrict__ v, int n, int start = 0) {
  int best = start, k = start;
  float bv = sigmoidf_acc(v[start]);
  for (int i = 1; i < n; ++i) {
    if (++k == n) k = 0;
    const float x = sigmoidf_acc(v[k]);
    if (x > bv || (x == bv && k < best)) { bv = x; best = k; }
  }
  return best;
}

// Region selection (DESIGN.md, "Region selection").  The bit of the grid point nearest to p: u_a = ((M_a0 p0 + M_a1 p1) +
// M_a2 p2) + c_a with every operation rounded once, i_a = rint(u_a); 1 or 0 when every i_a is in [0, dim - 1], -1 otherwise
// (NaN and inf included).  The render kernels, the stage composite and dmnerf_region_contains all call this one function.
__device__ __forceinline__ int region_bit(const Region& r, float p0, float p1, float p2) {
  int idx[3];
  const float top = (float)(r.dim - 1);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float* m = r.map + 4 * a;
    const float u = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], p0), __fmul_rn(m[1], p1)), __fmul_rn(m[2], p2)), m[3]);
    const float i = rintf(u);
    if (!(i >= 0.0f && i <= top)) return -1;
    idx[a] = (int)i;
  }
  const int v = (idx[0] * r.dim + idx[1]) * r.dim + idx[2];
  return (int)((__ldg(r.bits + (v >> 5)) >> (v & 31)) & 1u);
}

// Does the region give a sample with label `label` at p = o + d z alpha = 0?  Only for a label in r.applies: inside the grid
// when its bit is 0, outside it unless r.outside_keep.
__device__ __forceinline__ bool region_drops(const Region& r, int label, float p0, float p1, float p2) {
  if (!obj_kept(r.applies, label)) return false;
  const int b = region_bit(r, p0, p1, p2);
  return b == 0 || (b < 0 && !r.outside_keep);
}

// Object appearance (DESIGN.md, "Object appearance").  Row `label` of the table (APPEARANCE_ROW floats: the colour map [M | b],
// row-major 3x4, then the density scale s) applied to a kept sample: sg (its max(sigma, 0)) becomes s sg, and each channel of
// its sigmoid colour c becomes min(max(((M_a0 c0 + M_a1 c1) + M_a2 c2) + b_a, 0), 1), every operation rounded once.  The fused
// render kernels and the stage composite call this one function; a caller that needs only one of the two results discards the
// other, and the compiler drops that half.
__device__ __forceinline__ void appearance_apply(const float* __restrict__ table, int label, float& sg, float c[3]) {
  const float4* row = reinterpret_cast<const float4*>(table + APPEARANCE_ROW * label);
  sg = __fmul_rn(__ldg(row + 3).x, sg);
  const float4 m[3] = {__ldg(row), __ldg(row + 1), __ldg(row + 2)};
  const float c0 = c[0], c1 = c[1], c2 = c[2];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float u = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[a].x, c0), __fmul_rn(m[a].y, c1)), __fmul_rn(m[a].z, c2)), m[a].w);
    c[a] = fminf(fmaxf(u, 0.0f), 1.0f);
  }
}

// The sample point of depth z on the ray (o, d), as the network prologue computes it.
__device__ __forceinline__ void ray_point(const float* o, const float* d, float z, float p[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[c], __fmul_rn(d[c], z));
}

// [x, sin(2^k x), cos(2^k x)]_k for one 3-vector; out has 3 + 6*L entries (networks/dm_nerf.py:37-38).
__device__ __forceinline__ void posenc_one_freq(const float v[3], int k, float* out /* 6 */) {
  const float f = (float)(1 << k);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float s, co;
    sincosf(v[c] * f, &s, &co);
    out[c] = s;
    out[3 + c] = co;
  }
}

// Multiplicative inclusive warp scan.
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    float o = __shfl_up_sync(FULL, v, d);
    if (lane >= d) v *= o;
  }
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
  return v;
}

// sigma -> alpha -> exclusive-product transmittance -> weights for one ray (networks/render.py:7-18).
//   sigma(i), zval(i): accessors valid for 0 <= i < S;  w_out: shared/global array [S] written by the warp.
// Returns sum of weights (acc) reduced over the warp.
template <class SigmaFn, class ZFn>
__device__ __forceinline__ void ray_weights(int S, float dnorm, SigmaFn sigma, ZFn zval, float* w_out, int lane) {
  float carry = 1.0f;
  for (int base = 0; base < S; base += 32) {
    const int i = base + lane;
    float alpha = 0.0f, f = 1.0f;
    if (i < S) {
      const float zi = zval(i);
      float dist = (i == S - 1) ? 1e10f : __fsub_rn(zval(i + 1), zi);       // render.py:9-10
      dist = __fmul_rn(dist, dnorm);                                          // render.py:12
      const float sg = fmaxf(sigma(i), 0.0f);
      alpha = __fsub_rn(1.0f, expf(-__fmul_rn(sg, dist)));                    // render.py:7
      f = __fadd_rn(__fsub_rn(1.0f, alpha), 1e-10f);                          // render.py:18
    }
    const float incl = warp_scan_mul(f, lane);
    float excl = __shfl_up_sync(FULL, incl, 1);
    if (lane == 0) excl = 1.0f;
    if (i < S) w_out[i] = __fmul_rn(alpha, __fmul_rn(carry, excl));
    carry = __fmul_rn(carry, __shfl_sync(FULL, incl, 31));
  }
}

// torch.linspace(0, 1, n)[i] in fp32: ATen evaluates symmetrically, start + step*i for the lower half and a
// fused end - step*(n-1-i) for the upper half (checked against torch in tests/test_host.py).
__device__ __forceinline__ float linspace01(int i, int n) {
  const float step = 1.0f / (float)(n - 1);
  return (i < n / 2) ? __fmul_rn(step, (float)i) : __fmaf_rn(-step, (float)(n - 1 - i), 1.0f);
}

// Additive inclusive warp scan.
__device__ __forceinline__ float warp_scan_add(float v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const float o = __shfl_up_sync(FULL, v, d);
    if (lane >= d) v += o;
  }
  return v;
}

// Inverse-CDF sampling for one ray (networks/helpers.py:123-155).
//   bins: [nb] (shared), wts: accessor for nb-1 weights, cdf: shared scratch [nb], out: [ns].
//   u == nullptr => deterministic linspace.  The cdf is a warp prefix sum (the reference's GPU cumsum is a parallel fp32
//   scan as well; its CPU cumsum differs from either by ~1e-7, far below the 1e-5 bin-mass threshold of helpers.py:151).
// Part 1 (one warp): cdf[0..nb) of the nb-1 bin weights.
template <class WFn>
__device__ __forceinline__ void ray_build_cdf(WFn wts, int nb, float* cdf, int lane) {
  const int nw = nb - 1;
  float part = 0.0f;
  for (int j = lane; j < nw; j += 32) part += __fadd_rn(wts(j), 1e-5f);      // helpers.py:125
  const float total = warp_sum(part);
  float carry = 0.0f;
  if (lane == 0) cdf[0] = 0.0f;
  for (int base = 0; base < nw; base += 32) {                                 // helpers.py:126-128
    const int j = base + lane;
    const float pdf = (j < nw) ? __fdiv_rn(__fadd_rn(wts(j), 1e-5f), total) : 0.0f;
    const float incl = warp_scan_add(pdf, lane);
    if (j < nw) cdf[j + 1] = carry + incl;
    carry += __shfl_sync(FULL, incl, 31);
  }
}

// Part 2 (any thread): the sample for one value of u.
__device__ __forceinline__ float ray_sample_at(const float* bins, const float* cdf, int nb, float us) {
  // searchsorted(cdf, u, right=True): first index with cdf[idx] > u   (helpers.py:139)
  int lo = 0, hi = nb;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] > us) hi = mid; else lo = mid + 1;
  }
  const int below = max(lo - 1, 0), above = min(lo, nb - 1);
  const float cb = cdf[below], ca = cdf[above];
  float denom = __fsub_rn(ca, cb);
  if (denom < 1e-5f) denom = 1.0f;                                          // helpers.py:151
  const float t = __fdiv_rn(__fsub_rn(us, cb), denom);
  const float bb = bins[below], ba = bins[above];
  return __fadd_rn(bb, __fmul_rn(t, __fsub_rn(ba, bb)));                    // helpers.py:153
}

template <class WFn>
__device__ __forceinline__ void ray_sample_pdf(const float* bins, WFn wts, int nb, int ns, const float* u, float* cdf,
                                               float* out, int lane) {
  ray_build_cdf(wts, nb, cdf, lane);
  __syncwarp();
  for (int s = lane; s < ns; s += 32) out[s] = ray_sample_at(bins, cdf, nb, u ? u[s] : linspace01(s, ns));
  __syncwarp();
}

// Thread `tid` of `nthr` cooperating threads: is its share of v[0..n) (shared) non-decreasing?
__device__ __forceinline__ bool ray_sorted_part(const float* v, int n, int tid, int nthr) {
  bool ok = true;
  for (int i = tid + 1; i < n; i += nthr) ok = ok && (v[i] >= v[i - 1]);
  return ok;
}

// Warp-uniform: is v[0..n) (shared) non-decreasing?
__device__ __forceinline__ bool ray_is_sorted(const float* v, int n, int lane) {
  return __all_sync(FULL, ray_sorted_part(v, n, lane, 32));
}

// Merge of two ASCENDING runs a[0..na) and b[0..nb) (shared) into out[0..na+nb): each element's output position is its own
// index plus the number of elements of the other run that precede it (binary search; ties: run a first).  This is
// sort(cat(a, b)) (networks/render.py:70) when both inputs are sorted -- always true for the coarse depths, and true for
// the importance samples whenever u is non-decreasing (the deterministic linspace).  `nthr` threads share the elements.
__device__ __forceinline__ void ray_merge_part(const float* a, int na, const float* b, int nb, float* out, int tid, int nthr) {
  for (int e = tid; e < na + nb; e += nthr) {
    const bool from_a = e < na;
    const float v = from_a ? a[e] : b[e - na];
    const float* other = from_a ? b : a;
    int lo = 0, hi = from_a ? nb : na;
    while (lo < hi) {                                   // from_a: count other < v ; from_b: count other <= v
      const int mid = (lo + hi) >> 1;
      const float o = other[mid];
      if (from_a ? (o < v) : (o <= v)) lo = mid + 1; else hi = mid;
    }
    out[(from_a ? e : e - na) + lo] = v;
  }
}
__device__ __forceinline__ void ray_merge_sorted(const float* a, int na, const float* b, int nb, float* out, int lane) {
  ray_merge_part(a, na, b, nb, out, lane, 32);
  __syncwarp();
}

// Rank sort of vals[0..T) (shared) into out[0..T): ascending, ties by index (networks/render.py:70).
__device__ __forceinline__ void ray_rank_part(const float* vals, int T, float* out, int tid, int nthr) {
  for (int e = tid; e < T; e += nthr) {
    const float v = vals[e];
    int rank = 0;
    for (int j = 0; j < T; ++j) {
      const float o = vals[j];
      rank += (o < v) || (o == v && j < e);
    }
    out[rank] = v;
  }
}
__device__ __forceinline__ void ray_rank_sort(const float* vals, int T, float* out, int lane) {
  ray_rank_part(vals, T, out, lane, 32);
  __syncwarp();
}

}  // namespace dmnerf
