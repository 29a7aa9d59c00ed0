// sampler.cu — fused octree traversal + perspective-warp ray march for sm_90a.
//
// Replaces, behind f2b_sampler_count / f2b_sampler_fill, the reference's
//   FindRayOctreeIntersectionKernel<false/true>  (src/PtsSampler/PersSampler.cu:53-152)
//   RayMarchKernel<false/true>                   (src/PtsSampler/PersSampler.cu:189-314)
//   QueryFrameTransform / QueryFrameTransformJac (src/PtsSampler/PersSampler.cu:155-187)
// and GetEdgeSamplesKernel (:436-452), MarkVistNodeKernel (:475-526), MarkInvalidNodes (:528-534)
// plus the ATen vote/stat update of UpdateOctNodes (:579-592).
//
// Design (not a translation):
//  * traversal and march are ONE kernel: the DFS is a coroutine that yields the next leaf hit
//    when the march walks off the current leaf, so the (node, near, far) hit list is never
//    written to HBM and the reference's first host sync (.item() at :353) disappears;
//  * 16 lanes (half a warp) cooperate on one ray, two rays per warp: 12 lanes each evaluate one of
//    the 12 perspective projections, then each lane forms one of the 3x4 mixing sums serially in
//    exactly the summation tree Eigen's unrolled redux produces in the reference build
//    ((p0+(p1+p2)) + (p3+(p4+p5))) + ((p6+(p7+p8)) + (p9+(p10+p11))), so every fp32 rounding —
//    and hence every sample count / index — is bit-identical to the reference kernel
//    (sequence read off the reference's PTX; see DESIGN.md §march-rounding);
//  * 16x more warps than thread-per-ray and a much shorter dependent chain per step;
//  * DFS stack lives in shared memory (packed node<<4|cursor, one private copy per lane so no
//    intra-group ordering is assumed), not 192 B/thread of local memory.
#include "common.cuh"
#include "locate.cuh"
#include "scan.cuh"

namespace f2b {

constexpr int kMaxDepth = 24;               // reference MAX_STACK_SIZE 48 = 24 (node, cursor) pairs
constexpr int kStackPitch = kMaxDepth + 1;  // 25 is odd: conflict-free across the 32 lanes

struct Hit {
  int node;
  int trans_idx;
  float near, far;
};

// child visit order: search_order[st][k] = ((~st)&7) ^ bitrev3(k)   (PersSampler.cpp:106-117;
// the std::sort comparator orders by lowest differing bit, bit != st's bit first)
__device__ __forceinline__ int child_slot(int st, int k) {
  int rev = ((k & 1) << 2) | (k & 2) | ((k >> 2) & 1);
  return ((~st) & 7) ^ rev;
}

// GetIntersection (PersSampler.cu:21-51): slab test, +-1e-6 parallel guard. near/far in-out.
__device__ __forceinline__ void slab(const float o[3], const float d[3], const float c[3],
                                     float side, float& near, float& far) {
  const float hf = fmul(side, .5f);
  float lo[3], hi[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    if (fabsf(d[i]) < 1e-6f) {
      const bool inside = (o[i] > fsub(c[i], hf)) && (o[i] < fadd(c[i], hf));
      lo[i] = inside ? -1e6f : 1e6f;
      hi[i] = inside ? 1e6f : -1e6f;
    } else if (d[i] > 0.f) {
      lo[i] = fdiv(fsub(fsub(c[i], hf), o[i]), d[i]);
      hi[i] = fdiv(fsub(fadd(c[i], hf), o[i]), d[i]);
    } else {
      lo[i] = fdiv(fsub(fadd(c[i], hf), o[i]), d[i]);
      hi[i] = fdiv(fsub(fsub(c[i], hf), o[i]), d[i]);
    }
  }
  near = fmaxf(near, fmaxf(lo[0], fmaxf(lo[1], lo[2])));
  far = fminf(far, fminf(hi[0], fminf(hi[1], hi[2])));
}

struct Dfs {
  int* stack;     // shared, packed (node << 4) | (cursor + 1)
  int sp;
  int n_hits;
  int max_hits;
  int st;
};

// Yields the next valid leaf the ray crosses, front to back (PersSampler.cu:89-140).
__device__ __forceinline__ bool next_hit(Dfs& s, const TreeNode* __restrict__ nodes,
                                         const float o[3], const float d[3], float near0,
                                         float far0, Hit& hit) {
  while (s.sp >= 0 && s.n_hits < s.max_hits) {
    const int packed = s.stack[s.sp];
    const int u = packed >> 4;
    const int cursor = (packed & 15) - 1;
    const int4* np = reinterpret_cast<const int4*>(nodes + u);
    const int4 q1 = __ldg(np + 1), q2 = __ldg(np + 2), q3 = __ldg(np + 3);
    const int childs[8] = {q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x};
    int child_ptr;
    if (cursor < 0) {
      const int4 q0 = __ldg(np);
      const float c[3] = {__int_as_float(q0.x), __int_as_float(q0.y), __int_as_float(q0.z)};
      float cn = near0, cf = far0;
      slab(o, d, c, __int_as_float(q0.w), cn, cf);
      if (!(cn < cf)) { s.sp--; continue; }
      child_ptr = 0;
      while (child_ptr < 8 && childs[child_slot(s.st, child_ptr)] < 0) child_ptr++;
      if (child_ptr >= 8) {            // no live child: treated as a leaf
        s.sp--;
        if (q3.z >= 0) {               // trans_idx >= 0
          hit.node = u; hit.trans_idx = q3.z; hit.near = cn; hit.far = cf;
          s.n_hits++;
          return true;
        }
        continue;
      }
    } else {
      child_ptr = cursor + 1;
      while (child_ptr < 8 && childs[child_slot(s.st, child_ptr)] < 0) child_ptr++;
      if (child_ptr >= 8) { s.sp--; continue; }
    }
    s.stack[s.sp] = (u << 4) | (child_ptr + 1);
    if (s.sp + 1 >= kMaxDepth) { s.sp = -1; break; }   // deeper than the reference's stack: stop
    s.sp++;
    s.stack[s.sp] = childs[child_slot(s.st, child_ptr)] << 4;   // cursor -1
  }
  return false;
}

// ---------------------------------------------------------------------------------------------------------
// The march: two rays per warp, 16 lanes each (the march is latency bound: at 4 lanes/ray 4096 rays would be
// only 512 warps on 528 SM sub-partitions).  Measured on the headline batch (H100 SXM at 400 W, profiles/h100_march_probe.json):
// 8 and 4 lanes per ray cut the static instructions per ray-step from ~76 to ~59 / ~44, but the march then takes
// 1.36 / 1.80 ms instead of 1.15 ms alone and longer under the backward too, so 16 lanes stay.  What does help is a
// shorter step: one store per lane and step, and the noise read issued before phase A (1.05 ms).  Each step has two phases:
//   A  lane g < 12 evaluates perspective projection g: xz, 1/xz1, the Jacobian factors T0..T2 and the value V;
//   B  the 4 x 12 block {T0,T1,T2,V} x projections is transposed through 192 B of shared memory and lane
//      (r, c) = (g >> 2, g & 3) forms ONE of the 12 mixing sums S[r][c] = sum_i weight[r][i] * T_c[i] serially
//      in registers, in exactly the reference's order (Eigen's unrolled redux: g_s = fma(w0,t0,fma(w1,t1,w2*t2))
//      per triple, then (g0+g1)+(g2+g3)) — 15 flops instead of a 4-shuffle tree per sum (r01 profile: the
//      shuffle trees were 108 of the 366 instructions of a step).
// The three Jacobian-times-direction rows are then chained over lanes (r,2)->(r,1)->(r,0) with two shuffles, and
// every lane picks them up (3 shuffles) and derives den / step redundantly, so no broadcast is needed.
// Every lane advances t / walks the octree redundantly (private DFS stack in shared memory).
constexpr int kL16 = 16;
constexpr int kRaysPerBlock16 = 2;
enum { kOutNone, kOutSv, kOutDt, kOutT, kOutTrans, kOutNode, kOutConst };   // what a lane stores per sample

template <int MODE>   // 0: count only, 1: fill at pts_idx_bounds, 2: one pass into per-ray scratch slots of 1024 samples
__global__ void __launch_bounds__(32, 1)
march16_kernel(const TreeNode* __restrict__ nodes, const TransInfo* __restrict__ trans,
               const float* __restrict__ rays_o, const float* __restrict__ rays_d,
               const float* __restrict__ rays_noise, int n_rays, float near0, float far0,
               float sample_l, int scale_by_dis, int max_hits, int count_all_hits,
               int* __restrict__ ray_counts, int* __restrict__ total_hits, const int* __restrict__ bounds,
               float* __restrict__ o_pts, float* __restrict__ o_dirs, float* __restrict__ o_dt,
               float* __restrict__ o_t, int* __restrict__ o_anchors, float* __restrict__ first_oct_dis) {
  __shared__ int s_stack[32 * kStackPitch];
  __shared__ __align__(16) float s_T[2][4][12];     // [half-warp][T0,T1,T2,V][projection]
  const int lane = threadIdx.x;
  const int g = lane & 15;                          // lane inside the ray's half-warp
  const int pi = g < 12 ? g : 11;                   // phase A: my projection (idle lanes shadow 11)
  const int orow = g < 12 ? (g >> 2) : 2;           // phase B: my mixing sum S[orow][ocol]
  const int ocol = g & 3;
  float* const tb = &s_T[lane >> 4][0][0];
  int ray = blockIdx.x * kRaysPerBlock16 + (lane >> 4);
  const bool active = ray < n_rays;
  if (!active) ray = n_rays - 1;
  constexpr bool FILL = MODE != 0;

  const float o[3] = {__ldg(rays_o + ray * 3), __ldg(rays_o + ray * 3 + 1), __ldg(rays_o + ray * 3 + 2)};
  const float d[3] = {__ldg(rays_d + ray * 3), __ldg(rays_d + ray * 3 + 1), __ldg(rays_d + ray * 3 + 2)};
  const float dsel = ocol == 0 ? d[0] : (ocol == 1 ? d[1] : d[2]);
  const float* noise = rays_noise + ray;
  Dfs dfs;
  dfs.stack = s_stack + lane * kStackPitch;
  dfs.sp = 0; dfs.n_hits = 0; dfs.max_hits = max_hits;
  dfs.st = (int(d[0] > 0.f) << 2) | (int(d[1] > 0.f) << 1) | int(d[2] > 0.f);
  dfs.stack[0] = 0;

  int cap = F2B_MAX_SAMPLE_PER_RAY;
  size_t out_base = 0;
  if (MODE == 1) { out_base = bounds[ray * 2]; cap = bounds[ray * 2 + 1] - int(out_base); }
  else if (MODE == 2) out_base = size_t(ray) * F2B_MAX_SAMPLE_PER_RAY;

  // Output of a step: every lane of the ray stores at most ONE 32-bit word, through one predicated store, instead of
  // taking its own branch per output array.  Lanes (r, 3) hold pts[r]; the other lanes take dt, t, anchors and dirs.
  int role = kOutNone, comp = 0, stride = 1;
  unsigned* obase = nullptr;
  unsigned cbits = 0;                                            // the value of a kOutConst lane
  if (FILL) {
    const int m = g < 12 ? (ocol == 3 ? -1 : 3 * (g >> 2) + ocol) : 9 + g - 12;
    // m: -1 pts; 0 dt; 1 t; 2 anchors[0]; 3 anchors[1]; 4 anchors[2] (MODE 1); 5..7 dirs (MODE 1)
    if (m < 0)       { role = kOutSv;    obase = reinterpret_cast<unsigned*>(o_pts); stride = 3; comp = orow; }
    else if (m == 0) { role = kOutDt;    obase = reinterpret_cast<unsigned*>(o_dt); }
    else if (m == 1) { role = kOutT;     obase = reinterpret_cast<unsigned*>(o_t); }
    else if (m == 2) { role = kOutTrans; obase = reinterpret_cast<unsigned*>(o_anchors); stride = MODE == 1 ? 3 : 2; }
    else if (m == 3) { role = kOutNode;  obase = reinterpret_cast<unsigned*>(o_anchors); stride = MODE == 1 ? 3 : 2; comp = 1; }
    else if (MODE == 1 && m == 4) { role = kOutConst; obase = reinterpret_cast<unsigned*>(o_anchors); stride = 3; comp = 2; }
    else if (MODE == 1 && m <= 7) {
      role = kOutConst; obase = reinterpret_cast<unsigned*>(o_dirs); stride = 3; comp = m - 5;
      cbits = __float_as_uint(comp == 0 ? d[0] : (comp == 1 ? d[1] : d[2]));
    }
    if (!active) role = kOutNone;
  }
  unsigned* const optr = obase ? obase + out_base * stride + comp : nullptr;

  Hit hit;
  hit.node = 0; hit.trans_idx = 0; hit.near = 0.f; hit.far = 0.f;
  bool have = next_hit(dfs, nodes, o, d, near0, far0, hit);
  if (FILL && active && g == 0) first_oct_dis[ray] = have ? hit.near : 1e9f;

  int k = 0;
  float t = hit.near, far = hit.far;
  int cur_node = hit.node, cur_trans = hit.trans_idx, loaded_trans = -1;
  bool first = true;
  float pa[4] = {0.f, 0.f, 0.f, 0.f}, pb[4] = {0.f, 0.f, 0.f, 1.f};
  float wr[12];
#pragma unroll
  for (int i = 0; i < 12; i++) wr[i] = 0.f;
  float rclip = 1.f;
  bool running = have && cap > 0;
  while (__any_sync(0xffffffffu, running)) {
    if (running && cur_trans != loaded_trans) {
      const TransInfo* T = trans + cur_trans;
      const float4 ra = __ldg(reinterpret_cast<const float4*>(&T->w2xz[pi][0]));
      const float4 rb = __ldg(reinterpret_cast<const float4*>(&T->w2xz[pi][4]));
      pa[0] = ra.x; pa[1] = ra.y; pa[2] = ra.z; pa[3] = ra.w;
      pb[0] = rb.x; pb[1] = rb.y; pb[2] = rb.z; pb[3] = rb.w;
      const float4* wp = reinterpret_cast<const float4*>(&T->weight[orow][0]);
      const float4 w0 = __ldg(wp), w1 = __ldg(wp + 1), w2 = __ldg(wp + 2);
      wr[0] = w0.x; wr[1] = w0.y; wr[2] = w0.z; wr[3] = w0.w; wr[4] = w1.x; wr[5] = w1.y; wr[6] = w1.z; wr[7] = w1.w;
      wr[8] = w2.x; wr[9] = w2.y; wr[10] = w2.z; wr[11] = w2.w;
      const float4 cd = __ldg(reinterpret_cast<const float4*>(&T->center[0]));
      const float ex = fsub(o[0], cd.x), ey = fsub(o[1], cd.y), ez = fsub(o[2], cd.z);
      rclip = fmaxf(fdiv(fsqrt(ffma(ex, ex, ffma(ey, ey, fmul(ez, ez)))), cd.w), 1.f);
      loaded_trans = cur_trans;
    }
    const float nz = __ldg(noise + k);                         // issued first: its latency hides under phase A
    // ---- phase A: my projection -------------------------------------------------------------------
    const float X = ffma(t, d[0], o[0]), Y = ffma(t, d[1], o[1]), Z = ffma(t, d[2], o[2]);
    const float xz0 = fadd(ffma(X, pa[0], fmul(Y, pa[1])), ffma(Z, pa[2], pa[3]));
    const float xz1 = fadd(ffma(X, pb[0], fmul(Y, pb[1])), ffma(Z, pb[2], pb[3]));
    const float rr = frcp(xz1);
    const float q = fdiv(-xz0, fmul(xz1, xz1));
    const float T0 = ffma(pa[0], rr, fmul(pb[0], q));
    const float T1 = ffma(rr, pa[1], fmul(q, pb[1]));
    const float T2 = ffma(rr, pa[2], fmul(q, pb[2]));
    if (g < 12) {
      tb[g] = T0; tb[12 + g] = T1; tb[24 + g] = T2;
      if (FILL) tb[36 + g] = fdiv(xz0, xz1);
    }
    __syncwarp();
    // ---- phase B: my mixing sum, serial in the reference's order ------------------------------------
    const float4* tv = reinterpret_cast<const float4*>(tb + ocol * 12);
    const float4 ta = tv[0], tc = tv[1], te = tv[2];
    __syncwarp();                                              // the block may be overwritten by the next step
    const float g0 = ffma(wr[0], ta.x, ffma(wr[1], ta.y, fmul(wr[2], ta.z)));
    const float g1 = ffma(wr[3], ta.w, ffma(wr[4], tc.x, fmul(wr[5], tc.y)));
    const float g2 = ffma(wr[6], tc.z, ffma(wr[7], tc.w, fmul(wr[8], te.x)));
    const float g3 = ffma(wr[9], te.y, ffma(wr[10], te.z, fmul(wr[11], te.w)));
    const float Sv = fadd(fadd(g0, g1), fadd(g2, g3));         // S[orow][ocol]
    // proj[r] = fma(j0,d0, fma(j1,d1, j2*d2)) chained over lanes (r,2) -> (r,1) -> (r,0)
    const float m2 = fmul(Sv, dsel);
    const float v1 = ffma(Sv, dsel, __shfl_down_sync(0xffffffffu, m2, 1, 16));
    const float pj = ffma(Sv, dsel, __shfl_down_sync(0xffffffffu, v1, 1, 16));          // meaningful in lanes 0, 4, 8
    const float p0 = __shfl_sync(0xffffffffu, pj, 0, 16), p1 = __shfl_sync(0xffffffffu, pj, 4, 16),
                p2 = __shfl_sync(0xffffffffu, pj, 8, 16);
    const float den = fadd(fsqrt(ffma(p0, p0, ffma(p1, p1, fmul(p2, p2)))), 1e-6f);
    float step = fdiv(fmul(sample_l, nz), den);
    if (scale_by_dis) step = fmul(rclip, step);

    if (running) {
      if (!first) {
        if (FILL && role != kOutNone) {
          unsigned v = cbits;
          v = role == kOutSv ? __float_as_uint(Sv) : v;
          v = role == kOutDt ? __float_as_uint(fmul(step, den)) : v;
          v = role == kOutT ? __float_as_uint(t) : v;
          v = role == kOutTrans ? unsigned(cur_trans) : v;
          v = role == kOutNode ? unsigned(cur_node) : v;
          optr[size_t(k) * stride] = v;
        }
        k++;
      }
      float tn = fadd(t, step);
      if (tn > far) {
        for (;;) {
          have = next_hit(dfs, nodes, o, d, near0, far0, hit);
          if (!have) break;
          far = hit.far; cur_node = hit.node; cur_trans = hit.trans_idx;
          const float nf = ceilf(fmaxf(fdiv(fsub(hit.near, t), step), 1.f));
          const int n = (int)nf;
          tn = ffma(step, (float)n, t);
          if (!(tn > far)) break;
        }
      }
      t = tn;
      first = false;
      running = (k < cap) && have;
    }
  }
  if (MODE != 1) {
    if (count_all_hits) {
      while (next_hit(dfs, nodes, o, d, near0, far0, hit)) {}
    }
    if (active && g == 0) {
      ray_counts[ray] = k;
      if (dfs.n_hits) atomicAdd(total_hits, dfs.n_hits);
    }
  }
}

// Second half of the one-pass sampler: copy each ray's samples from its scratch slot to the compact,
// ray-ordered outputs (the reference's cumsum layout), regenerating dirs / anchors[:,2]; warp per ray.
__global__ void __launch_bounds__(256)
sampler_gather_kernel(const float* __restrict__ rays_d, const int* __restrict__ bounds, int n_rays,
                      const float* __restrict__ s_pts, const float* __restrict__ s_dt, const float* __restrict__ s_t,
                      const int* __restrict__ s_anchors, float* __restrict__ pts, float* __restrict__ dirs,
                      float* __restrict__ dt, float* __restrict__ t, int* __restrict__ anchors) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], n = bounds[2 * ray + 1] - beg;
  const size_t src = size_t(ray) * F2B_MAX_SAMPLE_PER_RAY;
  const float d0 = rays_d[ray * 3], d1 = rays_d[ray * 3 + 1], d2 = rays_d[ray * 3 + 2];
  for (int i = lane; i < 3 * n; i += 32) {              // 12-byte rows as flat float streams: fully coalesced
    pts[size_t(beg) * 3 + i] = s_pts[src * 3 + i];
    const int c = i % 3;
    dirs[size_t(beg) * 3 + i] = c == 0 ? d0 : (c == 1 ? d1 : d2);
    const int j = i / 3;
    anchors[size_t(beg) * 3 + i] = c == 2 ? 0 : s_anchors[(src + j) * 2 + c];
  }
  for (int i = lane; i < n; i += 32) { dt[beg + i] = s_dt[src + i]; t[beg + i] = s_t[src + i]; }
}

// ---- edge samples (PersSampler.cu:436-452; warp_point in locate.cuh) ----------------------------
__global__ void edge_samples_kernel(int n_pts, const EdgePool* __restrict__ edge_pool,
                                    const TransInfo* __restrict__ trans,
                                    const int* __restrict__ edge_idx,
                                    const float* __restrict__ edge_coord,
                                    float* __restrict__ out_pts, int* __restrict__ out_idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts) return;
  const EdgePool* e = edge_pool + edge_idx[i];
  const float c0 = edge_coord[2 * i], c1 = edge_coord[2 * i + 1];
  // center + dir_0*c0 + dir_1*c1, contracted as fma(dir_1,c1, fma(dir_0,c0, center))
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; k++) w[k] = ffma(e->dir_1[k], c1, ffma(e->dir_0[k], c0, e->center[k]));
  float pa[3], pb[3];
  const int a = e->t_idx_a, b = e->t_idx_b;
  warp_point(trans + a, w[0], w[1], w[2], pa);
  warp_point(trans + b, w[0], w[1], w[2], pb);
#pragma unroll
  for (int k = 0; k < 3; k++) { out_pts[i * 6 + k] = pa[k]; out_pts[i * 6 + 3 + k] = pb[k]; }
  out_idx[2 * i] = a; out_idx[2 * i + 1] = b;
}

// ---- octree occupancy votes (PersSampler.cu:475-534, 579-603) -----------------------------------
// one warp per ray: lanes stride the ray's samples for the two maxima, then lane 0 walks the
// runs (run boundaries are data dependent; the per-node votes are atomicMax => order free, bit exact).
__global__ void mark_visit_kernel(int n_rays, const int* __restrict__ bounds,
                                  const int* __restrict__ oct_idx, int oct_stride,
                                  const float* __restrict__ weights, const float* __restrict__ alphas,
                                  int* __restrict__ vote_w, int* __restrict__ vote_a,
                                  int* __restrict__ mark, int* __restrict__ visit_cnt) {
  const int ray = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (ray >= n_rays) return;
  const int beg = bounds[2 * ray], end = bounds[2 * ray + 1];
  if (beg >= end) return;
  float mw = 0.f, ma = 0.f;
  for (int i = beg + lane; i < end; i += 32) { mw = fmaxf(mw, weights[i]); ma = fmaxf(ma, alphas[i]); }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    mw = fmaxf(mw, __shfl_xor_sync(0xffffffffu, mw, o));
    ma = fmaxf(ma, __shfl_xor_sync(0xffffffffu, ma, o));
  }
  const float w_thr = fminf(fmul(mw, 0.1f), 0.01f);
  const float a_thr = fminf(fmul(ma, 0.1f), 0.02f);
  // each lane handles the runs that START in its 32-strided positions? runs are contiguous, so
  // instead: lane l scans chunk [beg + l*len, ...) and merges partial runs at chunk borders via atomics.
  // atomicMax of (occupied ? base : -1) over sub-runs equals the vote of the whole run because
  // max(run) > thr  <=>  any sub-run max > thr; visit_cnt needs the full run length, handled by
  // letting a run be owned by the lane where it starts and continuing past the chunk border.
  const int n = end - beg;
  const int per = (n + 31) / 32;
  int i = beg + lane * per;
  const int stop = min(i + per, end);
  if (i >= end) return;
  // skip a run that started in a previous lane's chunk
  if (i > beg) {
    const int prev = oct_idx[size_t(i - 1) * oct_stride];
    while (i < stop && oct_idx[size_t(i) * oct_stride] == prev) i++;
  }
  while (i < stop) {
    const int node = oct_idx[size_t(i) * oct_stride];
    float rw = 0.f, ra = 0.f;
    int cnt = 0;
    while (i < end && oct_idx[size_t(i) * oct_stride] == node) {   // may run past `stop`: owner finishes it
      rw = fmaxf(rw, weights[i]); ra = fmaxf(ra, alphas[i]); cnt++; i++;
    }
    if (node >= 0) {
      atomicMax(vote_w + node, rw > w_thr ? 512 : -1);
      atomicMax(vote_a + node, ra > a_thr ? 32 : -1);
      atomicMax(visit_cnt + node, cnt);
      mark[node] = 1;
    }
  }
}

__global__ void update_stats_kernel(int n_nodes, const int* __restrict__ vote_w,
                                    const int* __restrict__ vote_a, const int* __restrict__ mark,
                                    int* __restrict__ stats_w, int* __restrict__ stats_a,
                                    TreeNode* __restrict__ nodes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_nodes) return;
  const int m = mark[i];
  int sw, sa;
  {
    const int v = vote_w[i], occ = v > 0 ? 1 : 0;
    int s = max(stats_w[i], occ * v);
    s += m * (1 - occ) * v;
    sw = min(max(s, -100), 1 << 20);
    stats_w[i] = sw;
  }
  {
    const int v = vote_a[i], occ = v > 0 ? 1 : 0;
    int s = max(stats_a[i], occ * v);
    s += m * (1 - occ) * v;
    sa = min(max(s, -100), 1 << 20);
    stats_a[i] = sa;
  }
  if (sw < 0 || sa < 0) nodes[i].trans_idx = -1;
}

}  // namespace f2b

using namespace f2b;

#define F2B_LAUNCH_MARCH(MODE, st, ...) \
  march16_kernel<MODE><<<div_up(n_rays, kRaysPerBlock16), 32, 0, st>>>(__VA_ARGS__)

extern "C" int f2b_sampler_count(const void* tree_nodes, int n_nodes, const void* trans, int n_trans,
                                 const float* rays_o, const float* rays_d, const float* rays_noise,
                                 int n_rays, float near, float far, float sample_l, int scale_by_dis,
                                 int max_oct_intersect_per_ray, int count_all_hits, int* ray_counts,
                                 int* pts_idx_bounds, int* totals, void* stream) {
  F2B_REQUIRE(n_rays >= 0 && n_nodes > 0 && n_trans >= 0, "f2b_sampler_count: bad sizes");
  F2B_REQUIRE(totals, "f2b_sampler_count: null totals");
  cudaStream_t st = as_stream(stream);
  cudaMemsetAsync(totals, 0, 2 * sizeof(int), st);
  if (n_rays == 0) return check_launch("f2b_sampler_count");      // empty batch: totals = {0, 0}
  F2B_REQUIRE(tree_nodes && trans && rays_o && rays_d && rays_noise && ray_counts && pts_idx_bounds,
              "f2b_sampler_count: null pointer");
  F2B_LAUNCH_MARCH(0, st,
      (const TreeNode*)tree_nodes, (const TransInfo*)trans, rays_o, rays_d, rays_noise, n_rays, near,
      far, sample_l, scale_by_dis, max_oct_intersect_per_ray, count_all_hits, ray_counts, totals + 1, nullptr, nullptr,
      nullptr, nullptr, nullptr, nullptr, nullptr);
  scan_counts_kernel<<<1, 1024, 0, st>>>(ray_counts, n_rays, pts_idx_bounds, totals);
  return check_launch("f2b_sampler_count");
}

extern "C" int f2b_sampler_fill(const void* tree_nodes, int n_nodes, const void* trans, int n_trans,
                                const float* rays_o, const float* rays_d, const float* rays_noise,
                                int n_rays, float near, float far, float sample_l, int scale_by_dis,
                                int max_oct_intersect_per_ray, const int* pts_idx_bounds, float* pts,
                                float* dirs, float* dt, float* t, int* anchors, float* first_oct_dis,
                                void* stream) {
  F2B_REQUIRE(n_rays >= 0 && n_nodes > 0, "f2b_sampler_fill: bad sizes");
  if (n_rays == 0) return F2B_OK;
  F2B_REQUIRE(tree_nodes && trans && pts_idx_bounds && first_oct_dis, "f2b_sampler_fill: null pointer");
  F2B_LAUNCH_MARCH(1, as_stream(stream),
      (const TreeNode*)tree_nodes, (const TransInfo*)trans, rays_o, rays_d, rays_noise, n_rays, near,
      far, sample_l, scale_by_dis, max_oct_intersect_per_ray, 0, nullptr, nullptr, pts_idx_bounds, pts,
      dirs, dt, t, anchors, first_oct_dis);
  return check_launch("f2b_sampler_fill");
}

extern "C" int f2b_sampler_march(const void* tree_nodes, int n_nodes, const void* trans, int n_trans,
                                 const float* rays_o, const float* rays_d, const float* rays_noise, int n_rays,
                                 float near, float far, float sample_l, int scale_by_dis,
                                 int max_oct_intersect_per_ray, int count_all_hits, float* s_pts, float* s_dt,
                                 float* s_t, int* s_anchors, int* ray_counts, int* pts_idx_bounds, int* totals,
                                 float* first_oct_dis, void* stream) {
  F2B_REQUIRE(n_rays >= 0 && n_nodes > 0 && n_trans >= 0, "f2b_sampler_march: bad sizes");
  F2B_REQUIRE(totals, "f2b_sampler_march: null totals");
  cudaStream_t st = as_stream(stream);
  cudaMemsetAsync(totals, 0, 2 * sizeof(int), st);
  if (n_rays == 0) return check_launch("f2b_sampler_march");
  F2B_REQUIRE(tree_nodes && trans && rays_o && rays_d && rays_noise && s_pts && s_dt && s_t && s_anchors && ray_counts &&
              pts_idx_bounds && first_oct_dis, "f2b_sampler_march: null pointer");
  F2B_LAUNCH_MARCH(2, st,
      (const TreeNode*)tree_nodes, (const TransInfo*)trans, rays_o, rays_d, rays_noise, n_rays, near, far, sample_l,
      scale_by_dis, max_oct_intersect_per_ray, count_all_hits, ray_counts, totals + 1, nullptr, s_pts, nullptr, s_dt, s_t,
      s_anchors, first_oct_dis);
  scan_counts_kernel<<<1, 1024, 0, st>>>(ray_counts, n_rays, pts_idx_bounds, totals);
  return check_launch("f2b_sampler_march");
}

extern "C" int f2b_sampler_gather(const float* rays_d, const int* pts_idx_bounds, int n_rays, const float* s_pts,
                                  const float* s_dt, const float* s_t, const int* s_anchors, float* pts, float* dirs,
                                  float* dt, float* t, int* anchors, void* stream) {
  if (n_rays <= 0) return F2B_OK;
  F2B_REQUIRE(rays_d && pts_idx_bounds && s_pts && s_dt && s_t && s_anchors, "f2b_sampler_gather: null pointer");
  sampler_gather_kernel<<<div_up(int64_t(n_rays) * 32, 256), 256, 0, as_stream(stream)>>>(
      rays_d, pts_idx_bounds, n_rays, s_pts, s_dt, s_t, s_anchors, pts, dirs, dt, t, anchors);
  return check_launch("f2b_sampler_gather");
}

extern "C" int f2b_edge_samples(const void* edge_pool, const void* trans, const int* edge_idx,
                                const float* edge_coord, int n_pts, float* out_pts, int* out_idx,
                                void* stream) {
  if (n_pts <= 0) return F2B_OK;
  edge_samples_kernel<<<div_up(n_pts, 128), 128, 0, as_stream(stream)>>>(
      n_pts, (const EdgePool*)edge_pool, (const TransInfo*)trans, edge_idx, edge_coord, out_pts, out_idx);
  return check_launch("f2b_edge_samples");
}

extern "C" int f2b_oct_mark_visit(const int* pts_idx_bounds, int n_rays, const int* oct_idx,
                                  int oct_stride, const float* weights, const float* alphas,
                                  int* vote_weight, int* vote_alpha, int* visit_mark, int* visit_cnt,
                                  void* stream) {
  if (n_rays <= 0) return F2B_OK;
  mark_visit_kernel<<<div_up(int64_t(n_rays) * 32, 256), 256, 0, as_stream(stream)>>>(
      n_rays, pts_idx_bounds, oct_idx, oct_stride, weights, alphas, vote_weight, vote_alpha, visit_mark,
      visit_cnt);
  return check_launch("f2b_oct_mark_visit");
}

extern "C" int f2b_oct_update_stats(const int* vote_weight, const int* vote_alpha, const int* visit_mark,
                                    int* weight_stats, int* alpha_stats, void* tree_nodes, int n_nodes,
                                    void* stream) {
  if (n_nodes <= 0) return F2B_OK;
  update_stats_kernel<<<div_up(n_nodes, 256), 256, 0, as_stream(stream)>>>(
      n_nodes, vote_weight, vote_alpha, visit_mark, weight_stats, alpha_stats, (TreeNode*)tree_nodes);
  return check_launch("f2b_oct_update_stats");
}
