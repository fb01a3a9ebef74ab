// Wavefront kernels of the H100 path tracer (sm_90a).  One iteration of the loop =
//   k_regen        : SobolPathSampler::startPath + ReconstructionFilter::sample + PinholeCamera::sampleDirection for the camera
//                    paths that replace finished ones (appended behind the compacted survivors)
//   k_trace        : TraceableScene::intersect (closest hit): persistent CTAs pull rays from the coherence-sorted queue and walk
//                    the 4-ary BVH of 64-byte quantised nodes over all mesh triangles (+ curve segments, + the analytic
//                    primitives when they are many) as a warp state machine (bvh_traverse_persistent).
//                    Few analytic primitives are tested by the kernel that creates the ray instead
//   k_shade        : makeLocalScatterEvent + handleSurface (NEE/MIS query generation, emission, BSDF sample, Russian roulette);
//                    instantiations: material-sorted window, all-Lambert lobe set, curves
//   k_shadow_prep  : analytic part of the NEE/MIS queries, top-level BVH cut, compaction of what is left
//   k_shadow_bvh   : attenuatedEmission / generalizedShadowRay for those (same traversal + epilogue)
//   k_accum        : folds the bounce's direct-light estimate into the path, NaN guards, compacts survivors into the other
//                    state buffer, analytic test + BVH cut + coherence key of their next ray
//   k_iter_end     : (one block) scan of the key histogram + the loop's bookkeeping: the sizes of the next iteration live in
//                    a device-resident control block, the host only reads them one iteration late (no sync in the loop)
//   k_bin_scatter  : counting sort of the survivors' slot indices by ray-coherence key
//   k_resolve      : OutputBuffer::addSample running mean, samples folded in sample-index order
// Tuning comparisons marked (B200) were measured on the project's previous GPU and are kept on the H100, which has the same
// 64 K registers and 228 KB of shared memory per SM; they have not been measured again.  Those marked (H100) were.
// Path state is stored as 16-byte records, one array per record kind (one LDG/STG.128 per record, 512 contiguous bytes per warp
// instruction): four traversal/shading records + emission + RNG state per slot, double buffered (k_accum compacts from one
// buffer into the other); per-bounce scratch records for the direct-light estimate.
#pragma once
#include "tgb_device.cuh"

namespace tgb {

// ---- path state ----------------------------------------------------------------------------------
// Persistent per slot (double buffered), one float4 array per record so that the streaming kernels move 512 contiguous bytes
// per warp instruction:
//   T0[s] = (ray origin, tmin)                    T1[s] = (ray direction, info)     info = dimension[0:16) | bounce[16:24) | flags
//   T2[s] = closest hit (t, u, v, id)             T3[s] = (throughput, path id)     path id = (sample within the call << pix_bits) | pixel_list_index
// (One 64-byte record per slot -- a single line per gathered ray in k_trace -- was measured slower for k_shade and k_accum (B200):
// the 64-byte lane stride quarters the bytes each of their load/store instructions moves per cache line.)
struct PathBuf {
    float4 *T0, *T1, *T2, *T3;
    float4 *E;          // (emission accumulated so far = the sample's radiance, unused)
    uint64_t *pcg;      // supplemental PCG state
};
// Per-bounce scratch (written by k_shade for the paths that issue NEE/MIS queries, read by k_shadow_bvh and k_accum):
struct Scratch {
    float4 *P;          // (shading point, IntersectionInfo::epsilon)
    float4 *N0, *N1;    // NEE: (direction, distance | t of the light's own hit), (f | finished lightF, pdfL)
    float4 *M0, *M1;    // MIS: (direction, pdfB | t of the light's own hit), (weight | finished bsdfF, NEE's pdfB)
    float4 *D0, *D1;    // (throughput before the bounce, light-pick weight), (surface emission term, light primitive)
    uint32_t *vis;      // vis[2s + mis] = 1 when that query's light term counts (nothing but the light in the way)
    float4 *SH;         // per closest-hit shadow-queue entry: the query's initial (analytic) hit
    uint32_t *cut_mask; // per any-hit shadow-queue entry: the top-level cut boxes its segment enters (bit k = DScene::cut box k)
    float4 *R;          // finished radiance per path of the step, indexed by path id (not by slot)
};

enum : uint32_t { F_WAS_SPECULAR = 1u << 24, F_ALIVE = 1u << 25, F_FINAL_CHECK = 1u << 26, F_HAS_NEE = 1u << 27,
                  F_HAS_SURF = 1u << 28 };
constexpr int HID_MISS = -1;

struct Counters { unsigned long long rays, hits, shadow_rays, shadow_hits; };   // path queries / NEE+MIS queries

// Device-resident control block of the wavefront loop.  k_iter_end writes the sizes of the NEXT iteration; every kernel of
// an iteration reads them from here, its grid is only an upper bound chosen by the host from a snapshot one iteration old (k_regen,
// k_shadow_prep and k_bin_scatter loop over the sizes with at most the blocks that are resident at once).
struct Ctl {
    uint32_t n;             // slots in use this iteration: survivors [0, n_surv) + new camera paths [n_surv, n)
    uint32_t n_surv;
    uint32_t n_sorted;      // survivors the traversal visits (prefix of order[]); the others miss the BVH's top-level cut
    uint32_t n_new;
    uint32_t first_path;    // path id of the first new camera path
    uint32_t issued;        // camera paths started so far, this iteration included
    uint32_t total;         // camera paths of the (sub)step
    uint32_t capacity;
    uint32_t next_count;    // survivors appended by k_accum
    uint32_t shadow_count;  // NEE/MIS queries emitted by k_shade
    uint32_t shadow_count2; // ... of which k_shadow_prep could not resolve analytically, any-hit: k_shadow_bvh's first queue
    uint32_t cursor_trace, cursor_shadow;       // ray cursors of the persistent traversal kernels
    uint32_t shadow_count_closest, cursor_closest;    // ... closest-hit (mesh-light) ones: its second queue, and its cursor
    unsigned long long traversed, shadow_traversed;   // statistics: queries that reached k_trace / k_shadow_bvh
    uint32_t iterations;
};

// ---- closest-hit traversal -------------------------------------------------------------------
struct Hit { float t, u, v; int id; };

TGB_D float xor_sign(float a, uint32_t sgn) { return __uint_as_float(__float_as_uint(a) ^ sgn); }
// Embree's Vec3 dot: x*x' + (y*y' + z*z') (thirdparty/embree/common/math/vec3.h:182)
TGB_D float edot(V3 a, V3 b) { return a.x*b.x + (a.y*b.y + a.z*b.z); }

// Quad::intersect (primitives/Quad.cpp:71-99)
TGB_D void quad_intersect(const DPrim &q, int self, V3 o, V3 d, float tnear, Hit &h) {
    float nDotW = dot(d, q.normal);
    if (fabsf(nDotW) < 1e-6f) return;
    float t = dot(q.normal, q.base - o)/nDotW;
    if (t < tnear || t > h.t) return;
    V3 qq = o + d*t;
    V3 v = qq - q.base;
    float l0 = dot(v, q.edge0)*q.inv_uv_sq0;
    float l1 = dot(v, q.edge1)*q.inv_uv_sq1;
    if (l0 < 0.0f || l0 > 1.0f || l1 < 0.0f || l1 > 1.0f) return;
    h.t = t; h.u = l0; h.v = l1; h.id = -(self + 2);
}
// Cube::intersect (primitives/Cube.cpp:94-127); backside flag travels in h.u
TGB_D void cube_intersect(const DPrim &c, int self, V3 o, V3 d, float tnear, Hit &h) {
    V3 p = m3mul(c.inv_rot, o - c.pos);
    V3 dl = m3mul(c.inv_rot, d);
    V3 invD = v3(1.0f/dl.x, 1.0f/dl.y, 1.0f/dl.z);
    V3 relMin = -c.scale - p;
    V3 relMax = c.scale - p;
    float ttMin = tnear, ttMax = h.t;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float id = comp(invD, i), rmin = comp(relMin, i), rmax = comp(relMax, i);
        if (id >= 0.0f) { ttMin = maxf(ttMin, rmin*id); ttMax = minf(ttMax, rmax*id); }
        else            { ttMax = minf(ttMax, rmin*id); ttMin = maxf(ttMin, rmax*id); }
    }
    if (ttMin <= ttMax) {
        if (ttMin > tnear && ttMin < h.t) { h.t = ttMin; h.u = 0.0f; h.v = 0.0f; h.id = -(self + 2); }
        else if (ttMax > tnear && ttMax < h.t) { h.t = ttMax; h.u = 1.0f; h.v = 0.0f; h.id = -(self + 2); }
    }
}

// Analytic primitives (quads, cubes) are few and are tested coherently -- every lane runs the same loop -- by the
// kernel that CREATES a ray (k_raygen, k_accum, k_shadow_prep); the BVH kernels then start from that hit.
TGB_D Hit analytic_closest(const DScene &sc, V3 o, V3 d, float tnear, float tfar) {
    Hit h; h.t = tfar; h.u = 0.0f; h.v = 0.0f; h.id = HID_MISS;
    for (int i = 0; i < sc.n_analytic; ++i) {
        int pi = sc.analytic[i];
        const DPrim &p = sc.prims[pi];
        if (p.type == TGB_PRIM_QUAD) quad_intersect(p, pi, o, d, tnear, h);
        else cube_intersect(p, pi, o, d, tnear, h);
    }
    return h;
}
// first blocker among the analytic primitives other than `ignore` (generalizedShadowRay's test, TraceBase.cpp:79-83)
TGB_D bool analytic_any(const DScene &sc, V3 o, V3 d, float tnear, float tfar, int ignore) {
    Hit h; h.t = tfar; h.u = 0.0f; h.v = 0.0f; h.id = HID_MISS;
    for (int i = 0; i < sc.n_analytic; ++i) {
        int pi = sc.analytic[i];
        if (pi == ignore) continue;
        const DPrim &p = sc.prims[pi];
        if (p.type == TGB_PRIM_QUAD) quad_intersect(p, pi, o, d, tnear, h);
        else cube_intersect(p, pi, o, d, tnear, h);
        if (h.id != HID_MISS) return true;
    }
    return false;
}


// ---- curve segments (primitives/Curves.cpp:51-99,134-221,223-227,431-470) ---------------------
// A segment = three consecutive B-spline nodes (x, y, z, width), projected into the ray's frame (x, y across the ray,
// z along it) and bisected five times (Nakamaru & Ohno); the 32 leaf pieces are tested as half cylinders.
struct CurveFrame { V3 lx, ly; };
TGB_D CurveFrame curve_frame(V3 lz) {
    CurveFrame f;
    float d = sqrtf(lz.x*lz.x + lz.z*lz.z);
    if (d == 0.0f) { f.lx = v3(1.0f, 0.0f, 0.0f); f.ly = v3(0.0f, 0.0f, -lz.y); }
    else { f.lx = v3(lz.z/d, 0.0f, -lz.x/d); f.ly = v3(f.lx.z*lz.y, d, -lz.y*f.lx.x); }
    return f;
}
TGB_D float4 f4add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
TGB_D float4 f4sub(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
TGB_D float4 f4scale(float4 a, float s) { return make_float4(a.x*s, a.y*s, a.z*s, a.w*s); }
TGB_D float4 curve_project(V3 o, const CurveFrame &f, V3 lz, float4 q) {
    V3 p = v3(q.x - o.x, q.y - o.y, q.z - o.z);
    return make_float4(dot(f.lx, p), dot(f.ly, p), dot(lz, p), q.w);
}
// BVH primitives per segment.  Bounding each quarter of a segment's parameter range separately (4) gives four times
// tighter boxes for the long thin segments, but every primitive still has to run the reference's bisection of the WHOLE
// segment: its leaf pieces accept hits on the extension of their chord and its pruning bound is not conservative, so the
// answer depends on the visiting order of the 32 leaves (starting the bisection from a quarter changes 17 % of the pixels
// of tests/golden/hair, measured with the oracle; culling by the quarter's box changes none).  On C4 (650 k segments, B200) 4 is
// slower than 1 (more, not fewer, full bisections per ray); 4 with quarter-start bisection is faster but not the reference's
// image.  A segment already tested for this ray is skipped (a repeat can only find a
// subset of what the first test found).
constexpr int kCurvePieces = 1;
struct CurvePiece { float4 p0, p1; float tMin, tMax; int depth; };
// intersectHalfCylinder: updates (t, u, w) and the closest depth when the flattened piece is hit in (tMin, tMax)
TGB_D void curve_half_cylinder(const CurvePiece &node, float tMin, float &tMax, float &ht, float &hu, float &hw) {
    float vx = node.p1.x - node.p0.x, vy = node.p1.y - node.p0.y;
    float lengthSq = 0.0f; lengthSq += vx*vx; lengthSq += vy*vy;
    float invLengthSq = 1.0f/lengthSq;
    float invLength = sqrtf(invLengthSq);
    float d0 = node.p0.x*vx; d0 += node.p0.y*vy;
    float segmentT = -d0*invLengthSq;
    float signedUnnormalized = node.p0.x*vy - node.p0.y*vx;
    float distance = fabsf(signedUnnormalized)*invLength;
    float width = node.p0.w*(1.0f - segmentT) + node.p1.w*segmentT;
    if (distance > width) return;
    float depth = node.p0.z*(1.0f - segmentT) + node.p1.z*segmentT;
    float dz = node.p1.z - node.p0.z;
    float ySq = sqr(width) - sqr(distance);
    float lSq = ySq*(1.0f + dz*dz*invLengthSq);
    float deltaT = sqrtf(maxf(lSq, 0.0f));
    float t0 = depth - deltaT;
    V3 w3 = v3(node.p0.x - node.p1.x, node.p0.y - node.p1.y, node.p0.z - node.p1.z);
    lengthSq = 0.0f; lengthSq += w3.x*w3.x; lengthSq += w3.y*w3.y; lengthSq += w3.z*w3.z;
    segmentT = dot(v3(node.p0.x, node.p0.y, node.p0.z - t0), w3)/lengthSq;
    if (segmentT < 0.0f || t0 >= tMax || t0 <= tMin) return;
    float newT = segmentT*(node.tMax - node.tMin) + node.tMin;
    if (newT >= 0.0f && newT <= 1.0f) { hu = newT; ht = t0; hw = width; tMax = t0; }
}
// pointOnSpline<false> runs in bvh_traverse_persistent's BISECT / CYL states.  The reference keeps an explicit stack of pieces
// (tMin, tMax, both end points).  Every end point is the same function of its dyadic parameter (q0*t*t + q1*t + q2, t = k/2^depth,
// exact in float), and the stack is strictly LIFO with one pending sibling per depth, so the stack is a 5-bit mask there and a
// popped piece's end points are re-evaluated with curve_eval: same values, same visiting order, no local-memory traffic.
TGB_D float4 curve_eval(float4 q0, float4 q1, float4 q2, float t) {
    return f4add(f4add(f4scale(q0, t*t), f4scale(q1, t)), q2);
}
// ---- BVH traversal ------------------------------------------------------------------------------
// Traversal stack: the first kSmemStack entries of every lane live in shared memory, laid out [entry][thread] so that lane i
// always hits bank i (conflict-free whatever the lanes' depths); deeper entries spill to local memory.
#ifndef TGB_TRACE_BLOCK
#define TGB_TRACE_BLOCK 128
#endif
#ifndef TGB_SMEM_STACK
#define TGB_SMEM_STACK 32
#endif
// resident blocks per SM the traversal kernels are compiled for: 6 x 128 threads caps them at 85 registers (of 5..8 blocks,
// 6 measured fastest on C1, B200)
#ifndef TGB_MINB
#define TGB_MINB 6
#endif
constexpr int kTraceBlock = TGB_TRACE_BLOCK;
constexpr int kSmemStack = TGB_SMEM_STACK;
constexpr int kStackSize = 80;
constexpr int kLocalStack = kStackSize - kSmemStack;

TGB_D uint32_t smem_addr(const void *p) { return uint32_t(__cvta_generic_to_shared(p)); }
// The stack pointer lives in a plain register variable next to this struct (a member would be spilled with the array).
struct TravStack {
    uint32_t base;                   // shared-space byte address of this thread's column of the shared stack (entry 0)
    int local[kLocalStack];
    static TGB_D void sts(uint32_t addr, int v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }
    static TGB_D int lds(uint32_t addr) { int v; asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory"); return v; }
    TGB_D void push(int &sp, int v) {
        if (sp < kSmemStack) sts(base + uint32_t(sp)*(kTraceBlock*4u), v);
        else if (sp < kStackSize) local[sp - kSmemStack] = v;
        sp++;
    }
    TGB_D int pop(int &sp) {
        --sp;
        return sp < kSmemStack ? lds(base + uint32_t(sp)*(kTraceBlock*4u)) : local[sp - kSmemStack];
    }
};

// BVH traversal over the mesh triangles: one ray per lane over the 4-ary BVH.
// Node visit (QNode4, bvh_build.h) = 4 x 16-byte loads from global memory,
// per axis a = S/d, b = (origin - o)/d - a once per node, then per child plane ONE byte permute (1 + q*2^-15 assembled
// straight into float bits) and ONE fma; the hit children are ordered near-to-far with a 5-exchange sorting network, the
// nearest is entered and the others are pushed far-to-near (three predicated shared-memory stores).  The any-hit walk stops the
// network after the 3 exchanges that find the nearest and pushes the others unsorted.
// Triangle test = Embree's MoellerTrumboreIntersector1 (thirdparty/embree/kernels/geometry/
// triangle_intersector_moeller.h:75-111) with IEEE division for t,u,v.
// `any`: occlusion query, stop at the first triangle hit.
// Alternatives measured and rejected (B200): warp-synchronous speculative
// traversal, if-if state machines with and without several rays per lane, 32-byte quantised BINARY nodes, higher occupancy.
// Measured, lost and removed: the top nodes staged in shared memory by a bulk-async copy (H100, C1: 459 vs 486 Msamples/s);
// (B200) an L2 persistence window over nodes + triangle records (little gain in k_trace, a loss in the streaming kernels),
// 128-byte float nodes (7 dependent loads per visit against 4), a per-lane while-while walk (slower than the state machine),
// the whole leaf or one triangle per LEAF trip instead of two, a triangle record or a node fetched one trip ahead (+12 / +16
// registers, no gain), several rays reserved per atomicAdd.
#define TGB_CSWAP(ta, la, tb, lb) { bool sw_ = tb < ta; float tt_ = sw_ ? tb : ta; tb = sw_ ? ta : tb; ta = tt_; \
                                    int ll_ = sw_ ? lb : la; lb = sw_ ? la : lb; la = ll_; }
// 1 + q*2^-15 for byte K of word W: result bytes (0x3F, 0x80, q, 0x00).  The selector is an immediate and the constant word
// 0x3F80 sits in ONE register for all 24 planes of a visit (left to itself the compiler keeps the selector in a register
// and re-materialises it per plane: +28 instructions per visit).
template <int K> TGB_D float qplane(uint32_t w, uint32_t y) {
    uint32_t r;
    if (K == 0) asm("prmt.b32 %0, %1, %2, 0x5406;" : "=r"(r) : "r"(w), "r"(y));
    else if (K == 1) asm("prmt.b32 %0, %1, %2, 0x5416;" : "=r"(r) : "r"(w), "r"(y));
    else if (K == 2) asm("prmt.b32 %0, %1, %2, 0x5426;" : "=r"(r) : "r"(w), "r"(y));
    else asm("prmt.b32 %0, %1, %2, 0x5436;" : "=r"(r) : "r"(w), "r"(y));
    return __uint_as_float(r);
}
#define TGB_QF(W, K) qplane<K>(W, qy)
// CURVES: leaves whose code has bit 2 set hold curve segments (three float4 nodes per record, stored after the triangles);
// a curve hit keeps (t, position along the segment, interpolated width) in (t, u, v) and id >= n_tris.
// One lane's ray and its node / primitive tests; bvh_traverse_persistent drives it.
template <bool CURVES>
struct Traversal {
    V3 o, d; float tnear; bool any; Hit h;
    float idx, idy, idz, oodx, oody, oodz; int nx, ny, nz;
    CurveFrame cf; int last_seg; int cur;
    int ignore;         // analytic primitive an occlusion query must not count (the light it is aimed at), -1 = none
    // (the stack is a separate object: its dynamically indexed spill array would drag this whole struct into local memory)

    TGB_D void begin(V3 o_, V3 d_, float tnear_, bool any_, const Hit &h_) {
        o = o_; d = d_; tnear = tnear_; any = any_; h = h_;
        const float ooeps = 1e-30f;
        idx = 1.0f/(fabsf(d.x) > ooeps ? d.x : copysignf(ooeps, d.x));
        idy = 1.0f/(fabsf(d.y) > ooeps ? d.y : copysignf(ooeps, d.y));
        idz = 1.0f/(fabsf(d.z) > ooeps ? d.z : copysignf(ooeps, d.z));
        oodx = o.x*idx; oody = o.y*idy; oodz = o.z*idz;
        // The entry plane of a slab is its lo plane when the direction component is positive, else its hi plane (fma is
        // monotone, so this IS min(a, b) / max(a, b) of the two plane distances): pick which to read per axis once per ray.
        nx = idx < 0.0f ? 1 : 0; ny = idy < 0.0f ? 3 : 2; nz = idz < 0.0f ? 5 : 4;
        last_seg = -1; ignore = -1;
        if (CURVES) cf = curve_frame(d);
        cur = 0;
    }

    // one node visit: entry distances of the four children (INFINITY = culled) and their links
    TGB_D void visit(const DScene &sc, float &t0, float &t1, float &t2, float &t3, int4 &lk) {
        const uint4 *nd = sc.qnodes + 4*size_t(cur);
        const uint4 c0 = __ldg(nd), c1 = __ldg(nd + 1), c2 = __ldg(nd + 2); lk = __ldg(reinterpret_cast<const int4 *>(nd + 3));
        const float ax_ = __uint_as_float(c0.w)*idx, ay_ = __uint_as_float(c1.x)*idy, az_ = __uint_as_float(c1.y)*idz;
        const float bx_ = __fmaf_rn(__uint_as_float(c0.x), idx, -oodx) - ax_;
        const float by_ = __fmaf_rn(__uint_as_float(c0.y), idy, -oody) - ay_;
        const float bz_ = __fmaf_rn(__uint_as_float(c0.z), idz, -oodz) - az_;
        const uint32_t qy = sc.qy;          // 0x3F80 from the kernel parameters: a value ptxas cannot fold into the PRMT as an immediate
        const uint32_t nxw = nx ? c1.w : c1.z, fxw = nx ? c1.z : c1.w;
        const uint32_t nyw = (ny & 1) ? c2.y : c2.x, fyw = (ny & 1) ? c2.x : c2.y;
        const uint32_t nzw = (nz & 1) ? c2.w : c2.z, fzw = (nz & 1) ? c2.z : c2.w;
#define TGB_SLAB(K, LK, OUT) { \
            float ax = __fmaf_rn(TGB_QF(nxw, K), ax_, bx_), bx = __fmaf_rn(TGB_QF(fxw, K), ax_, bx_); \
            float ay = __fmaf_rn(TGB_QF(nyw, K), ay_, by_), by = __fmaf_rn(TGB_QF(fyw, K), ay_, by_); \
            float az = __fmaf_rn(TGB_QF(nzw, K), az_, bz_), bz = __fmaf_rn(TGB_QF(fzw, K), az_, bz_); \
            float tmn = fmaxf(fmaxf(fmaxf(ax, ay), az), tnear); float tmx = fminf(fminf(fminf(bx, by), bz), h.t); \
            OUT = tmn <= tmx ? tmn : INFINITY; }
        // (an empty child slot holds the inverted box lo = 255, hi = 0: its entry distance exceeds its exit distance by 255
        // grid steps for every ray, so it needs no test of its own)
        TGB_SLAB(0, lk.x, t0) TGB_SLAB(1, lk.y, t1) TGB_SLAB(2, lk.z, t2) TGB_SLAB(3, lk.w, t3)
#undef TGB_SLAB
    }

    // Moeller-Trumbore on leaf-order record k (a, b, c = its three float4); true (and h updated) when it is hit closer than h.t
    TGB_D bool triangle(const float4 a, const float4 b, const float4 c, int k) {
        V3 v0 = v3(a.x, a.y, a.z), e1 = v3(a.w, b.x, b.y), e2 = v3(b.z, b.w, c.x), ng = v3(c.y, c.z, c.w);
        V3 C = v0 - o;
        V3 R = cross(d, C);
        float den = edot(ng, d);
        float absDen = fabsf(den);
        uint32_t sgn = __float_as_uint(den) & 0x80000000u;
        float U = xor_sign(edot(R, e2), sgn);
        float V = xor_sign(edot(R, e1), sgn);
        if (!(den != 0.0f && U >= 0.0f && V >= 0.0f && U + V <= absDen)) return false;
        float T = xor_sign(edot(ng, C), sgn);
        if (!(T > absDen*tnear && T < absDen*h.t)) return false;
        h.t = T/absDen; h.u = U/absDen; h.v = V/absDen; h.id = k;
        return true;
    }

    // leaf of analytic primitives (scenes with many quads / cubes keep them in the BVH): Quad::intersect / Cube::intersect on the
    // primitives at leaf positions first .. first + count; true when an occlusion query is done
    TGB_D bool analytic_leaf(const DScene &sc, int first, int count) {
        for (int i = 0; i < count; ++i) {
            const int pi = __ldg(sc.analytic + (first - sc.analytic_base) + i);
            if (pi == ignore) continue;
            const DPrim &p = sc.prims[pi];
            const int before = h.id;
            if (p.type == TGB_PRIM_QUAD) quad_intersect(p, pi, o, d, tnear, h);
            else cube_intersect(p, pi, o, d, tnear, h);
            if (any && h.id != before) return true;
        }
        return false;
    }
};

// Persistent form used by the renderer's traversal kernels: a fixed grid of warps pulls rays from a shared counter, and
// each warp runs a STATE MACHINE over its lanes' rays.  A ray's traversal length is heavy-tailed, and a segment test is a
// data-dependent bisection of 1..63 steps: with a per-lane walk the kernel was issue bound with a few of 32 threads active
// per instruction -- every lane waiting for the warp's longest ray or bisection.  Here each lane is in one of four states and
// every trip of the loop runs ONE block of code for all the lanes that are in the state most lanes are in:
//      NODE    one 4-ary node visit                          LEAF   next primitive of the leaf: triangle tests, or the set-up
//      BISECT  one step of pointOnSpline (box test, split     CYL    intersectHalfCylinder of a depth-5 piece, then pop
//              or pop)
// so a lane in a long bisection no longer stalls the others: they go on visiting nodes and starting their own segment tests in
// the same trips.  A ray's arithmetic and the order of ITS node visits / segment tests are unchanged (parity unaffected).
// Once enough lanes are idle, the warp pulls the next rays of the (coherence-sorted) queue into them.
// resident blocks the CURVE instantiations of the traversal kernels are compiled for (4 x 128 threads: up to 128 registers; the
// state machine keeps a ray's traversal AND bisection state live, and it is issue bound, not latency bound)
#ifndef TGB_MINB_CURVES
#define TGB_MINB_CURVES 5
#endif
// idle lanes a warp tolerates before it pulls new rays
#ifndef TGB_CURVE_REFILL_IDLE
#define TGB_CURVE_REFILL_IDLE 8
#endif
#ifndef TGB_TRI_REFILL_IDLE
#define TGB_TRI_REFILL_IDLE 16
#endif
enum : int { CM_IDLE = 0, CM_NODE = 1, CM_LEAF = 2, CM_BISECT = 3, CM_CYL = 4 };
// ANY (k_shadow_bvh's any-hit queries only): an occlusion query's answer -- is there any primitive in [tnear, t_light]? -- does not
// depend on the order of its node visits nor on where its walk starts, so this walk skips the near-to-far sort (the nearest hit child
// is entered, the others are pushed unsorted) and starts below the top-level cut (pol.enter pushes the subtrees of the cut boxes the
// segment enters).  A closest-hit walk cannot do either: the visiting order decides which of two equally distant hits wins.
template <bool CURVES, bool ANY = false, class P>
TGB_D void bvh_traverse_persistent(const DScene &sc, int *smem_stack, P &pol, uint32_t n, uint32_t *counter) {
    const unsigned FULL = 0xffffffffu, lane = threadIdx.x & 31u;
    Traversal<CURVES> tr; TravStack stk; stk.base = smem_addr(smem_stack + threadIdx.x); int sp = 0;
    int mode = CM_IDLE; bool exhausted = false;
    int li = 0, prim = 0; bool seg_hit = false;                                        // leaf cursor, BVH primitive under test
    float4 q0 = {}, q1 = {}, q2 = {}, c0 = {}, c1 = {};                                 // the segment's quadratic, the current piece's end points
    float tFlatX = 0.0f, tFlatY = 0.0f, xFlat = 0.0f, yFlat = 0.0f, pMin = 0.0f, pMax = 1.0f;
    uint32_t bidx = 0, pending = 0; int depth = 0;                                      // piece = [bidx, bidx + 1]/2^depth; pending siblings by depth
    auto finish_ray = [&]() { pol.finish(tr.h); mode = CM_IDLE; };
    auto pop_node = [&]() {                                                             // leave a leaf: next stack entry or done
        if (sp == 0) { finish_ray(); return; }
        tr.cur = stk.pop(sp); li = 0; mode = tr.cur >= 0 ? CM_NODE : CM_LEAF;
    };
    // box test of pointOnSpline's loop head for the piece (a, b) = the curve on [ta, tb]
    auto piece_box = [&](const float4 &a, const float4 &b, float ta, float tb) {
        float mnx = b.x < a.x ? b.x : a.x, mny = b.y < a.y ? b.y : a.y;
        float mxx = b.x > a.x ? b.x : a.x, mxy = b.y > a.y ? b.y : a.y;
        if (tFlatX > ta && tFlatX < tb) { mnx = minf(mnx, xFlat); mxx = maxf(mxx, xFlat); }
        if (tFlatY > ta && tFlatY < tb) { mny = minf(mny, yFlat); mxy = maxf(mxy, yFlat); }
        const float mw = maxf(a.w, b.w);
        return mnx <= mw && mny <= mw && mxx >= -mw && mxy >= -mw;
    };
    // The do-while at the end of pointOnSpline's loop.  Only pieces whose box test passed are ever marked pending (the test does
    // not depend on the closest hit, so it is made when the parent is split), hence a popped piece goes straight on.
    auto pop_piece = [&]() {
        do {
            if (pending == 0) {                                                          // segment finished
                if (seg_hit && tr.any) finish_ray(); else mode = CM_LEAF;
                return;
            }
            const int L = 31 - __clz(pending); pending ^= 1u << L;
            bidx = (bidx >> (depth - L)) ^ 1u; depth = L;
            const float scale = __uint_as_float(uint32_t(127 - L) << 23);                // 2^-L
            pMin = float(bidx)*scale; pMax = float(bidx + 1)*scale;
            const float4 e0 = curve_eval(q0, q1, q2, pMin);
            c0 = bidx == 0 ? q2 : e0;
            c1 = curve_eval(q0, q1, q2, pMax);
        } while (minf(c0.z - c0.w, c1.z - c1.w) > tr.h.t);
        mode = depth >= 5 ? CM_CYL : CM_BISECT;
    };
    for (;;) {
        const unsigned idle = __ballot_sync(FULL, mode == CM_IDLE);
        if (!exhausted && __popc(idle) >= (CURVES ? TGB_CURVE_REFILL_IDLE : TGB_TRI_REFILL_IDLE)) {
            const uint32_t cnt = unsigned(__popc(idle)), leader = unsigned(__ffs(int(idle))) - 1u;
            const uint32_t rank = unsigned(__popc(idle & ((1u << lane) - 1u)));
            uint32_t first_ray = 0;
            if (lane == leader) first_ray = atomicAdd(counter, cnt);
            first_ray = __shfl_sync(FULL, first_ray, int(leader));
            exhausted = first_ray + cnt >= n;
            if (mode == CM_IDLE && rank < cnt && first_ray + rank < n) {
                V3 o, d; float tnear; Hit h; bool any;
                if (pol.fetch(first_ray + rank, o, d, tnear, h, any)) {
                    tr.begin(o, d, tnear, any, h); tr.ignore = pol.ignore(); sp = 0; mode = CM_NODE;
                    if constexpr (ANY) { pol.enter(stk, sp); pop_node(); }
                }
            }
            continue;
        }
        if (idle == FULL) break;                                                        // (only reached once the cursor is exhausted)
        // the block most lanes are in runs (ties: BISECT, CYL, NODE, LEAF); triangle scenes have no curve states
        const int sN = __popc(__ballot_sync(FULL, mode == CM_NODE)), sL = __popc(__ballot_sync(FULL, mode == CM_LEAF));
        const int sB = CURVES ? __popc(__ballot_sync(FULL, mode == CM_BISECT)) : -1, sC = CURVES ? __popc(__ballot_sync(FULL, mode == CM_CYL)) : -1;
        const int best = max(max(sN, sL), max(sB, sC));
        if (CURVES && sB == best) {
            // BISECT: split a piece that passed its box test (depth < 5) and test BOTH halves: the near half is entered if it
            // passes, the far half is marked pending if it passes (the reference pushes it untested and tests it when popped;
            // a failing piece has no side effect, so dropping it here changes nothing).  With only the far half left it is
            // entered the way the reference reaches it -- through a pop, i.e. after the pruning comparison.
            if (mode == CM_BISECT) {
                const float splitT = (pMin + pMax)*0.5f;
                const float4 qS = curve_eval(q0, q1, q2, splitT);
                const bool first_near = c0.z < qS.z;
                const bool passA = piece_box(c0, qS, pMin, splitT), passB = piece_box(qS, c1, splitT, pMax);
                const bool passN = first_near ? passA : passB, passF = first_near ? passB : passA;
                depth++;
                bool second = !first_near;                                              // which half becomes the current piece
                bool enter = passN;
                if (passN) { if (passF) pending |= 1u << depth; }
                else if (passF) {
                    second = first_near;
                    const float4 f0 = second ? qS : c0, f1 = second ? c1 : qS;
                    enter = !(minf(f0.z - f0.w, f1.z - f1.w) > tr.h.t);
                }
                bidx = 2*bidx + (second ? 1u : 0u);
                if (enter) {
                    if (second) { pMin = splitT; c0 = qS; } else { pMax = splitT; c1 = qS; }
                    if (depth >= 5) mode = CM_CYL;
                } else pop_piece();
            }
        } else if (CURVES && sC == best) {
            if (mode == CM_CYL) {
                CurvePiece pc; pc.p0 = c0; pc.p1 = c1; pc.tMin = pMin; pc.tMax = pMax; pc.depth = depth;
                const float before = tr.h.t;
                float ht = 0.0f, hu = 0.0f, hw = 0.0f, closest = before;
                curve_half_cylinder(pc, tr.tnear, closest, ht, hu, hw);
                if (closest != before) { tr.h.t = ht; tr.h.u = hu; tr.h.v = hw; tr.h.id = prim; seg_hit = true; }
                pop_piece();
            }
        } else if (sN == best) {
            if (mode == CM_NODE) {
                float t0, t1, t2, t3; int4 lk;
                tr.visit(sc, t0, t1, t2, t3, lk);
                int l0 = lk.x, l1 = lk.y, l2 = lk.z, l3 = lk.w;
                // the first three exchanges leave the nearest child in slot 0; the last two sort the other three
                TGB_CSWAP(t0, l0, t1, l1) TGB_CSWAP(t2, l2, t3, l3) TGB_CSWAP(t0, l0, t2, l2)
                if (!ANY) { TGB_CSWAP(t1, l1, t3, l3) TGB_CSWAP(t1, l1, t2, l2) }
                if (t0 == INFINITY) pop_node();
                else {
                    // closest hit: sorted, so the nearest of the pushed children ends up on top
                    const bool p1 = t1 != INFINITY, p2 = t2 != INFINITY, p3 = t3 != INFINITY;
                    if (sp + 3 <= kSmemStack) {
                        const uint32_t a3 = stk.base + uint32_t(sp)*(kTraceBlock*4u);
                        const uint32_t a2 = a3 + (p3 ? kTraceBlock*4u : 0u), a1 = a2 + (p2 ? kTraceBlock*4u : 0u);
                        if (p3) TravStack::sts(a3, l3);
                        if (p2) TravStack::sts(a2, l2);
                        if (p1) TravStack::sts(a1, l1);
                        sp += int(p1) + int(p2) + int(p3);
                    } else {
                        if (p3) stk.push(sp, l3);
                        if (p2) stk.push(sp, l2);
                        if (p1) stk.push(sp, l1);
                    }
                    tr.cur = l0;
                    if (l0 < 0) { mode = CM_LEAF; li = 0; }
                }
            }
        } else {
            if (mode == CM_LEAF) {
                const int code = ~tr.cur, first = code >> 3, count = (code & 3) + 1;
                if ((code & 4) && (!CURVES || first >= sc.analytic_base)) {
                    if (tr.analytic_leaf(sc, first, count)) finish_ray(); else pop_node();
                } else if (CURVES && (code & 4)) {
                    bool started = false;
                    while (li < count) {
                        const int i = li++;
                        const int seg = int(__ldg(sc.tri_global + first + i) - sc.n_tris)/kCurvePieces;
                        if (seg == tr.last_seg) continue;
                        tr.last_seg = seg;
                        const float4 *cr = sc.tri_isect + 3*size_t(first + i);
                        const float4 p0 = curve_project(tr.o, tr.cf, tr.d, __ldg(cr)), p1 = curve_project(tr.o, tr.cf, tr.d, __ldg(cr + 1)), p2 = curve_project(tr.o, tr.cf, tr.d, __ldg(cr + 2));
                        q0 = f4add(f4sub(f4scale(p0, 0.5f), p1), f4scale(p2, 0.5f));
                        q1 = f4sub(p1, p0);
                        q2 = f4scale(f4add(p0, p1), 0.5f);
                        tFlatX = -q1.x*0.5f/q0.x; tFlatY = -q1.y*0.5f/q0.y;
                        xFlat = q0.x*tFlatX*tFlatX + q1.x*tFlatX + q2.x;
                        yFlat = q0.y*tFlatY*tFlatY + q1.y*tFlatY + q2.y;
                        c0 = q2; c1 = f4add(f4add(q0, q1), q2); pMin = 0.0f; pMax = 1.0f; depth = 0; bidx = 0; pending = 0;
                        if (!piece_box(c0, c1, 0.0f, 1.0f)) continue;                    // the whole segment misses: nothing else happens in pointOnSpline
                        prim = first + i; seg_hit = false; mode = CM_BISECT; started = true;
                        break;
                    }
                    if (!started) pop_node();
                } else {
                    // two records in flight: the second triangle's loads are issued before the first is tested
                    bool hit_any = false;
                    for (int i = 0; i < count && !hit_any; i += 2) {
                        const float4 *t = sc.tri_isect + 3*size_t(first + i);
                        const bool two = i + 1 < count;
                        const float4 a0 = __ldg(t), b0 = __ldg(t + 1), c0 = __ldg(t + 2);
                        const float4 a1 = __ldg(t + (two ? 3 : 0)), b1 = __ldg(t + (two ? 4 : 1)), c1 = __ldg(t + (two ? 5 : 2));
                        hit_any = tr.triangle(a0, b0, c0, first + i) && tr.any;
                        if (two && !hit_any) hit_any = tr.triangle(a1, b1, c1, first + i + 1) && tr.any;
                    }
                    if (hit_any) finish_ray(); else pop_node();
                }
            }
        }
    }
}

// Coherent pre-test of a new ray against the BVH's top-level cut (DScene::cut), with fused slab arithmetic on the float
// boxes the tree was built from (the quantised node boxes contain them): false means every subtree would be culled, i.e.
// the query's answer is the ray's analytic hit.  MASK: the set of boxes entered instead (bit k = box k), where an any-hit walk starts.
// TODO(open item, tests/test_gpu_tree_shapes.py CUT_DROPS): a curve's half-cylinder piece accepts hits on the extension of its chord,
// which can lie outside the segment's box and so outside every cut box; the full traversal (looser quantised boxes) finds a few such
// hits that this pre-test drops, so k_trace and tgb200_trace_closest with TGB_HOOK_CUT=0 differ on them.
template <bool MASK>
TGB_D uint32_t mesh_cut_test(const DScene &sc, V3 o, V3 d, float tnear, float tfar) {
    const float ooeps = 1e-30f;
    const float idx = 1.0f/(fabsf(d.x) > ooeps ? d.x : copysignf(ooeps, d.x));
    const float idy = 1.0f/(fabsf(d.y) > ooeps ? d.y : copysignf(ooeps, d.y));
    const float idz = 1.0f/(fabsf(d.z) > ooeps ? d.z : copysignf(ooeps, d.z));
    const float oodx = o.x*idx, oody = o.y*idy, oodz = o.z*idz;
    bool hit = false; uint32_t mask = 0;
    // groups of four boxes with static indices inside a group (the boxes are read straight from the kernel parameters); the
    // number of groups is uniform across the grid
#pragma unroll
    for (int g = 0; g < 4; ++g) {
        if (4*g < sc.n_cut) {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int k = 4*g + j;
                float ax = __fmaf_rn(sc.cut[0][k], idx, -oodx), bx = __fmaf_rn(sc.cut[1][k], idx, -oodx);
                float ay = __fmaf_rn(sc.cut[2][k], idy, -oody), by = __fmaf_rn(sc.cut[3][k], idy, -oody);
                float az = __fmaf_rn(sc.cut[4][k], idz, -oodz), bz = __fmaf_rn(sc.cut[5][k], idz, -oodz);
                float tmn = fmaxf(fmaxf(fminf(ax, bx), fminf(ay, by)), fmaxf(fminf(az, bz), tnear));
                float tmx = fminf(fminf(fmaxf(ax, bx), fmaxf(ay, by)), fminf(fmaxf(az, bz), tfar));
                if (MASK) mask |= (k < sc.n_cut && tmn <= tmx) ? 1u << k : 0u;
                else hit = hit || (k < sc.n_cut && tmn <= tmx);
            }
        }
    }
    return MASK ? mask : uint32_t(hit);
}
TGB_D bool mesh_cut_hit(const DScene &sc, V3 o, V3 d, float tnear, float tfar) { return mesh_cut_test<false>(sc, o, d, tnear, tfar) != 0; }

// Fill a Surface from a hit: Primitive::intersectionInfo for mesh/quad/cube
// (TriangleMesh.cpp:323-331,344-355; Quad.cpp:112-120; Cube.cpp:157-171) + TraceableScene::intersect (:183-188)
template <bool CURVES>
TGB_D void make_surface(const DScene &sc, const Hit &h, V3 o, V3 d, Surface &s) {
    s.p = o + d*h.t;
    s.w = d;
    s.eps = 5e-4f; s.curve = false;
    if (CURVES && h.id >= int(sc.n_tris)) {
        // Curves::intersectionInfo (primitives/Curves.cpp:484-516); the record holds the segment's three nodes
        uint32_t g = __ldg(sc.tri_global + h.id);
        int pi = int(__ldg(sc.tri_prim + g));
        const DPrim &c = sc.prims[pi];
        s.prim = pi; s.curve = true; s.backside = false;
        const float4 *cr = sc.tri_isect + 3*size_t(h.id);
        const float4 n0 = __ldg(cr), n1 = __ldg(cr + 1), n2 = __ldg(cr + 2);
        float t = h.u;
        V3 a0 = v3(n0.x, n0.y, n0.z), a1 = v3(n1.x, n1.y, n1.z), a2 = v3(n2.x, n2.y, n2.z);
        s.tangent = (a0 - a1*2.0f + a2)*t + (a1 - a0);                                       // BSpline::quadraticDeriv
        V3 tangent = normalize(s.tangent);
        if (c.curve_mode == TGB_CURVE_BCSDF_CYLINDER) {
            V3 mw = -d;
            s.Ng = s.Ns = normalize(mw - tangent*dot(tangent, mw));
        } else {
            V3 point = (a0*0.5f - a1 + a2*0.5f)*t*t + (a1 - a0)*t + (a0 + a1)*0.5f;          // BSpline::quadratic
            V3 localP = s.p - point;
            localP = localP - tangent*dot(localP, tangent);
            s.Ng = s.Ns = normalize(localP);
        }
        s.u = h.u; s.v = 0.5f;            // CurveIntersection::uv.y (distance across the strand) is not kept: constant textures only
        s.bsdf = int(__ldg(sc.slots + c.bsdf_first));
        s.eps = maxf(s.eps, (c.curve_mode == TGB_CURVE_CYLINDER ? 0.1f : 0.01f)*h.v);
    } else if (h.id >= 0) {
        // shading record of the triangle, stored in BVH leaf order like the intersection records: one hop from the hit id
        // (no leaf order -> triangle id -> primitive chain of dependent gathers); its last word packs material | primitive << 10
        const float4 *sh = sc.tri_shade + 4*size_t(h.id);
        const float4 s0 = __ldg(sh), s1 = __ldg(sh + 1), s2 = __ldg(sh + 2), s3 = __ldg(sh + 3);
        const float4 c = __ldg(sc.tri_isect + 3*size_t(h.id) + 2);
        const uint32_t packed = __float_as_uint(s3.w);
        int pi = int(packed >> 10);
        const DPrim &m = sc.prims[pi];
        s.prim = pi;
        // (p1-p0)x(p2-p0) == -(e1 x e2) exactly (e1 = p0-p1, e2 = p2-p0; negation is exact in IEEE)
        V3 isectNg = v3(-c.y, -c.z, -c.w);
        s.backside = dot(isectNg, d) > 0.0f;
        s.Ng = normalize(isectNg);
        float u = h.u, v = h.v;
        if (m.flags & PF_SMOOTH) {
            V3 n0 = v3(s0.x, s0.y, s0.z), n1 = v3(s0.w, s1.x, s1.y), n2 = v3(s1.z, s1.w, s2.x);
            s.Ns = normalize(n0*(1.0f - u - v) + n1*u + n2*v);
        } else s.Ns = s.Ng;
        float w0 = 1.0f - u - v;
        s.u = w0*s2.y + u*s2.w + v*s3.y;
        s.v = w0*s2.z + u*s3.x + v*s3.z;
        int mat = int(packed & 1023u);
        s.bsdf = int(__ldg(sc.slots + m.bsdf_first + mat));
    } else {
        int pi = -h.id - 2;
        const DPrim &p = sc.prims[pi];
        s.prim = pi;
        s.bsdf = int(__ldg(sc.slots + p.bsdf_first));
        if (p.type == TGB_PRIM_QUAD) {
            s.Ng = s.Ns = p.normal; s.u = h.u; s.v = h.v;
            s.backside = dot(d, p.normal) >= 0.0f;
        } else {
            V3 q = m3mul(p.inv_rot, s.p - p.pos);
            V3 dd = vabs(q) - p.scale;
            int dim = 0; float mx = dd.x; if (dd.y > mx) { mx = dd.y; dim = 1; } if (dd.z > mx) { mx = dd.z; dim = 2; }
            float sgn = comp(q, dim) < 0.0f ? -1.0f : 1.0f;
            V3 n = v3(dim == 0 ? sgn : 0.0f, dim == 1 ? sgn : 0.0f, dim == 2 ? sgn : 0.0f);
            V3 uvw = v3((q.x/p.scale.x)*0.5f + 0.5f, (q.y/p.scale.y)*0.5f + 0.5f, (q.z/p.scale.z)*0.5f + 0.5f);
            s.Ns = s.Ng = m3mul(p.rot, n);
            s.u = comp(uvw, (dim + 1) % 3); s.v = comp(uvw, (dim + 2) % 3);
            s.backside = h.u != 0.0f;
        }
    }
}

// Primitive::evalDirect (Quad.cpp:235-238, TriangleMesh.cpp:493-496, Cube evalDirect); ES: the emitter set (light_sample_direct)
template <int ES = 0>
TGB_D V3 eval_direct(const DScene &sc, const Surface &s) {
    const DPrim &p = sc.prims[s.prim];
    if (p.emission_tex < 0 || s.backside) return v3s(0.0f);
    return tex_eval<ES == 1>(sc.tex[p.emission_tex], s.u, s.v);
}

// light.intersect(ray) for a quad light, resolved in the shading kernel (Quad.cpp:71-99 on the light alone,
// as TraceBase::attenuatedEmission does at TraceBase.cpp:160) so that the traced query is a pure occlusion test.
TGB_D bool quad_light_hit(const DPrim &l, V3 p, V3 d, float tnear, float &t, float &l0, float &l1, bool &backside) {
    float nDotW = dot(d, l.normal);
    if (fabsf(nDotW) < 1e-6f) return false;
    t = dot(l.normal, l.base - p)/nDotW;
    if (t < tnear) return false;
    V3 v = (p + d*t) - l.base;
    l0 = dot(v, l.edge0)*l.inv_uv_sq0;
    l1 = dot(v, l.edge1)*l.inv_uv_sq1;
    if (l0 < 0.0f || l0 > 1.0f || l1 < 0.0f || l1 > 1.0f) return false;
    backside = nDotW >= 0.0f;
    return true;
}

// attenuatedEmission's light.intersect + evalDirect (TraceBase.cpp:160-165) and the light's directPdf along d from p, for a quad,
// infinite sphere cap or environment light (Quad.cpp:216-222,235-238; InfiniteSphereCap.cpp:173-177; InfiniteSphere.cpp:218-229,
// 241-244).  A quad hit closer than expected_dist/(1 + 1e-3) is a miss (the NEE query passes the sampled distance, the BSDF-sampled
// query -1).  Returns whether the light is hit; tfar = its distance (INFINITY for the infinite lights).
template <int ES = 0>
TGB_D bool light_hit_direct(const DScene &sc, const DPrim &l, V3 p, V3 d, float epsilon, float expected_dist, V3 &em, float &tfar,
                            float &direct_pdf) {
    em = v3s(0.0f); tfar = INFINITY;
    bool hitL = true;
    if (ES == 1 || l.type == TGB_PRIM_QUAD) {
        float t, l0, l1; bool back;
        hitL = quad_light_hit(l, p, d, epsilon, t, l0, l1, back) && !(t*(1.0f + 1e-3f) < expected_dist);
        if (hitL && !back) em = tex_eval<ES == 1>(sc.tex[l.emission_tex], l0, l1);
        tfar = t;
        direct_pdf = t*t/(fabsf(dot(l.normal, d))*l.area);
    } else if (l.type == TGB_PRIM_INFINITE_SPHERE_CAP) {
        hitL = cap_hit(l, d);
        if (hitL) em = tex_eval(sc.tex[l.emission_tex], 0.0f, 0.0f);                    // InfiniteSphereCap::evalDirect looks up uv (0, 0)
        direct_pdf = INV_TWO_PI_F/(1.0f - l.area);
    } else {
        float u, v, sinTheta; direction_to_uv(l, d, u, v, &sinTheta);
        const DTex &et = sc.tex[l.emission_tex];
        em = tex_eval(et, u, v);
        direct_pdf = et.type == TGB_TEX_CONSTANT ? INV_FOUR_PI_F : INV_PI_F*INV_TWO_PI_F*bitmap_pdf_uv(et, u, v)/sinTheta;
    }
    return hitL;
}
// TriangleMesh::directPdf (TriangleMesh.cpp:477-481) from the light's hit ls, seen along d from p
TGB_D float mesh_direct_pdf(const DPrim &l, V3 p, V3 d, const Surface &ls) {
    return length_sq(p - ls.p)/(-dot(d, ls.Ng)*l.total_area);
}
// The shadow query of one NEE (mis = false: lightSample, TraceBase.cpp:246-285) or MIS (bsdfSample, :287-321) estimate towards
// light l, as k_shade emits it; true when there is a query to trace.  f = the BSDF value (NEE) or sample weight (MIS), pdf = pdfL
// (NEE) or the BSDF sample's pdf (MIS), pdf_b = NEE's BSDF pdf, dist = the sampled distance (NEE).
//  * quad, cap and environment lights: the light's own hit is resolved here (light_hit_direct), lightF / bsdfF are finished into
//    x.xyz and the query is a blocker test up to the light (any = true, t = its distance); none when the light is missed or
//    emits nothing along d;
//  * mesh lights: a closest-hit query that shadow_resolve_closest finishes: x = (f, pdfL) (NEE) or x.xyz = weight (MIS), t = the
//    sampled distance (NEE) or the BSDF pdf (MIS).
// The MIS query keeps x.w (NEE's pdfB shares that record).
template <int ES = 0>
TGB_D bool light_query(const DScene &sc, const DPrim &l, V3 p, V3 d, float epsilon, bool mis, V3 f, float pdf, float pdf_b,
                       float dist, float4 &x, float &t, bool &any) {
    if (ES == 0 && l.type == TGB_PRIM_MESH) {
        any = false; x = make_float4(f.x, f.y, f.z, mis ? x.w : pdf); t = mis ? pdf : dist;
        return true;
    }
    V3 em; float tfar, directPdf;
    const bool hitL = light_hit_direct<ES>(sc, l, p, d, epsilon, mis ? -1.0f : dist, em, tfar, directPdf);
    if (!hitL || is_zero(em)) return false;
    V3 r;
    if (mis) { r = em*f; r = r*power_heuristic(pdf, directPdf); }
    else { r = (f*em)/pdf; r = r*power_heuristic(pdf, pdf_b); }
    any = true; x = make_float4(r.x, r.y, r.z, mis ? x.w : 0.0f); t = tfar;
    return true;
}

TGB_D float4 pack_hit(const Hit &h) { return make_float4(h.t, h.u, h.v, __int_as_float(h.id)); }
TGB_D Hit unpack_hit(float4 v) { Hit h; h.t = v.x; h.u = v.y; h.v = v.z; h.id = __float_as_int(v.w); return h; }

// Ray-coherence key of a path ray: direction octant (3 bits) + origin cell on a 16^3 grid over the scene bounds (12 bits).
// k_trace visits the survivors in key order (counting sort of slot indices: k_accum histogram, k_bin_scan, k_bin_scatter),
// so the lanes of a warp start close together and walk the BVH in the same front-to-back order; only the 48 bytes of
// packed ray + hit record are gathered through the index, all other state stays in slot order (coalesced).
constexpr uint32_t kBinBits = 15, kBins = 1u << kBinBits;
TGB_D uint32_t ray_bin(const DScene &sc, V3 o, V3 d) {
    uint32_t oct = (d.x < 0.0f ? 1u : 0u) | (d.y < 0.0f ? 2u : 0u) | (d.z < 0.0f ? 4u : 0u);
    int cx = min(max(int((o.x - sc.bin_lo.x)*sc.bin_inv.x), 0), 15);
    int cy = min(max(int((o.y - sc.bin_lo.y)*sc.bin_inv.y), 0), 15);
    int cz = min(max(int((o.z - sc.bin_lo.z)*sc.bin_inv.z), 0), 15);
    return (oct << 12) | (uint32_t(cx) << 8) | (uint32_t(cy) << 4) | uint32_t(cz);       // (Morton order of the cell: no gain)
}
// ---- kernels ---------------------------------------------------------------------------------
// One render call = a list of pixels (tile-major) x a sample range per pixel.  Uniform steps give every pixel the samples
// [spp_begin, spp_begin + ns); adaptive steps (PathTraceIntegrator::generateWork, PathTraceIntegrator.cpp:110-134) give the
// pixels of each 4x4 block their own count and first sample index.  The host renders a call in passes (sample ranges, or runs
// of tiles for adaptive steps), and a BatchInfo describes one pass.  A path carries (k << pix_bits) | pixel_list_index, k = its
// sample's position within the pass; its result slot is k*n_pix + pix (uniform) or pix_first[pix] + k (adaptive).
struct BatchInfo {
    const uint32_t *pix_id, *pix_seed; uint32_t n_pix, spp_begin;
    const uint32_t *pix_first, *pix_base;       // adaptive only (else nullptr): n_pix + 1 result-slot offsets, first sample index per pixel
    uint32_t pix_bits;
};
TGB_D void path_decode(const BatchInfo &bi, uint32_t packed, uint32_t &pix, uint32_t &k) { pix = packed & ((1u << bi.pix_bits) - 1u); k = packed >> bi.pix_bits; }
TGB_D uint32_t path_sample_index(const BatchInfo &bi, uint32_t pix, uint32_t k) { return (bi.pix_base ? __ldg(bi.pix_base + pix) : bi.spp_begin) + k; }
TGB_D size_t path_result_slot(const BatchInfo &bi, uint32_t pix, uint32_t k) { return bi.pix_first ? size_t(__ldg(bi.pix_first + pix)) + k : size_t(k)*bi.n_pix + pix; }

// Path (re)generation: the ctl.n_new camera paths [first_path, first_path + n_new) of the step start in slots
// [n_surv, n_surv + n_new), right behind the survivors that k_accum compacted to the front of the same buffer.  Consecutive
// slots are neighbouring pixels of one sample index, so the primary rays stay coherent and every state access is coalesced.
// = SobolPathSampler::startPath + ReconstructionFilter::sample + PinholeCamera::sampleDirection + the analytic
// part of the first TraceableScene::intersect.  Also clears the ray-coherence histogram for this iteration's k_accum.
// The grid is what is resident at once (or less), each thread loops over the slots j, j + grid size, ...
__global__ void __launch_bounds__(256) k_regen(DScene sc, PathBuf pb, BatchInfo bi, const Ctl *ctl, uint32_t *order, uint32_t *hist) {
    const uint32_t stride = gridDim.x*blockDim.x;
    for (uint32_t k = blockIdx.x*blockDim.x + threadIdx.x; k < kBins; k += stride) hist[k] = 0u;
    const uint32_t n_new = ctl->n_new, n_surv = ctl->n_surv, first_path = ctl->first_path;
    for (uint32_t j = blockIdx.x*blockDim.x + threadIdx.x; j < n_new; j += stride) {
    const uint32_t i = n_surv + j;
    const uint32_t path = first_path + j;
    uint32_t pix, k;
    if (!bi.pix_first) { pix = path % bi.n_pix; k = path/bi.n_pix; }
    else {                                              // adaptive: the pixel whose result slots contain `path`
        uint32_t lo = 0, hi = bi.n_pix;                 // pix_first[lo] <= path < pix_first[hi]
        while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (__ldg(bi.pix_first + mid) <= path) lo = mid; else hi = mid; }
        pix = lo; k = path - __ldg(bi.pix_first + lo);
    }
    const uint32_t smp_i = path_sample_index(bi, pix, k);
    uint32_t pixel_id = __ldg(bi.pix_id + pix);
    Sampler smp; sampler_start(smp, sc.sobol, __ldg(bi.pix_seed + pix), pixel_id, smp_i);
    uint32_t px = pixel_id % sc.cam.res_x, py = pixel_id/sc.cam.res_x;
    // PinholeCamera::sampleDirection (cameras/PinholeCamera.cpp:70-86)
    float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
    float fu, fv;
    if (sc.cam.filter == TGB_FILTER_DIRAC) { fu = 0.0f; fv = 0.0f; }
    else if (sc.cam.filter == TGB_FILTER_BOX) { fu = xa - 0.5f; fv = xb - 0.5f; }
    else { fu = filter_sample1(sc.cam, xa); fv = filter_sample1(sc.cam, xb); }
    V3 localD = normalize(v3(-1.0f + (float(px) + 0.5f + fu)*2.0f*sc.cam.pixel_size_x,
                             sc.cam.ratio - (float(py) + 0.5f + fv)*2.0f*sc.cam.pixel_size_x,
                             sc.cam.plane_dist));
    V3 d = m3mul(sc.cam.m, localD);
    Hit h = analytic_closest(sc, sc.cam.pos, d, 1e-4f, INFINITY);
    pb.T0[i] = make_float4(sc.cam.pos.x, sc.cam.pos.y, sc.cam.pos.z, 1e-4f);                  // nearT: math/Ray.hpp:24
    pb.T1[i] = make_float4(d.x, d.y, d.z, __uint_as_float(smp.dimension | F_WAS_SPECULAR | F_ALIVE));
    pb.T2[i] = pack_hit(h);
    pb.T3[i] = make_float4(1.0f, 1.0f, 1.0f, __uint_as_float((k << bi.pix_bits) | pix));
    pb.E[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    pb.pcg[i] = smp.pcg;
    order[i] = i;                    // new camera paths are already coherent: visited in slot order, after the sorted survivors
    }   // j
}

TGB_D void count_block(unsigned long long *rays, unsigned long long *hits, bool valid, bool hit) {
    unsigned mv = __ballot_sync(0xffffffffu, valid), mh = __ballot_sync(0xffffffffu, valid && hit);
    if ((threadIdx.x & 31) == 0 && mv) {
        atomicAdd(rays, (unsigned long long)__popc(mv));
        if (mh) atomicAdd(hits, (unsigned long long)__popc(mh));
    }
}
// The same for counts each thread has summed over the items it handled: reduced over the block in shared memory, one atomic
// per counter and block.  Every thread of the block calls it.
TGB_D void count_block_total(unsigned long long *rays, unsigned long long *hits, uint32_t n_rays, uint32_t n_hits) {
    __shared__ uint32_t sum[2];
    if (threadIdx.x == 0) { sum[0] = 0u; sum[1] = 0u; }
    __syncthreads();
    n_rays = __reduce_add_sync(0xffffffffu, n_rays); n_hits = __reduce_add_sync(0xffffffffu, n_hits);
    if ((threadIdx.x & 31) == 0 && n_rays) { atomicAdd(&sum[0], n_rays); if (n_hits) atomicAdd(&sum[1], n_hits); }
    __syncthreads();
    if (threadIdx.x == 0 && sum[0]) {
        atomicAdd(rays, (unsigned long long)sum[0]);
        if (sum[1]) atomicAdd(hits, (unsigned long long)sum[1]);
    }
}
// Queue allocation with one atomicAdd per block and queue: the lanes with take[q] set get consecutive entries of queue q, warp
// after warp in block order (as per-warp allocations made in that order would hand them out).  Every thread of the block calls
// it; at[q] is the lane's entry where take[q] is set.
template <int Q, int BLOCK>
TGB_D void block_alloc(uint32_t *const (&counter)[Q], const bool (&take)[Q], uint32_t (&at)[Q]) {
    constexpr int WARPS = BLOCK/32;
    static_assert(WARPS <= 32, "one warp scans the per-warp counts");
    __shared__ uint32_t cnt[Q][WARPS];
    const unsigned FULL = 0xffffffffu, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, lt = (1u << lane) - 1u;
    unsigned m[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) m[q] = __ballot_sync(FULL, take[q]);
    __syncthreads();                                            // a previous call's readers are done with cnt
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < Q; ++q) cnt[q][warp] = __popc(m[q]);
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int q = 0; q < Q; ++q) {
            const uint32_t c = lane < unsigned(WARPS) ? cnt[q][lane] : 0u;
            uint32_t incl = c;
#pragma unroll
            for (uint32_t off = 1; off < unsigned(WARPS); off <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, off); if (lane >= off) incl += v; }
            const uint32_t total = __shfl_sync(FULL, incl, WARPS - 1);
            uint32_t base = 0;
            if (lane == 0 && total) base = atomicAdd(counter[q], total);
            base = __shfl_sync(FULL, base, 0);
            if (lane < unsigned(WARPS)) cnt[q][lane] = base + incl - c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < Q; ++q) at[q] = cnt[q][warp] + __popc(m[q] & lt);
}

// TraceableScene::intersect for the path rays: the analytic part of the query was done by the kernel that made the
// ray (k_regen / k_accum); this kernel walks the BVH.  A ray is reached through the sort index: 48 bytes read (origin,
// direction, analytic hit: three 16-byte records) + 16 bytes written (closest hit).
struct PathRayPolicy {
    const float4 *T0, *T1; float4 *T2; const uint32_t *order; uint32_t n_sorted, n_surv, n_all; uint32_t s;
    TGB_D bool fetch(uint32_t i, V3 &o, V3 &d, float &tnear, Hit &h, bool &any) {
        // order[] = [survivors to trace, key order | unused (survivors that miss the BVH cut) | new camera paths]
        if (i >= n_sorted) { i += n_surv - n_sorted; if (i >= n_all) return false; }
        s = order[i];
        float4 a = T0[s], b = T1[s];
        o = v3(a.x, a.y, a.z); tnear = a.w; d = v3(b.x, b.y, b.z);
        h = unpack_hit(T2[s]); any = false;
        return true;
    }
    TGB_D void finish(const Hit &h) { T2[s] = pack_hit(h); }
    TGB_D int ignore() const { return -1; }
};
template <bool CURVES>
__global__ void __launch_bounds__(kTraceBlock, CURVES ? TGB_MINB_CURVES : TGB_MINB) k_trace(DScene sc, PathBuf pb, const uint32_t *order, Ctl *ctl) {
    __shared__ int smem_stack[kSmemStack*kTraceBlock];
    PathRayPolicy pol; pol.T0 = pb.T0; pol.T1 = pb.T1; pol.T2 = pb.T2; pol.order = order; pol.n_sorted = ctl->n_sorted; pol.n_surv = ctl->n_surv; pol.n_all = ctl->n; pol.s = 0;
    // rays to pull: the sorted survivors + the new camera paths
    const uint32_t n = ctl->n_sorted + ctl->n_new;
    bvh_traverse_persistent<CURVES>(sc, smem_stack, pol, n, &ctl->cursor_trace);
}

// Parity hook (tgb200_trace_closest): rays in AoS tgb_ray, hits out as tgb_hit, through the same analytic pass and
// the same persistent BVH traversal as the renderer.
// Rays the analytic pass settled through the BVH's top-level cut are not in `list` (k_hook_analytic).
struct HookPolicy {
    const tgb_ray *rays; Hit *out; const uint32_t *list, *count; uint32_t i;
    TGB_D bool fetch(uint32_t idx, V3 &o, V3 &d, float &tnear, Hit &h, bool &any) {
        if (idx >= *count) return false;
        i = list[idx];
        o = v3(rays[i].o[0], rays[i].o[1], rays[i].o[2]); d = v3(rays[i].d[0], rays[i].d[1], rays[i].d[2]); tnear = rays[i].tmin;
        h = out[i]; any = false;
        return true;
    }
    TGB_D void finish(const Hit &h) { out[i] = h; }
    TGB_D int ignore() const { return -1; }
};
// The analytic part of each query, then (cut = 1) the BVH's top-level cut as k_accum applies it: a ray that misses every cut box
// before its analytic hit is settled here; the others are listed for the BVH kernel.
__global__ void __launch_bounds__(256) k_hook_analytic(DScene sc, const tgb_ray *rays, Hit *out, uint32_t n, int cut, uint32_t *list,
                                                       uint32_t *count) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const V3 o = v3(rays[i].o[0], rays[i].o[1], rays[i].o[2]), d = v3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    const Hit h = analytic_closest(sc, o, d, rays[i].tmin, rays[i].tmax);
    out[i] = h;
    if (!cut || mesh_cut_hit(sc, o, d, rays[i].tmin, h.t)) list[atomicAdd(count, 1u)] = i;
}
template <bool CURVES>
__global__ void __launch_bounds__(kTraceBlock, CURVES ? TGB_MINB_CURVES : TGB_MINB) k_hook_persist(DScene sc, const tgb_ray *rays, Hit *out, const uint32_t *list,
                                                                                          const uint32_t *count, uint32_t n, uint32_t *counter) {
    __shared__ int smem_stack[kSmemStack*kTraceBlock];
    HookPolicy pol; pol.rays = rays; pol.out = out; pol.list = list; pol.count = count; pol.i = 0;
    bvh_traverse_persistent<CURVES>(sc, smem_stack, pol, n, counter);
}
__global__ void __launch_bounds__(256) k_hook_finish(DScene sc, const tgb_ray *rays, const Hit *in, tgb_hit *hits, uint32_t n) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    V3 o = v3(rays[i].o[0], rays[i].o[1], rays[i].o[2]), d = v3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    Hit h = in[i];
    tgb_hit out; out.primitive = -1; out.prim_id = 0; out.t = h.t; out.u = 0.0f; out.v = 0.0f; out.backside = 0;
    if (h.id != HID_MISS) {
        Surface s; make_surface<true>(sc, h, o, d, s);
        out.primitive = s.prim; out.backside = s.backside ? 1u : 0u;
        if (h.id >= 0) {
            uint32_t g = sc.tri_global[h.id]; out.prim_id = int(g - sc.prims[s.prim].tri_first); out.u = h.u; out.v = h.v;
            if (s.curve) out.prim_id /= kCurvePieces;                // BVH primitive -> segment
        }
        else if (sc.prims[s.prim].type == TGB_PRIM_QUAD) { out.u = h.u; out.v = h.v; }
    }
    hits[i] = out;
}

// handleSurface (integrators/TraceBase.cpp:516-568) + the loop tail of traceSample (PathTracer.cpp:108-126)
// k_shade is latency bound (scattered shading-record gathers): 8 resident blocks (64 registers) beat the
// compiler's free choice of 95 registers / 5 blocks (B200)
#ifndef TGB_SHADE_MINB
#define TGB_SHADE_MINB 8
#endif
// ES (emitter set): 1 = every light is a quad, there is no infinite emitter and every BSDF albedo and emission texture is
// constant; only with LS = 1.  Light selection, sampling and hits then compile the quad case alone: no mesh-light CDF search,
// no environment importance sampling, no cap or skydome, no infinite-light lookup on misses, no checker or bitmap lookup.
// The arithmetic and the draws are those of ES = 0.  TGB_QUAD_EMITTERS=0 builds a library that never takes it (A/B runs).
// Its launch bounds: TGB_SHADE_MINB_QUAD blocks of 128 per SM.  At 8 blocks (64 registers) it spills 144 B per thread and
// at 6 (80 registers) 36 B; at 5 (88 registers) nothing, and 5 measured fastest (H100, C1: 646.6 Msamples/s against 641.7
// at 6; 8 blocks measured 8 % slower than 6 before the emitter set had its BSDF records).
#ifndef TGB_QUAD_EMITTERS
#define TGB_QUAD_EMITTERS 1
#endif
#ifndef TGB_SHADE_MINB_QUAD
#define TGB_SHADE_MINB_QUAD 5
#endif
// MATSORT ("active-ray sort by material" of the path): scenes with several lobe models make the lanes of a warp run
// different BSDF code one after the other (C2: k_shade many times slower per path than on the Lambert-only C1).  The paths of a
// block are therefore dealt to its threads by BSDF type (block-local counting sort in shared memory: 512 consecutive
// slots, so every state array is still read in full sectors by the block as a whole); which thread shades which slot
// cannot change a result.  The key costs the hit -> primitive -> material gathers once more, so scenes with a single
// lobe model keep the unsorted kernel.
#ifndef TGB_SHADE_SORT_BLOCK
#define TGB_SHADE_SORT_BLOCK 1024
#endif
#ifndef TGB_SHADE_SORT_ITEMS
#define TGB_SHADE_SORT_ITEMS 2
#endif
constexpr int kShadeSortBlock = TGB_SHADE_SORT_BLOCK, kShadeSortItems = TGB_SHADE_SORT_ITEMS;
TGB_D uint32_t shade_sort_key(const DScene &sc, const Hit &h) {
    if (h.id == HID_MISS) return 0u;
    int bsdf;
    if (h.id >= 0) {
        if (uint32_t(h.id) >= sc.n_tris) {                       // curve segment: one material per primitive
            const DPrim &m = sc.prims[__ldg(sc.tri_prim + __ldg(sc.tri_global + h.id))];
            bsdf = int(__ldg(sc.slots + m.bsdf_first));
        } else {
            const uint32_t packed = __float_as_uint(__ldg(sc.tri_shade + 4*size_t(h.id) + 3).w);
            bsdf = int(__ldg(sc.slots + sc.prims[packed >> 10].bsdf_first + (packed & 1023u)));
        }
    } else bsdf = int(__ldg(sc.slots + sc.prims[-h.id - 2].bsdf_first));
    return 1u + min(sc.bsdfs[bsdf].type, 13u);
}

// attenuatedEmission + generalizedShadowRay (TraceBase.cpp:144-174,62-125) for the NEE and MIS queries.
//  * "any" queries (quad / environment lights): lightF / bsdfF were finished by k_shade; what remains is the
//    search for a blocker in [epsilon, t_light] other than the light; vis[] is set if there is none;
//  * mesh-light queries: one closest-hit query decides visibility (the light is part of the scene) and the epilogue
//    evaluates evalDirect / directPdf on the light hit: lightF (TraceBase.cpp:279-284) or bsdfF (:316-320).
// The tail of k_shade tests the analytic primitives, resolves what it can and compacts the rest for k_shadow_bvh
// (persistent traversal of the BVH).
template <bool CURVES>
TGB_D void shadow_resolve_closest(const DScene &sc, const Scratch &sr, uint32_t s, bool mis, int li, V3 p, V3 d, const Hit &h) {
    if (h.id == HID_MISS) return;
    const DPrim &l = sc.prims[li];
    Surface ls; make_surface<CURVES>(sc, h, p, d, ls);
    bool visible = ls.prim == li;
    if (visible && !mis && h.t*(1.0f + 1e-3f) < sr.N0[s].w) visible = false;                    // TraceBase.cpp:160
    if (!visible) return;
    V3 em = eval_direct(sc, ls);
    if (is_zero(em)) return;
    if (!mis) {
        float *n1 = reinterpret_cast<float *>(sr.N1 + s);
        V3 f = v3(n1[0], n1[1], n1[2]);
        float pdfL = n1[3], pdfB = reinterpret_cast<const float *>(sr.M1 + s)[3];
        V3 lightF = (f*em)/pdfL;
        lightF = lightF*power_heuristic(pdfL, pdfB);
        n1[0] = lightF.x; n1[1] = lightF.y; n1[2] = lightF.z;
    } else {
        float directPdf = mesh_direct_pdf(l, p, d, ls);
        float *m1 = reinterpret_cast<float *>(sr.M1 + s);                                      // (the NEE query of this path may be reading m1[3])
        V3 w = v3(m1[0], m1[1], m1[2]);
        V3 bsdfF = em*w;
        bsdfF = bsdfF*power_heuristic(sr.M0[s].w, directPdf);
        m1[0] = bsdfF.x; m1[1] = bsdfF.y; m1[2] = bsdfF.z;
    }
    sr.vis[2*size_t(s) + (mis ? 1 : 0)] = 1u;
}

template <bool CURVES, bool MATSORT, int LS = 0, int ES = 0>
__global__ void __launch_bounds__(MATSORT ? kShadeSortBlock : 128, MATSORT ? 1024/kShadeSortBlock : (LS == 1 ? (ES == 1 ? TGB_SHADE_MINB_QUAD : 6) : TGB_SHADE_MINB))
k_shade(DScene sc, PathBuf pb, Scratch sr, BatchInfo bi, Ctl *ctl, uint32_t *squeue, Counters *ctr) {
    const uint32_t n = ctl->n;
    // MATSORT: the block owns a window of kShadeSortItems x blockDim consecutive slots, counting-sorts them by BSDF type in shared
    // memory and shades them in sorted order, kShadeSortItems per thread (a wider window = purer warps: C2 with 512 / 1024 /
    // 2048 slots per window)
    constexpr int ITEMS = MATSORT ? kShadeSortItems : 1;
    __shared__ uint16_t perm[MATSORT ? kShadeSortBlock*kShadeSortItems : 1];
    const uint32_t window = blockIdx.x*blockDim.x*ITEMS;
    if (MATSORT) {
        __shared__ uint32_t bucket[16];
        if (threadIdx.x < 16) bucket[threadIdx.x] = 0u;
        __syncthreads();
        uint32_t key[ITEMS], rank[ITEMS];
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
            const uint32_t j = window + it*blockDim.x + threadIdx.x;
            const bool v = j < n;
            // one path query (TraceableScene::intersect) was completed for every slot in the queue
            const Hit hk = v ? unpack_hit(pb.T2[j]) : Hit{0.0f, 0.0f, 0.0f, HID_MISS};
            count_block(&ctr->rays, &ctr->hits, v, v && hk.id != HID_MISS);
            key[it] = v ? shade_sort_key(sc, hk) : 15u;                               // slots past the end sort last
            rank[it] = atomicAdd(&bucket[key[it]], 1u);
        }
        __syncthreads();
#pragma unroll
        for (int it = 0; it < ITEMS; ++it) {
            uint32_t before = 0;
            for (uint32_t k = 0; k < key[it]; ++k) before += bucket[k];
            perm[before + rank[it]] = uint16_t(it*blockDim.x + threadIdx.x);
        }
        __syncthreads();
    } else {
        const uint32_t j = window + threadIdx.x;
        count_block(&ctr->rays, &ctr->hits, j < n, j < n && __float_as_int(pb.T2[j < n ? j : 0].w) != HID_MISS);
    }
    for (int item = 0; item < ITEMS; ++item) {
    const uint32_t i = window + (MATSORT ? uint32_t(perm[item*blockDim.x + threadIdx.x]) : threadIdx.x);
    const bool valid = i < n;
    // this bounce's NEE / MIS queries: direction, far end (t of the light for occlusion queries), kind
    bool qn = false, qm = false, qn_any = false, qm_any = false;
    uint32_t s = 0;
    if (valid) {
        s = i;
        const float4 t0 = pb.T0[s], t1 = pb.T1[s], t2 = pb.T2[s], t3 = pb.T3[s];
        uint32_t info = __float_as_uint(t1.w);
        int bounce = int((info >> 16) & 0xFFu);
        bool wasSpecular = (info & F_WAS_SPECULAR) != 0;
        V3 o = v3(t0.x, t0.y, t0.z), d = v3(t1.x, t1.y, t1.z);
        V3 thr = v3(t3.x, t3.y, t3.z);
        Hit h = unpack_hit(t2);
        const tgb_settings &set = sc.set;
        uint32_t flags = 0;

        if (h.id == HID_MISS) {
            // loop exit with didHit == false: handleInfiniteLights (TraceBase.cpp:570-578, TraceableScene.hpp:194-209)
            if (ES == 0 && bounce >= set.min_bounces && bounce < set.max_bounces && sc.n_inf_lights > 0) {
                int li = infinite_light_hit(sc, d);
                if (li >= 0) {
                    const DPrim &l = sc.prims[li];
                    if (!set.enable_light_sampling || wasSpecular || !(l.flags & PF_SAMPLABLE)) {
                        float u = 0.0f, v = 0.0f;                                        // InfiniteSphereCap::evalDirect looks up uv (0, 0)
                        if (l.type != TGB_PRIM_INFINITE_SPHERE_CAP) direction_to_uv(l, d, u, v, nullptr);
                        V3 em = tex_eval(sc.tex[l.emission_tex], u, v);
                        float4 e4 = pb.E[s];
                        e4.x += thr.x*em.x; e4.y += thr.y*em.y; e4.z += thr.z*em.z;
                        pb.E[s] = e4;
                    }
                }
            }
            pb.T1[s] = make_float4(d.x, d.y, d.z, __uint_as_float((info & 0x00FFFFFFu) | F_FINAL_CHECK));
        } else {
            Sampler smp; smp.sobol = sc.sobol; smp.pcg = pb.pcg[s]; smp.dimension = info & 0xFFFFu;
            {
                uint32_t pix, k; path_decode(bi, __float_as_uint(t3.w), pix, k);
                smp.index = path_sample_index(bi, pix, k);
                smp.scramble = __ldg(bi.pix_seed + pix) ^ hash32(__ldg(bi.pix_id + pix));
            }
            Surface sf; make_surface<CURVES>(sc, h, o, d, sf);
            const DBsdf &b = sc.bsdfs[sf.bsdf];
            LambertRec lb; if (ES == 1) lb = lambert_rec(sc, sf.bsdf);
            const uint32_t lobes = ES == 1 ? lb.lobes : b.lobes;
            const float epsilon = sf.eps;                                                    // IntersectionInfo::epsilon
            int qli = 0;

            // makeLocalScatterEvent (TraceBase.cpp:24-51)
            Event e;
            {
                Frame frame = frame_from_normal(sf.Ns);
                if (CURVES && sf.curve && (b.lobes & LOBE_ANISO)) {
                    // anisotropic lobe: Curves::tangentSpace (Curves.cpp:518-530) + Primitive::setupTangentFrame (Primitive.cpp:134-162)
                    V3 B = normalize(sf.tangent);
                    V3 T_ = cross(B, sf.Ng), N = sf.Ns;
                    T_ = T_ - N*dot(N, T_);
                    if (!is_zero(T_)) { T_ = normalize(T_); frame.n = N; frame.t = T_; frame.b = cross(N, T_); }
                }
                bool hitBackside = dot(frame.n, d) > 0.0f;
                bool isTransmissive = (lobes & LOBE_TRANSMISSIVE) != 0;
                bool flipFrame = set.enable_two_sided_shading && hitBackside && !isTransmissive;
                if (flipFrame) { frame.n = -frame.n; frame.t = -frame.t; }
                e.frame = frame; e.wi = to_local(frame, -d); e.wo = v3s(0.0f); e.weight = v3s(1.0f); e.pdf = 1.0f;
                e.requested = LOBE_ALL; e.sampled = 0; e.flipped = flipFrame;
            }
            // forward-transparency coin flip: transparency == 0 for every lobe in scope, the draw is still made (:525-529)
            (void)sampler_boolean(smp, 0.0f);

            // TODO(open deviation, tests/test_gpu_bounce.py _NAN_THR): handleSurface adds estimateDirect(...)*throughput even when
            // the estimate is zero, which is NaN for a non-finite throughput; here a bounce without shadow queries adds nothing.
            if (set.enable_light_sampling && bounce < set.max_bounces - 1) {
                // estimateDirect -> chooseLight -> sampleDirect (TraceBase.cpp:483-494,416-459,383-400)
                float weight;
                int li = choose_light<ES>(sc, sf.p, smp, weight);
                bool pureSpecular = lobes != 0 && (lobes & ~uint32_t(LOBE_SPECULAR)) == 0;
                if (li >= 0 && !pureSpecular && lobes != LOBE_FORWARD) {
                    const DPrim &l = sc.prims[li];
                    // lightSample (TraceBase.cpp:246-285).  For quad / environment lights the light's own hit
                    // (attenuatedEmission, :160-165) and lightF (:279-284) are resolved here and the query that is
                    // traced is a pure blocker test; mesh lights keep the closest-hit query + epilogue.
                    float4 n1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), m1 = make_float4(0.0f, 0.0f, 0.0f, 0.0f); float mpb = 0.0f;
                    V3 qnd = v3s(0.0f), qmd = v3s(0.0f); float qnt = INFINITY, qmt = INFINITY;
                    LightSample ls;
                    if (light_sample_direct<ES>(sc, l, sf.p, smp, ls)) {
                        e.wo = to_local(e.frame, ls.d);
                        bool ok = true;
                        if (set.enable_consistency_checks)                                     // isConsistent (:53-60)
                            ok = (dot(ls.d, sf.Ng) < 0.0f) == ((e.wo.z < 0.0f) != e.flipped);
                        if (ok) {
                            e.requested = LOBE_ALL_BUT_SPECULAR;
                            V3 f = ES == 1 ? lambert_eval(lb, e) : bsdf_eval<CURVES, LS>(sc, b, sf, e);
                            if (!is_zero(f)) {
                                float pdfB = ES == 1 ? lambert_pdf(lb, e) : bsdf_pdf<CURVES, LS>(sc, b, sf, e);
                                qn = light_query<ES>(sc, l, sf.p, ls.d, epsilon, false, f, ls.pdf, pdfB, ls.dist, n1, qnt, qn_any);
                                m1.w = pdfB;
                                if (qn) qnd = ls.d;
                            }
                        }
                    }
                    // bsdfSample (TraceBase.cpp:287-321)
                    e.requested = LOBE_ALL_BUT_SPECULAR;
                    if ((ES == 1 ? lambert_sample(lb, smp, e) : bsdf_sample<CURVES, LS>(sc, b, sf, smp, e)) && !is_zero(e.weight)) {
                        V3 wo = to_global(e.frame, e.wo);
                        bool ok = true;
                        if (set.enable_consistency_checks)
                            ok = (dot(wo, sf.Ng) < 0.0f) == ((e.wo.z < 0.0f) != e.flipped);
                        if (ok) {
                            qm = light_query<ES>(sc, l, sf.p, wo, epsilon, true, e.weight, e.pdf, 0.0f, -1.0f, m1, mpb, qm_any);
                            if (qm) { qmd = wo; qmt = mpb; }
                        }
                    }
                    // generalizedShadowRay returns 0 unless bounce+1 >= minBounces (TraceBase.cpp:117)
                    if (bounce + 1 < set.min_bounces) { qn = false; qm = false; }
                    if (qn || qm) {
                        flags |= F_HAS_NEE; qli = li;
                        sr.P[s] = make_float4(sf.p.x, sf.p.y, sf.p.z, epsilon);
                        if (qn) { sr.N0[s] = make_float4(qnd.x, qnd.y, qnd.z, qnt); }
                        sr.N1[s] = n1;
                        if (qm) { sr.M0[s] = make_float4(qmd.x, qmd.y, qmd.z, qmt); }
                        sr.M1[s] = m1;
                        sr.D0[s] = make_float4(thr.x, thr.y, thr.z, weight);
                    }
                }
            }

            // emission of the surface itself (TraceBase.cpp:540-543)
            const DPrim &prim = sc.prims[sf.prim];
            float4 d1 = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(qli));
            if ((prim.flags & PF_EMISSIVE) && bounce >= set.min_bounces) {
                if (!set.enable_light_sampling || wasSpecular || !(prim.flags & PF_SAMPLABLE)) {
                    V3 em = eval_direct<ES>(sc, sf)*thr;
                    d1.x = em.x; d1.y = em.y; d1.z = em.z;
                    flags |= F_HAS_SURF;
                }
            }
            if (flags & (F_HAS_SURF | F_HAS_NEE)) sr.D1[s] = d1;

            // continuation sample (TraceBase.cpp:545-565)
            uint32_t status = 0;
            e.requested = LOBE_ALL;
            bool cont = ES == 1 ? lambert_sample(lb, smp, e) : bsdf_sample<CURVES, LS>(sc, b, sf, smp, e);
            V3 wo = v3s(0.0f);
            if (cont) {
                wo = to_global(e.frame, e.wo);
                if (set.enable_consistency_checks && (dot(wo, sf.Ng) < 0.0f) != ((e.wo.z < 0.0f) != e.flipped)) cont = false;
            }
            V3 no = o, nd = d; float ntmin = t0.w;
            if (cont) {
                thr = thr*e.weight;
                wasSpecular = (e.sampled & LOBE_SPECULAR) != 0;
                no = sf.p; nd = wo; ntmin = epsilon;                            // ray.hitpoint() == info.p for every primitive in scope
                // PathTracer.cpp:108-117
                if (max_comp(thr) == 0.0f) status = F_FINAL_CHECK;
                else {
                    float roulettePdf = max_comp(vabs(thr));
                    bool alive = true;
                    if (bounce > 2 && roulettePdf < 0.1f) {
                        if (sampler_boolean(smp, roulettePdf)) thr = thr/roulettePdf;
                        else alive = false;
                    }
                    if (alive) {
                        bounce++;
                        status = bounce < set.max_bounces ? F_ALIVE : (F_ALIVE | F_FINAL_CHECK);
                    }
                }
                pb.T0[s] = make_float4(no.x, no.y, no.z, ntmin);
                pb.T3[s] = make_float4(thr.x, thr.y, thr.z, t3.w);
            }
            pb.pcg[s] = smp.pcg;
            pb.T1[s] = make_float4(nd.x, nd.y, nd.z, __uint_as_float((smp.dimension & 0xFFFFu) | (uint32_t(bounce) << 16) | (wasSpecular ? F_WAS_SPECULAR : 0u) | status | flags));
        }
    }
    // enqueue this bounce's shadow queries: warp-vote compaction, one atomic per warp
    if (qn || qm) *reinterpret_cast<uint2 *>(sr.vis + 2*size_t(s)) = make_uint2(0u, 0u);
    {
        const unsigned FULL = 0xffffffffu;
        unsigned mn = __ballot_sync(FULL, qn), mm = __ballot_sync(FULL, qm);
        unsigned total = __popc(mn) + __popc(mm);
        if (total) {
            unsigned lane = threadIdx.x & 31, base = 0;
            if (lane == 0) base = atomicAdd(&ctl->shadow_count, total);
            base = __shfl_sync(FULL, base, 0);
            unsigned lt = (1u << lane) - 1u;
            if (qn) squeue[base + __popc(mn & lt)] = (s << 2) | (qn_any ? 2u : 0u);
            if (qm) squeue[base + __popc(mn) + __popc(mm & lt)] = (s << 2) | 1u | (qm_any ? 2u : 0u);
        }
    }
    }   // item
}

// Analytic part of the NEE/MIS queries (quads and cubes are tested coherently, every lane runs the same loop), top-level
// BVH cut, and compaction of what is left for k_shadow_bvh.  (Fusing this into k_shade's tail was measured (B200): the 13 values it
// needs stay live across the BSDF code, k_shade spills and gets slower than both kernels together.)
// The queries left for the BVH are compacted into two queues, so that every warp of k_shadow_bvh runs one kind: any-hit queries
// (quad / cap / environment lights) into squeue2 with the mask of the cut boxes they enter, closest-hit (mesh-light) queries into
// squeue_cl with their analytic hit.
// The grid is what is resident at once (or less): a block takes the runs of 256 queries [base, base + 256), base = its index
// times 256 plus multiples of the grid's width, so every thread of a block makes the same number of trips (block_alloc).
template <bool CURVES>
__global__ void __launch_bounds__(256) k_shadow_prep(DScene sc, Scratch sr, const uint32_t *squeue, Ctl *ctl, uint32_t *squeue2,
                                                     uint32_t *squeue_cl, Counters *ctr) {
    const uint32_t n = ctl->shadow_count;
    uint32_t n_valid = 0, n_blocked = 0;
    for (uint32_t base = blockIdx.x*blockDim.x; base < n; base += gridDim.x*blockDim.x) {
    const uint32_t i = base + threadIdx.x;
    const bool valid = i < n;
    bool keep = false, blocked = false, any = false; uint32_t q = 0, cut = 0; Hit h; h.t = INFINITY; h.u = h.v = 0.0f; h.id = HID_MISS;
    if (valid) {
        q = squeue[i];
        uint32_t s = q >> 2; bool mis = q & 1u; any = q & 2u;
        const float4 P = sr.P[s], D = mis ? sr.M0[s] : sr.N0[s];
        V3 p = v3(P.x, P.y, P.z), d = v3(D.x, D.y, D.z);
        const float eps = P.w;                                        // info.epsilon of the shading point (TraceBase.cpp:254,295)
        if (any) {
            const int li = __float_as_int(sr.D1[s].w);
            blocked = analytic_any(sc, p, d, eps, D.w, li);
            if (!blocked) { cut = mesh_cut_test<true>(sc, p, d, eps, D.w); if (!cut) sr.vis[2*size_t(s) + (mis ? 1 : 0)] = 1u; else keep = true; }
        } else {
            h = analytic_closest(sc, p, d, eps, INFINITY);
            if (!mesh_cut_hit(sc, p, d, eps, h.t)) blocked = h.id != HID_MISS;       // an analytic primitive is never the (mesh) light: not visible
            else keep = true;
        }
    }
    n_valid += valid ? 1u : 0u; n_blocked += blocked ? 1u : 0u;
    uint32_t *const queue[2] = {&ctl->shadow_count2, &ctl->shadow_count_closest};
    const bool take[2] = {keep && any, keep && !any};
    uint32_t at[2];
    block_alloc<2, 256>(queue, take, at);
    if (take[0]) { squeue2[at[0]] = q; sr.cut_mask[at[0]] = cut; }
    if (take[1]) { squeue_cl[at[1]] = q; sr.SH[at[1]] = pack_hit(h); }
    }   // base
    count_block_total(&ctr->shadow_rays, &ctr->shadow_hits, n_valid, n_blocked);
}

// ANY: the queue of any-hit queries (squeue2), else that of closest-hit queries (squeue_cl)
template <bool CURVES, bool ANY>
struct ShadowPolicy {
    DScene sc; Scratch sr; const uint32_t *squeue;
    uint32_t s, cut, blocked; bool mis; int li, ign; V3 p, d;      // blocked: the lane's queries that found a surface
    TGB_D bool fetch(uint32_t i, V3 &o, V3 &dd, float &tnear, Hit &h, bool &anyq) {
        uint32_t q = squeue[i];
        s = q >> 2; mis = q & 1u;
        const float4 P = sr.P[s], D = mis ? sr.M0[s] : sr.N0[s];
        p = v3(P.x, P.y, P.z); d = v3(D.x, D.y, D.z);
        o = p; dd = d; tnear = P.w; anyq = ANY; li = 0;
        if (ANY) {
            h.t = D.w; h.u = 0.0f; h.v = 0.0f; h.id = HID_MISS;
            // analytic primitives in the BVH: the query must not count the light it is aimed at (generalizedShadowRay's
            // `hit == endCap`, TraceBase.cpp:79-83); with the usual per-ray loop k_shadow_prep has dealt with them already
            ign = sc.n_analytic == 0 && sc.analytic_base != 0x7fffffff ? __float_as_int(sr.D1[s].w) : -1;
            cut = sr.cut_mask[i];
        } else { h = unpack_hit(sr.SH[i]); li = __float_as_int(sr.D1[s].w); ign = -1; }
        return true;
    }
    // any-hit walk: start in the subtrees of the cut boxes the segment enters, box 0 first (a segment that enters none never
    // gets here, and no primitive outside the cut boxes can block it)
    TGB_D void enter(TravStack &stk, int &sp) const {
        if (!sc.cut_entry) { stk.push(sp, 0); return; }
#pragma unroll
        for (int k = 15; k >= 0; --k) if (cut & (1u << k)) stk.push(sp, sc.cut_link[k]);
    }
    TGB_D int ignore() const { return ign; }
    TGB_D void finish(const Hit &h) {
        if (h.id != HID_MISS) blocked++;
        if (ANY) { if (h.id == HID_MISS) sr.vis[2*size_t(s) + (mis ? 1 : 0)] = 1u; }
        else shadow_resolve_closest<CURVES>(sc, sr, s, mis, li, p, d, h);
    }
};
// One launch for both queues: a warp walks any-hit queries until that queue is exhausted and its lanes are done, then (scenes with
// mesh lights) closest-hit ones, so the end of the first walk overlaps other warps' second and the launch has one drain tail.
// (Two launches, one per queue, measured 2.7 % slower on C2, H100: a second tail per iteration.)
template <bool CURVES, bool MESH_LIGHTS>
__global__ void __launch_bounds__(kTraceBlock, CURVES ? TGB_MINB_CURVES : TGB_MINB) k_shadow_bvh(DScene sc, Scratch sr, const uint32_t *squeue2,
                                                                                                const uint32_t *squeue_cl, Ctl *ctl, Counters *ctr) {
    __shared__ int smem_stack[kSmemStack*kTraceBlock];
    uint32_t blocked;
    {
        ShadowPolicy<CURVES, true> pol; pol.sc = sc; pol.sr = sr; pol.squeue = squeue2; pol.blocked = 0u;
        bvh_traverse_persistent<CURVES, true>(sc, smem_stack, pol, ctl->shadow_count2, &ctl->cursor_shadow);
        blocked = pol.blocked;
    }
    if (MESH_LIGHTS) {
        ShadowPolicy<CURVES, false> pol; pol.sc = sc; pol.sr = sr; pol.squeue = squeue_cl; pol.blocked = blocked;
        bvh_traverse_persistent<CURVES, false>(sc, smem_stack, pol, ctl->shadow_count_closest, &ctl->cursor_closest);
        blocked = pol.blocked;
    }
    // every lane of the warp is here (the walks end when the whole warp is idle): one atomic per warp
    blocked = __reduce_add_sync(0xffffffffu, blocked);
    if ((threadIdx.x & 31) == 0 && blocked) atomicAdd(&ctr->shadow_hits, (unsigned long long)blocked);
}

// A survivor's ray-coherence key into the histogram of the counting sort, one atomic per distinct key and warp (skewed keys would
// serialise per-lane atomics on the hot bins).  m: the lanes of the warp that call it, each with its own key; kBins is not counted.
TGB_D void bin_count(uint32_t *hist, unsigned m, uint32_t key) {
    const unsigned lane = threadIdx.x & 31u;
    const unsigned peers = __match_any_sync(m, key);
    if (key != kBins && lane == unsigned(__ffs(int(peers))) - 1u) atomicAdd(hist + key, unsigned(__popc(peers)));
}

// Fold this bounce's direct light + surface emission into the path (order as in handleSurface:537-543), apply the
// NaN guards of traceSample (PathTracer.cpp:119-122,130), store finished samples, and MOVE the survivors' persistent
// state to the front of the other state buffer (physical compaction: all later accesses are coalesced, no slot
// indirection).  The survivors' next ray gets the analytic part of its TraceableScene::intersect here.
__global__ void __launch_bounds__(256) k_accum(DScene sc, PathBuf pb, PathBuf dst, Scratch sr, BatchInfo bi, Ctl *ctl, uint32_t *keys, uint32_t *hist) {
    uint32_t s = blockIdx.x*blockDim.x + threadIdx.x;
    bool valid = s < ctl->n;
    bool alive = false; uint32_t info = 0; V3 em = v3s(0.0f);
    float4 t0 = make_float4(0.0f, 0.0f, 0.0f, 0.0f), t1 = t0, t3 = t0;
    if (valid) {
        t1 = pb.T1[s]; t3 = pb.T3[s];
        info = __float_as_uint(t1.w);
        const float4 e4 = pb.E[s];
        em = v3(e4.x, e4.y, e4.z);
        if (info & F_HAS_NEE) {
            const uint2 vis = *reinterpret_cast<const uint2 *>(sr.vis + 2*size_t(s));
            V3 L = v3s(0.0f), B = v3s(0.0f);
            if (vis.x) { const float4 n1 = sr.N1[s]; L = v3(n1.x, n1.y, n1.z); }
            if (vis.y) { const float4 m1 = sr.M1[s]; B = v3(m1.x, m1.y, m1.z); }
            const float4 d0 = sr.D0[s];
            V3 r = ((L + B)*d0.w)*v3(d0.x, d0.y, d0.z);
            em = em + r;
        }
        if (info & F_HAS_SURF) { const float4 d1 = sr.D1[s]; em = em + v3(d1.x, d1.y, d1.z); }
        alive = (info & F_ALIVE) != 0;
        bool finalCheck = (info & F_FINAL_CHECK) != 0;
        if (alive || finalCheck) {
            V3 thr = v3(t3.x, t3.y, t3.z);
            bool bad = false;
            if (alive) {
                t0 = pb.T0[s];
                bad = isnan(sum(v3(t1.x, t1.y, t1.z)) + sum(v3(t0.x, t0.y, t0.z)));
            }
            bad = bad || isnan(sum(thr) + sum(em));
            if (bad) { em = v3s(0.0f); alive = false; }
        }
        if (alive && finalCheck) alive = false;                  // bounce reached maxBounces: loop exits
        if (!alive) {                                                                           // the sample's radiance
            uint32_t pix, k; path_decode(bi, __float_as_uint(t3.w), pix, k);
            sr.R[path_result_slot(bi, pix, k)] = make_float4(em.x, em.y, em.z, 0.0f);
        }
    }
    uint32_t *const next[1] = {&ctl->next_count};
    const bool take[1] = {alive};
    uint32_t at[1];
    block_alloc<1, 256>(next, take, at);
    {
        const unsigned m = __ballot_sync(0xffffffffu, alive);
        if (alive) {
            const uint32_t t = at[0];
            V3 o = v3(t0.x, t0.y, t0.z), d = v3(t1.x, t1.y, t1.z); float tmin = t0.w;
            Hit h = analytic_closest(sc, o, d, tmin, INFINITY);
            dst.T0[t] = t0;
            dst.T1[t] = make_float4(t1.x, t1.y, t1.z, __uint_as_float((info & ~(F_HAS_NEE | F_HAS_SURF | F_ALIVE | F_FINAL_CHECK)) | F_ALIVE));
            dst.T2[t] = pack_hit(h);
            dst.T3[t] = t3;
            dst.E[t] = make_float4(em.x, em.y, em.z, 0.0f);
            dst.pcg[t] = pb.pcg[s];
            uint32_t key = mesh_cut_hit(sc, o, d, tmin, h.t) ? ray_bin(sc, o, d) : kBins;       // kBins: nothing to traverse
            keys[t] = key;
            bin_count(hist, m, key);
        }
    }
}

// End of an iteration (one block): exclusive scan of the ray-coherence histogram -> cursors of the counting sort, then the
// loop's bookkeeping for the NEXT iteration (what the host used to do after a stream sync).
__global__ void __launch_bounds__(1024) k_iter_end(uint32_t *hist, Ctl *ctl, int has_bvh) {
    // 32 Ki bins, 32 consecutive bins per thread (8 x 16-byte loads), block-wide scan of the 1024 partial sums with
    // warp shuffles (two levels), exclusive bases written back in place
    __shared__ uint32_t warp_sum[32];
    __shared__ uint32_t total_sorted;
    constexpr uint32_t per = kBins/1024u;
    static_assert(per % 4u == 0u, "vector loads");
    const uint32_t t = threadIdx.x, lane = t & 31u, warp = t >> 5;
    if (t == 0) total_sorted = 0u;
    if (has_bvh) {
        uint4 *h4 = reinterpret_cast<uint4 *>(hist) + size_t(t)*(per/4u);
        uint4 v[per/4u];
        uint32_t sum = 0;
#pragma unroll
        for (uint32_t i = 0; i < per/4u; ++i) { v[i] = h4[i]; sum += v[i].x + v[i].y + v[i].z + v[i].w; }
        uint32_t incl = sum;
#pragma unroll
        for (uint32_t off = 1; off < 32u; off <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, incl, off); if (lane >= off) incl += n; }
        if (lane == 31u) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = warp_sum[lane], wi = w;
#pragma unroll
            for (uint32_t off = 1; off < 32u; off <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, wi, off); if (lane >= off) wi += n; }
            warp_sum[lane] = wi - w;                       // exclusive base of each warp
            if (lane == 31u) total_sorted = wi;            // the culled survivors follow the sorted ones
        }
        __syncthreads();
        uint32_t base = warp_sum[warp] + incl - sum;
#pragma unroll
        for (uint32_t i = 0; i < per/4u; ++i) {
            uint4 o;
            o.x = base; base += v[i].x; o.y = base; base += v[i].y; o.z = base; base += v[i].z; o.w = base; base += v[i].w;
            h4[i] = o;
        }
    }
    __syncthreads();
    if (t == 0) {
        if (has_bvh) { ctl->traversed += (unsigned long long)ctl->n_sorted + ctl->n_new; ctl->shadow_traversed += ctl->shadow_count2 + ctl->shadow_count_closest; }
        ctl->iterations++;
        const uint32_t n_surv = ctl->next_count;
        const uint32_t n_new = min(ctl->capacity - n_surv, ctl->total - ctl->issued);
        ctl->first_path = ctl->issued; ctl->issued += n_new;
        ctl->n_surv = n_surv; ctl->n_new = n_new; ctl->n = n_surv + n_new; ctl->n_sorted = total_sorted;
        ctl->next_count = 0u; ctl->shadow_count = 0u; ctl->shadow_count2 = 0u; ctl->cursor_trace = 0u; ctl->cursor_shadow = 0u;
        ctl->shadow_count_closest = 0u; ctl->cursor_closest = 0u;
    }
}
// ... and scatter of the slot indices (4 bytes each) to their sorted positions.  The grid is what is resident at once (or less),
// a block takes runs of blockDim survivors as k_shadow_prep does, so every lane of a warp makes the same trips.  The lanes of a
// warp with the same key take consecutive positions with one atomic (the order inside a bin is free: a ray's result does not
// depend on when or by which lane it is traced).
__global__ void __launch_bounds__(256) k_bin_scatter(const uint32_t *keys, uint32_t *cursor, const Ctl *ctl, uint32_t *order) {
    const uint32_t n = ctl->n_surv, lane = threadIdx.x & 31u;
    for (uint32_t base = blockIdx.x*blockDim.x; base < n; base += gridDim.x*blockDim.x) {
        const uint32_t t = base + threadIdx.x;
        const uint32_t key = t < n ? keys[t] : kBins;
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        if (key == kBins) continue;                               // culled survivors are not visited: no entry needed
        const unsigned leader = unsigned(__ffs(int(peers))) - 1u;
        uint32_t at = 0;
        if (lane == leader) at = atomicAdd(cursor + key, unsigned(__popc(peers)));
        at = __shfl_sync(peers, at, int(leader));
        order[at + __popc(peers & ((1u << lane) - 1u))] = t;
    }
}

// OutputBuffer::addSample (cameras/OutputBuffer.hpp:104-132): running mean in sample order, NaN/Inf samples dropped
__global__ void __launch_bounds__(256) k_resolve(const float4 *R, BatchInfo bi, uint32_t spp_count, float *fb, uint32_t *fb_count) {
    uint32_t pix = blockIdx.x*blockDim.x + threadIdx.x;
    if (pix >= bi.n_pix) return;
    uint32_t pid = bi.pix_id[pix];
    float mx = fb[3*size_t(pid)], my = fb[3*size_t(pid) + 1], mz = fb[3*size_t(pid) + 2];
    uint32_t cnt = fb_count[pid];
    if (bi.pix_first) spp_count = bi.pix_first[pix + 1] - bi.pix_first[pix];
    for (uint32_t k = 0; k < spp_count; ++k) {
        const float4 c = R[path_result_slot(bi, pix, k)];
        float cx = c.x, cy = c.y, cz = c.z;
        if (isnan(cx) || isnan(cy) || isnan(cz) || isinf(cx) || isinf(cy) || isinf(cz)) continue;
        float n = float(cnt + 1u); cnt++;
        mx += (cx - mx)/n; my += (cy - my)/n; mz += (cz - mz)/n;
    }
    fb[3*size_t(pid)] = mx; fb[3*size_t(pid) + 1] = my; fb[3*size_t(pid) + 2] = mz;
    fb_count[pid] = cnt;
}

// SampleRecord::addSample for every sample of an adaptive step (integrators/path_tracer/SampleRecord.hpp:44-55): one thread per
// 4x4 variance block folds the luminance of its pixels' samples in the order renderTile produces them
// (PathTraceIntegrator.cpp:136-156: rows, then columns, then sample index; a block never straddles a 16x16 tile).  bi is one
// run of the call's pixel list, from list index pix_lo on (pix_slot holds indices into the whole list).
struct SampleRecordD { uint32_t sample_count, next_sample_count, sample_index; float adaptive_weight, mean, running_variance; };
__global__ void __launch_bounds__(128) k_block_stats(const float4 *R, BatchInfo bi, const uint32_t *pix_slot, uint32_t pix_lo, uint32_t res_x,
                                                     uint32_t res_y, uint32_t var_w, uint32_t n_blocks, SampleRecordD *rec) {
    uint32_t b = blockIdx.x*blockDim.x + threadIdx.x;
    if (b >= n_blocks) return;
    SampleRecordD r = rec[b];
    const uint32_t bx = (b % var_w)*4u, by = (b/var_w)*4u;
    for (uint32_t y = by; y < min(by + 4u, res_y); ++y)
        for (uint32_t x = bx; x < min(bx + 4u, res_x); ++x) {
            const uint32_t pix = pix_slot[x + y*res_x] - pix_lo;
            if (pix >= bi.n_pix) continue;                          // pixel not in this run (0xFFFFFFFF: not in the call's tile list)
            const uint32_t first = bi.pix_first[pix], cnt = bi.pix_first[pix + 1] - first;
            for (uint32_t k = 0; k < cnt; ++k) {
                const float4 c = R[size_t(first) + k];
                const float lum = c.x*0.2126f + c.y*0.7152f + c.z*0.0722f;              // Vec3f::luminance (math/Vec.hpp:195-199)
                r.sample_count++;
                const float delta = lum - r.mean;
                r.mean += delta/float(r.sample_count);
                r.running_variance += delta*(lum - r.mean);
            }
        }
    rec[b] = r;
}

// Tile-major pack / unpack of the resident framebuffer: the send/receive side of the one collective on
// this path (all-gather of the rendered tiles across GPUs).
__global__ void __launch_bounds__(256) k_pack_tiles(const uint32_t *pix_id, uint32_t n_pix, const float *fb, float *out) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    size_t p = size_t(pix_id[i])*3;
    out[3*size_t(i)] = fb[p]; out[3*size_t(i) + 1] = fb[p + 1]; out[3*size_t(i) + 2] = fb[p + 2];
}
__global__ void __launch_bounds__(256) k_unpack_tiles(const uint32_t *pix_id, uint32_t n_pix, const float *in, float *fb, uint32_t *fb_count, uint32_t count) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    size_t p = size_t(pix_id[i])*3;
    fb[p] = in[3*size_t(i)]; fb[p + 1] = in[3*size_t(i) + 1]; fb[p + 2] = in[3*size_t(i) + 2];
    fb_count[pix_id[i]] = count;
}

// In-library multi-GPU hand-off (tgb_settings::devices): a member packs the pixels of its tile share as (mean.rgb, sample count)
// records, the records travel to the root GPU with one peer-to-peer copy over NVLink, the root de-tiles them into its framebuffer.
__global__ void __launch_bounds__(256) k_pack_share(const uint32_t *pix_id, uint32_t n_pix, const float *fb, const uint32_t *fb_count, float4 *out) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    const uint32_t pid = pix_id[i];
    size_t p = size_t(pid)*3;
    out[i] = make_float4(fb[p], fb[p + 1], fb[p + 2], __uint_as_float(fb_count[pid]));
}
__global__ void __launch_bounds__(256) k_unpack_share(const uint32_t *pix_id, uint32_t n_pix, const float4 *in, float *fb, uint32_t *fb_count) {
    uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n_pix) return;
    const uint32_t pid = pix_id[i];
    const float4 v = in[i];
    size_t p = size_t(pid)*3;
    fb[p] = v.x; fb[p + 1] = v.y; fb[p + 2] = v.z;
    fb_count[pid] = __float_as_uint(v.w);
}

}  // namespace tgb
