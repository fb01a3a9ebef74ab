// Host-side BVH construction for the sm_90a traversal kernels.
//
// Replaces (reference): Embree's BVH4.Triangle4 object-split SAH builder used by TriangleMesh
// (src/thirdparty/embree/kernels/bvh/bvh_builder_sah.cpp:759, selected in kernels/common/scene.cpp:92-131)
// and the top-level user-geometry BVH of TraceableScene (src/core/renderer/TraceableScene.hpp:112-134).
// Not a port: one flattened world-space binned-SAH binary tree over every mesh triangle of the scene, collapsed
// into 4-ary 128-byte nodes for the GPU traversal kernels.
#pragma once
#include <cstdint>
#include <vector>

namespace tgb {

struct BuildTri { float v0[3], v1[3], v2[3]; };

// 128-byte 4-ary node (the binned-SAH binary tree is collapsed: the child with the largest surface area is replaced by
// its own two children until there are four): per axis the four children's lo / hi planes as one float4 each, then links.
//   f[0..3] = lo.x of children 0..3, f[4..7] = hi.x, f[8..11] = lo.y, f[12..15] = hi.y, f[16..19] = lo.z, f[20..23] = hi.z
//   link[k] >= 0 inner node index; link[k] < 0 leaf: ~link = (first << 3) | (count-1); link[k] == kEmptyLink: no child
// Half as many dependent node fetches per ray as the binary layout (the traversal kernels are latency bound), leaves hold
// <= 4 triangles.
constexpr int32_t kEmptyLink = int32_t(0x80000000u);
struct alignas(128) Node4 {
    float f[24];
    int32_t link[4];
    int32_t pad[4];
};

struct Bvh4 {
    std::vector<Node4> nodes;      // nodes[0] is the root; empty if there are no triangles
    std::vector<uint32_t> order;   // leaf order -> input triangle index
    float lo[3], hi[3];
    uint32_t max_depth = 0;        // depth of the 4-ary tree (stack need <= 3*depth)
    double sah_cost = 0.0;
};

// ---- compressed device layout ("QNode4", 64 bytes = 4 x 16-byte loads per visit instead of 7) -------------------
// The four child boxes are stored as 8-bit offsets from the node's own origin on a power-of-two grid:
//     plane = origin + q * 2^e   (per axis),   q_lo = floor, q_hi = ceil  ->  the stored box CONTAINS the float box,
// so a traversal over QNode4 visits a superset of what the float tree visits and finds the same closest hit.
//   chunk 0: origin.x, origin.y, origin.z, Sx         S = 32768 * 2^e (the kernel builds 1 + q*2^-15 with one PRMT and
//   chunk 1: Sy, Sz, lo.x[4], hi.x[4]                   evaluates t = fma(1 + q*2^-15, S/d, (origin - o)/d - S/d))
//   chunk 2: lo.y[4], hi.y[4], lo.z[4], hi.z[4]       one byte per child, child k in bits 8k..8k+7
//   chunk 3: link[4]                                  as in Node4
// Rounding of the kernel's evaluation is covered by (a) the builder's abs_pad, exactly as for the float nodes, and
// (b) 1/256 of a grid step subtracted/added before floor/ceil (the S/d cancellation costs at most 1/512 step).
struct alignas(64) QNode4 {
    float ox, oy, oz, sx;
    float sy, sz; uint32_t lox, hix;
    uint32_t loy, hiy, loz, hiz;
    int32_t link[4];
};
static_assert(sizeof(QNode4) == 64, "QNode4 layout");

struct QBvh4 {
    std::vector<QNode4> nodes;        // renumbered depth-first from the root
    std::vector<int32_t> old_index;   // new index -> index in the Node4 array it was made from
};
// Quantise `in` (float 4-ary BVH) into `out`.
// Empty child slots get the inverted box (lo 255, hi 0), which no ray can enter, and `empty_link` instead of kEmptyLink: the
// kernels do not test for empty slots, so the link must be harmless to follow (the caller passes a one-primitive leaf that
// holds an all-zero record, which every primitive test rejects).
void quantize_bvh4(const Bvh4 &in, QBvh4 &out, int32_t empty_link = kEmptyLink);
// Host evaluation of one node visit with the kernels' arithmetic (tests + tgb200_qbvh_selftest): entry distance of the
// four children for the ray (o, 1/d), INFINITY where the slab test fails.
void qnode_slab_host(const QNode4 &nd, const float o[3], const float inv_d[3], float tnear, float tfar, float t_out[4]);

// Top-level cut of a 4-ary tree: start from the root's children and keep replacing the inner child with the largest surface area
// by its children while there are at most max_cut (<= 16) boxes.  Together the boxes cover every primitive; `link` is the
// Node4 index (or leaf code) below each.
struct CutBox { float lo[3], hi[3]; int32_t link; };
std::vector<CutBox> top_level_cut(const Bvh4 &bvh, size_t max_cut);
// Traversal stack entries a walk may need: a walk from the root pushes at most 3 per inner node on its path (3*max_depth + 2,
// kept from before the cut), an any-hit walk starts with the entered cut boxes less the one it enters (< cut.size()) and pushes
// at most 3 per inner node below a cut box.
uint32_t traversal_stack_need(const Bvh4 &bvh, const std::vector<CutBox> &cut);

// A primitive given by its bounds and the point the SAH binning sorts it by (curve segments).
struct BuildBox { float lo[3], hi[3], centroid[3]; };

// threads <= 0: hardware concurrency.
// abs_pad: every triangle box is grown by this absolute amount (covers the slab test's rounding).
void build_bvh4(const BuildTri *tris, uint32_t n, Bvh4 &out, int threads = 0, float abs_pad = 0.0f,
                uint32_t max_leaf = 4, float isect_cost = 1.0f);
// max_leaf (1..4) and isect_cost (SAH cost of one primitive test relative to one node visit) let expensive primitives get
// smaller leaves.
void build_bvh4_boxes(const BuildBox *boxes, uint32_t n, Bvh4 &out, int threads = 0, float abs_pad = 0.0f,
                      uint32_t max_leaf = 4, float isect_cost = 1.0f);

// ---- the scene's tree, as tgb200_create builds and uploads it ------------------------------------------------------
// Build switches (environment overrides: bvh_options in tgb200_api.cu).
struct BvhOptions {
    // SAH leaf cap and intersection cost of the triangle tree: chosen on C1 on the previous GPU (B200).  On an H100 (C1, 400 W
    // limit) cost 1 or leaf cap 2 measured ~1 % faster and cost 2 ~2 % slower; the default is kept, as a different tree changes
    // which of two equally distant hits wins.
    uint32_t tri_leaf = 4; float tri_cost = 0.5f;
    // a segment test (3 projections + up to 32 half-cylinder pieces) costs far more than a triangle test: small leaves (the
    // reference's BinaryBvh also keeps <= 2 segments per leaf, Curves.cpp:613)
    uint32_t curve_leaf = 2; float curve_cost = 4.0f;
    size_t max_cut = 16;            // boxes of the top-level cut: fewer = cheaper pre-test in k_accum / k_shadow_prep, looser cut
};

struct Aabb { float lo[3], hi[3]; };

// One 48-byte intersection record per leaf position, as the kernels read it (3 x float4).  Triangle (Embree TriangleM,
// kernels/geometry/triangle.h:54): v0, e1 = v0 - v1, e2 = v2 - v0, Ng = cross(e1, e2).  Curve piece: its segment's three nodes
// (x, y, z, width).
struct alignas(16) IsectRecord { float f[12]; };

struct SceneBvhInput {
    const BuildTri *tris = nullptr; uint32_t n_tris = 0;
    // curve pieces: bounds and intersection record of each
    const BuildBox *curve_boxes = nullptr; const IsectRecord *curve_recs = nullptr; uint32_t n_curve = 0;
    // analytic primitives that become leaves (quads / cubes): unpadded world bounds; n_analytic = 0 keeps them out of the tree
    const Aabb *analytic = nullptr; uint32_t n_analytic = 0;
    // largest coordinate magnitude in play besides the primitives' (the camera position): seeds the padding extent
    float extent = 0.0f;
};

// Leaf positions: [0, n_tris) triangles, [n_tris, n_tris + n_curve) curve pieces, one all-zero record (the target of empty
// child slots; every primitive test rejects it), then the analytic primitives from isect.size() on.  Leaves of the last two
// kinds carry bit 2 of the leaf code.
struct SceneBvh {
    Bvh4 tree;                           // every tree under one root; tree.order: leaf position -> triangle, then n_tris + curve piece
    QBvh4 qtree;                         // its device layout
    std::vector<uint32_t> analytic_order;   // analytic leaf position - isect.size() -> analytic input index
    std::vector<IsectRecord> isect;      // tris + curve pieces + 1, in leaf order
    std::vector<CutBox> cut;             // top-level cut, link = QNode4 index (or leaf code) below each box
    uint32_t stack_need = 0;             // traversal_stack_need of the tree and its cut
};
// One tree for the triangles, one for the curve pieces and one for the analytic primitives (those that exist), under a joint
// root when there are several, then the cut, the device layout and the records.
void build_scene_bvh(const SceneBvhInput &in, const BvhOptions &opt, SceneBvh &out);

}  // namespace tgb
