// Binned-SAH builder (host, multi-threaded) + collapse to the 4-ary device layout.  See bvh_build.h for what it replaces.
#include "bvh_build.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <limits>
#include <thread>

namespace tgb {
namespace {

struct Box {
    float lo[3], hi[3];
    void reset() { for (int a = 0; a < 3; ++a) { lo[a] = std::numeric_limits<float>::infinity(); hi[a] = -lo[a]; } }
    void grow(const Box &b) { for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], b.lo[a]); hi[a] = std::max(hi[a], b.hi[a]); } }
    void grow(const float *p) { for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], p[a]); hi[a] = std::max(hi[a], p[a]); } }
    float half_area() const {
        float dx = hi[0] - lo[0], dy = hi[1] - lo[1], dz = hi[2] - lo[2];
        if (!(dx >= 0.0f)) return 0.0f;
        return dx*dy + dy*dz + dz*dx;
    }
};

struct Tmp { Box box; int32_t left, right; uint32_t first, count; };

constexpr int kBins = 16;
constexpr float kTraversalCost = 1.0f;

struct Builder {
    const Box *tb; const float *cent; uint32_t *idx; std::vector<Tmp> nodes; std::atomic<uint32_t> n_nodes{0};
    std::atomic<int> free_threads{0};
    uint32_t kMaxLeaf = 4; float kIntersectCost = 1.0f;      // leaf size cap (<= 4: two bits in the leaf link) and SAH cost of one primitive test

    uint32_t alloc() { return n_nodes.fetch_add(1); }

    void build(uint32_t node, uint32_t first, uint32_t count, int depth) {
        Tmp &nd = nodes[node];
        Box box, cb; box.reset(); cb.reset();
        for (uint32_t i = 0; i < count; ++i) { uint32_t t = idx[first + i]; box.grow(tb[t]); cb.grow(cent + 3*t); }
        nd.box = box; nd.first = first; nd.count = count; nd.left = nd.right = -1;
        if (count <= 1) return;

        int best_axis = -1, best_split = -1; float best_cost = std::numeric_limits<float>::infinity();
        for (int a = 0; a < 3; ++a) {
            float ext = cb.hi[a] - cb.lo[a];
            if (!(ext > 0.0f)) continue;
            Box bb[kBins]; uint32_t bc[kBins];
            for (int b = 0; b < kBins; ++b) { bb[b].reset(); bc[b] = 0; }
            float scale = kBins/ext;
            for (uint32_t i = 0; i < count; ++i) {
                uint32_t t = idx[first + i];
                int b = std::min(kBins - 1, std::max(0, int((cent[3*t + a] - cb.lo[a])*scale)));
                bb[b].grow(tb[t]); bc[b]++;
            }
            float right_area[kBins]; Box acc; acc.reset();
            for (int b = kBins - 1; b > 0; --b) { acc.grow(bb[b]); right_area[b] = acc.half_area(); }
            acc.reset(); uint32_t nl = 0;
            for (int b = 0; b < kBins - 1; ++b) {
                acc.grow(bb[b]); nl += bc[b];
                if (nl == 0 || nl == count) continue;
                float cost = acc.half_area()*nl + right_area[b + 1]*(count - nl);
                if (cost < best_cost) { best_cost = cost; best_axis = a; best_split = b; }
            }
        }
        float leaf_cost = kIntersectCost*count;
        float split_cost = best_axis >= 0 ? kTraversalCost + kIntersectCost*best_cost/std::max(box.half_area(), 1e-30f)
                                          : std::numeric_limits<float>::infinity();
        if (count <= kMaxLeaf && !(split_cost < leaf_cost)) return;

        uint32_t mid;
        if (best_axis >= 0) {
            float ext = cb.hi[best_axis] - cb.lo[best_axis], scale = kBins/ext, lo = cb.lo[best_axis];
            const float *c = cent; int ax = best_axis, sp = best_split;
            uint32_t *m = std::partition(idx + first, idx + first + count, [=](uint32_t t) {
                int b = std::min(kBins - 1, std::max(0, int((c[3*t + ax] - lo)*scale)));
                return b <= sp;
            });
            mid = uint32_t(m - (idx + first));
        } else {
            mid = count/2;   // all centroids coincide: split by index
        }
        if (mid == 0 || mid == count) mid = count/2;
        uint32_t l = alloc(), r = alloc();
        nodes[node].left = int32_t(l); nodes[node].right = int32_t(r);
        bool spawned = false; std::thread th;
        if (count > 32768) {
            int avail = free_threads.load();
            while (avail > 0 && !free_threads.compare_exchange_weak(avail, avail - 1)) {}
            if (avail > 0) { spawned = true; th = std::thread([=] { build(l, first, mid, depth + 1); free_threads.fetch_add(1); }); }
        }
        if (!spawned) build(l, first, mid, depth + 1);
        build(r, first + mid, count - mid, depth + 1);
        if (spawned) th.join();
    }
};

inline float pad_down(float v) { return std::nextafter(std::nextafter(v, -std::numeric_limits<float>::infinity()), -std::numeric_limits<float>::infinity()); }
inline float pad_up(float v) { return std::nextafter(std::nextafter(v, std::numeric_limits<float>::infinity()), std::numeric_limits<float>::infinity()); }

Node4 empty_node() {
    Node4 nd; std::memset(&nd, 0, sizeof(nd));
    for (int k = 0; k < 4; ++k) nd.link[k] = kEmptyLink;
    return nd;
}

}  // namespace

static void build_from_boxes(std::vector<Box> &tb, std::vector<float> &cent, uint32_t n, Bvh4 &out, int threads, uint32_t max_leaf = 4, float isect_cost = 1.0f);

void build_bvh4(const BuildTri *tris, uint32_t n, Bvh4 &out, int threads, float abs_pad, uint32_t max_leaf, float isect_cost) {
    out.nodes.clear(); out.order.clear(); out.max_depth = 0; out.sah_cost = 0.0;
    for (int a = 0; a < 3; ++a) { out.lo[a] = std::numeric_limits<float>::infinity(); out.hi[a] = -out.lo[a]; }
    if (n == 0) return;
    std::vector<Box> tb(n); std::vector<float> cent(3*size_t(n));
    for (uint32_t i = 0; i < n; ++i) {
        Box b; b.reset(); b.grow(tris[i].v0); b.grow(tris[i].v1); b.grow(tris[i].v2);
        for (int a = 0; a < 3; ++a) { cent[3*size_t(i) + a] = 0.5f*b.lo[a] + 0.5f*b.hi[a]; b.lo[a] = pad_down(b.lo[a] - abs_pad); b.hi[a] = pad_up(b.hi[a] + abs_pad); }
        tb[i] = b;
    }
    build_from_boxes(tb, cent, n, out, threads, std::min<uint32_t>(std::max<uint32_t>(max_leaf, 1), 4), isect_cost);
}

void build_bvh4_boxes(const BuildBox *boxes, uint32_t n, Bvh4 &out, int threads, float abs_pad, uint32_t max_leaf, float isect_cost) {
    out.nodes.clear(); out.order.clear(); out.max_depth = 0; out.sah_cost = 0.0;
    for (int a = 0; a < 3; ++a) { out.lo[a] = std::numeric_limits<float>::infinity(); out.hi[a] = -out.lo[a]; }
    if (n == 0) return;
    std::vector<Box> tb(n); std::vector<float> cent(3*size_t(n));
    for (uint32_t i = 0; i < n; ++i)
        for (int a = 0; a < 3; ++a) {
            cent[3*size_t(i) + a] = boxes[i].centroid[a];
            tb[i].lo[a] = pad_down(boxes[i].lo[a] - abs_pad); tb[i].hi[a] = pad_up(boxes[i].hi[a] + abs_pad);
        }
    build_from_boxes(tb, cent, n, out, threads, std::min<uint32_t>(std::max<uint32_t>(max_leaf, 1), 4), isect_cost);
}

static void build_from_boxes(std::vector<Box> &tb, std::vector<float> &cent, uint32_t n, Bvh4 &out, int threads, uint32_t max_leaf, float isect_cost) {
    out.order.resize(n);
    for (uint32_t i = 0; i < n; ++i) out.order[i] = i;
    Builder bl; bl.tb = tb.data(); bl.cent = cent.data(); bl.idx = out.order.data(); bl.kMaxLeaf = max_leaf; bl.kIntersectCost = isect_cost;
    const float kIntersectCost = isect_cost;
    bl.nodes.resize(2*size_t(n) + 1);
    if (threads <= 0) threads = int(std::thread::hardware_concurrency());
    bl.free_threads = std::max(0, threads - 1);
    uint32_t root = bl.alloc();
    bl.build(root, 0, n, 0);
    for (int a = 0; a < 3; ++a) { out.lo[a] = bl.nodes[root].box.lo[a]; out.hi[a] = bl.nodes[root].box.hi[a]; }

    auto leaf_link = [](const Tmp &t) { return ~int32_t((t.first << 3) | (t.count - 1)); };
    const Tmp &rt = bl.nodes[root];
    double root_area = std::max(double(rt.box.half_area()), 1e-30);
    auto set_child = [](Node4 &nd, int k, const Box &b, int32_t link) {
        nd.f[k] = b.lo[0]; nd.f[4 + k] = b.hi[0]; nd.f[8 + k] = b.lo[1]; nd.f[12 + k] = b.hi[1]; nd.f[16 + k] = b.lo[2]; nd.f[20 + k] = b.hi[2];
        nd.link[k] = link;
    };
    if (rt.left < 0) {                       // the whole scene fits one leaf
        Node4 nd = empty_node();
        set_child(nd, 0, rt.box, leaf_link(rt));
        out.nodes.push_back(nd);
        out.max_depth = 1;
        return;
    }
    struct Item { uint32_t tmp; int32_t out_index; uint32_t depth; };
    std::vector<Item> stack; stack.push_back({root, 0, 1});
    out.nodes.resize(1);
    while (!stack.empty()) {
        Item it = stack.back(); stack.pop_back();
        const Tmp &t = bl.nodes[it.tmp];
        // collapse: start with the two children, split the largest inner child until four
        uint32_t ch[4]; int nc = 0;
        ch[nc++] = uint32_t(t.left); ch[nc++] = uint32_t(t.right);
        while (nc < 4) {
            int best = -1; float best_area = -1.0f;
            for (int k = 0; k < nc; ++k) {
                const Tmp &c = bl.nodes[ch[k]];
                if (c.left >= 0 && c.box.half_area() > best_area) { best_area = c.box.half_area(); best = k; }
            }
            if (best < 0) break;
            const Tmp &c = bl.nodes[ch[best]];
            ch[best] = uint32_t(c.left); ch[nc++] = uint32_t(c.right);
        }
        Node4 nd = empty_node();
        out.sah_cost += kTraversalCost*t.box.half_area()/root_area;
        out.max_depth = std::max(out.max_depth, it.depth + 1);
        for (int k = 0; k < nc; ++k) {
            const Tmp &c = bl.nodes[ch[k]];
            if (c.left < 0) {
                set_child(nd, k, c.box, leaf_link(c));
                out.sah_cost += kIntersectCost*c.count*c.box.half_area()/root_area;
            } else {
                int32_t idx = int32_t(out.nodes.size());
                set_child(nd, k, c.box, idx);
                out.nodes.emplace_back();
                stack.push_back({ch[k], idx, it.depth + 1});
            }
        }
        out.nodes[size_t(it.out_index)] = nd;
    }
}

std::vector<CutBox> top_level_cut(const Bvh4 &bvh, size_t max_cut) {
    std::vector<CutBox> cut;
    if (bvh.nodes.empty()) return cut;
    auto child = [&](const Node4 &nd, int k) { CutBox b; for (int a = 0; a < 3; ++a) { b.lo[a] = nd.f[8*a + k]; b.hi[a] = nd.f[8*a + 4 + k]; } b.link = nd.link[k]; return b; };
    auto area = [](const CutBox &b) { float e[3] = {b.hi[0] - b.lo[0], b.hi[1] - b.lo[1], b.hi[2] - b.lo[2]}; return e[0]*e[1] + e[1]*e[2] + e[2]*e[0]; };
    for (int k = 0; k < 4; ++k) if (bvh.nodes[0].link[k] != kEmptyLink) cut.push_back(child(bvh.nodes[0], k));
    while (true) {
        int best = -1;
        for (size_t i = 0; i < cut.size(); ++i) if (cut[i].link >= 0 && (best < 0 || area(cut[i]) > area(cut[size_t(best)]))) best = int(i);
        if (best < 0) break;
        const Node4 &nd = bvh.nodes[size_t(cut[size_t(best)].link)];
        int kids = 0; for (int k = 0; k < 4; ++k) kids += nd.link[k] != kEmptyLink;
        if (cut.size() - 1 + size_t(kids) > max_cut) break;
        cut.erase(cut.begin() + best);
        for (int k = 0; k < 4; ++k) if (nd.link[k] != kEmptyLink) cut.push_back(child(nd, k));
    }
    return cut;
}

uint32_t traversal_stack_need(const Bvh4 &bvh, const std::vector<CutBox> &cut) {
    // inner nodes on the longest path down from each node (0 for a leaf)
    std::vector<uint32_t> levels(bvh.nodes.size(), 0);
    for (size_t i = bvh.nodes.size(); i-- > 0;) {          // children follow their parent in Node4 order (build_from_boxes)
        uint32_t l = 0;
        for (int k = 0; k < 4; ++k) if (bvh.nodes[i].link[k] >= 0) l = std::max(l, levels[size_t(bvh.nodes[i].link[k])]);
        levels[i] = l + 1;
    }
    uint32_t below = 0;
    for (const CutBox &b : cut) if (b.link >= 0) below = std::max(below, levels[size_t(b.link)]);
    const uint32_t from_cut = cut.empty() ? 0u : uint32_t(cut.size()) - 1u + 3u*below;
    return std::max(3u*bvh.max_depth + 2u, from_cut);
}

// ---- quantised layout -------------------------------------------------------------------------------------------
void quantize_bvh4(const Bvh4 &in, QBvh4 &out, int32_t empty_link) {
    out.nodes.clear(); out.old_index.clear();
    const size_t n = in.nodes.size();
    if (n == 0) return;
    // order: depth-first from the root, children 0..3 in order (pushed 3..0)
    std::vector<int32_t> order; order.reserve(n);
    std::vector<int32_t> stack(1, 0);
    while (!stack.empty()) {
        const int32_t x = stack.back(); stack.pop_back();
        order.push_back(x);
        const Node4 &nd = in.nodes[size_t(x)];
        for (int k = 3; k >= 0; --k) if (nd.link[k] >= 0) stack.push_back(nd.link[k]);
    }
    std::vector<int32_t> new_index(n, -1);
    for (size_t i = 0; i < order.size(); ++i) new_index[size_t(order[i])] = int32_t(i);
    out.old_index = order;
    out.nodes.resize(order.size());
    for (size_t i = 0; i < order.size(); ++i) {
        const Node4 &nd = in.nodes[size_t(order[i])];
        QNode4 q; std::memset(&q, 0, sizeof(q));
        float org[3], S[3]; uint32_t lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
        for (int a = 0; a < 3; ++a) {
            double mn = std::numeric_limits<double>::infinity(), mx = -mn;
            for (int k = 0; k < 4; ++k) if (nd.link[k] != kEmptyLink) { mn = std::min(mn, double(nd.f[8*a + k])); mx = std::max(mx, double(nd.f[8*a + 4 + k])); }
            if (!(mx >= mn)) { mn = 0.0; mx = 0.0; }
            // grid: plane(q) = org + q*2^e.  org sits at least 1/128 step below the lowest child plane so that q = 0 keeps the
            // same 1/256-step guard as every other value; e = the smallest exponent for which the highest plane still maps to <= 255.
            const double ext = mx - mn;
            int e = ext > 0.0 ? std::max(-120, int(std::floor(std::log2(ext/255.0))) - 1) : -120;
            for (;; ++e) {
                const double st = std::ldexp(1.0, e);
                float og = float(mn - st/64.0);
                while (double(og) > mn - st/128.0) og = std::nextafter(og, -std::numeric_limits<float>::infinity());
                if (std::ceil((mx - double(og))/st + 1.0/256.0) <= 255.0) { org[a] = og; break; }
            }
            const double step = std::ldexp(1.0, e);
            S[a] = float(std::ldexp(1.0, e + 15));
            for (int k = 0; k < 4; ++k) {
                uint32_t ql = 255, qh = 0;                      // empty child: inverted box
                if (nd.link[k] != kEmptyLink) {
                    double l = (double(nd.f[8*a + k]) - double(org[a]))/step - 1.0/256.0;
                    double h = (double(nd.f[8*a + 4 + k]) - double(org[a]))/step + 1.0/256.0;
                    ql = uint32_t(std::min(255.0, std::max(0.0, std::floor(l))));
                    qh = uint32_t(std::min(255.0, std::max(0.0, std::ceil(h))));
                }
                lo[a] |= ql << (8*k); hi[a] |= qh << (8*k);
            }
        }
        q.ox = org[0]; q.oy = org[1]; q.oz = org[2]; q.sx = S[0]; q.sy = S[1]; q.sz = S[2];
        q.lox = lo[0]; q.hix = hi[0]; q.loy = lo[1]; q.hiy = hi[1]; q.loz = lo[2]; q.hiz = hi[2];
        for (int k = 0; k < 4; ++k) q.link[k] = nd.link[k] >= 0 ? new_index[size_t(nd.link[k])] : (nd.link[k] == kEmptyLink ? empty_link : nd.link[k]);
        out.nodes[i] = q;
    }
}

void qnode_slab_host(const QNode4 &nd, const float o[3], const float inv_d[3], float tnear, float tfar, float t_out[4]) {
    // mirrors Traversal::visit in tgb_wavefront.cuh operation for operation (fmaf = one rounding, as FFMA)
    const float org[3] = {nd.ox, nd.oy, nd.oz}, S[3] = {nd.sx, nd.sy, nd.sz};
    const uint32_t lo[3] = {nd.lox, nd.loy, nd.loz}, hi[3] = {nd.hix, nd.hiy, nd.hiz};
    float a[3], b[3]; uint32_t nearw[3], farw[3];
    for (int ax = 0; ax < 3; ++ax) {
        const float ood = o[ax]*inv_d[ax];
        a[ax] = S[ax]*inv_d[ax];
        b[ax] = std::fmaf(org[ax], inv_d[ax], -ood) - a[ax];
        const bool neg = inv_d[ax] < 0.0f;
        nearw[ax] = neg ? hi[ax] : lo[ax]; farw[ax] = neg ? lo[ax] : hi[ax];
    }
    auto F = [](uint32_t w, int k) { uint32_t bits = 0x3F800000u | (((w >> (8*k)) & 0xFFu) << 8); float f; std::memcpy(&f, &bits, 4); return f; };
    for (int k = 0; k < 4; ++k) {
        float tn = tnear, tf = tfar;
        for (int ax = 0; ax < 3; ++ax) {
            tn = std::fmax(tn, std::fmaf(F(nearw[ax], k), a[ax], b[ax]));
            tf = std::fmin(tf, std::fmaf(F(farw[ax], k), a[ax], b[ax]));
        }
        t_out[k] = (tn <= tf && nd.link[k] != kEmptyLink) ? tn : std::numeric_limits<float>::infinity();
    }
}

// ---- the scene's tree -------------------------------------------------------------------------------------------
void build_scene_bvh(const SceneBvhInput &in, const BvhOptions &opt, SceneBvh &out) {
    const uint32_t n_tris = in.n_tris, n_curve = in.n_curve, analytic_base = n_tris + n_curve + 1;
    // Box padding that covers the rounding of the fused slab test t = fma(lo, 1/d, -(o/d)): spatial error
    // <= (2|o| + |lo|) * 2^-24, so 1e-6 x the largest coordinate magnitude in play (scene or camera) is ample.
    float extent = in.extent;
    for (uint32_t i = 0; i < n_tris; ++i) {
        const BuildTri &t = in.tris[i];
        for (int k = 0; k < 3; ++k) extent = std::max(extent, std::max(std::fabs(t.v0[k]), std::max(std::fabs(t.v1[k]), std::fabs(t.v2[k]))));
    }
    for (uint32_t i = 0; i < n_curve; ++i)
        for (const float *q = in.curve_recs[i].f; q < in.curve_recs[i].f + 12; q += 4)
            extent = std::max(extent, std::max(std::fabs(q[0]), std::max(std::fabs(q[1]), std::fabs(q[2]))) + q[3]);
    Bvh4 &bvh = out.tree;                               // the triangle tree, then the merged one
    Bvh4 cb, ab;                                        // curve pieces, analytic primitives
    build_bvh4(in.tris, n_tris, bvh, 0, 1e-6f*extent, opt.tri_leaf, opt.tri_cost);
    if (n_curve) build_bvh4_boxes(in.curve_boxes, n_curve, cb, 0, 1e-6f*extent, opt.curve_leaf, opt.curve_cost);
    if (in.n_analytic) {
        std::vector<BuildBox> aboxes(in.n_analytic);
        for (uint32_t k = 0; k < in.n_analytic; ++k) {
            const Aabb &b = in.analytic[k];
            // the primitives' own tests work on a point o + d*t computed in fp32: pad by the rounding of that point as well.
            // Their unpadded bounds raise the extent for this tree only (the two above are already built).
            for (int a = 0; a < 3; ++a) {
                const float pad = 4e-6f*std::max(std::fabs(b.lo[a]), std::fabs(b.hi[a]));
                aboxes[k].lo[a] = b.lo[a] - pad; aboxes[k].hi[a] = b.hi[a] + pad; aboxes[k].centroid[a] = 0.5f*(b.lo[a] + b.hi[a]);
                extent = std::max(extent, std::max(std::fabs(b.lo[a]), std::fabs(b.hi[a])));
            }
        }
        build_bvh4_boxes(aboxes.data(), in.n_analytic, ab, 0, 2e-6f*extent, 2, 2.0f);
    }
    out.analytic_order = ab.order;
    {
        // the trees that exist hang under one new root (a single tree keeps its own root), so ONE traversal answers
        // TraceableScene::intersect
        struct Sub { const Bvh4 *b; uint32_t pos_base; bool flag; };
        std::vector<Sub> subs;
        if (!bvh.nodes.empty()) subs.push_back({&bvh, 0u, false});
        if (!cb.nodes.empty()) subs.push_back({&cb, n_tris, true});
        if (!ab.nodes.empty()) subs.push_back({&ab, analytic_base, true});
        const bool rooted = subs.size() > 1;
        if (rooted || (subs.size() == 1 && subs[0].b != &bvh)) {
            size_t total = rooted ? 1 : 0;
            for (const Sub &sb : subs) total += sb.b->nodes.size();
            std::vector<Node4> merged(total);
            Node4 root = empty_node();
            float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
            uint32_t depth = 0; double sah = 0.0;
            int32_t base = rooted ? 1 : 0;
            for (size_t t = 0; t < subs.size(); ++t) {
                const Sub &sb = subs[t];
                for (size_t k = 0; k < sb.b->nodes.size(); ++k) {
                    Node4 nd = sb.b->nodes[k];
                    for (int j = 0; j < 4; ++j) {
                        if (nd.link[j] >= 0) nd.link[j] += base;
                        else if (nd.link[j] != kEmptyLink) { const int32_t code = ~nd.link[j]; nd.link[j] = ~int32_t((((code >> 3) + int32_t(sb.pos_base)) << 3) | (sb.flag ? 4 : 0) | (code & 3)); }
                    }
                    merged[size_t(base) + k] = nd;
                }
                for (int a = 0; a < 3; ++a) {
                    root.f[8*a + t] = sb.b->lo[a]; root.f[8*a + 4 + t] = sb.b->hi[a];
                    lo[a] = std::min(lo[a], sb.b->lo[a]); hi[a] = std::max(hi[a], sb.b->hi[a]);
                }
                root.link[t] = base;
                depth = std::max(depth, sb.b->max_depth); sah += sb.b->sah_cost;
                base += int32_t(sb.b->nodes.size());
            }
            if (rooted) { merged[0] = root; depth += 1; }
            std::vector<uint32_t> order = bvh.order;
            for (uint32_t k : cb.order) order.push_back(n_tris + k);
            bvh.nodes.swap(merged); bvh.order.swap(order);
            bvh.max_depth = depth; bvh.sah_cost = sah;
            for (int a = 0; a < 3; ++a) { bvh.lo[a] = lo[a]; bvh.hi[a] = hi[a]; }
        }
    }
    out.cut = top_level_cut(bvh, opt.max_cut);
    out.stack_need = traversal_stack_need(bvh, out.cut);
    out.isect.assign(size_t(n_tris) + n_curve + 1, IsectRecord{});
    for (size_t k = n_tris; k < bvh.order.size(); ++k) out.isect[k] = in.curve_recs[bvh.order[k] - n_tris];
    for (size_t k = 0; k < n_tris; ++k) {
        const BuildTri &t = in.tris[bvh.order[k]];
        float *r = out.isect[k].f;                      // v0, e1, e2, then Ng = cross(e1, e2)
        for (int a = 0; a < 3; ++a) { r[a] = t.v0[a]; r[3 + a] = t.v0[a] - t.v1[a]; r[6 + a] = t.v2[a] - t.v0[a]; }
        r[9] = r[4]*r[8] - r[5]*r[7]; r[10] = r[5]*r[6] - r[3]*r[8]; r[11] = r[3]*r[7] - r[4]*r[6];
    }
    // empty child slots link to a one-primitive leaf holding the all-zero record
    quantize_bvh4(bvh, out.qtree, ~int32_t((n_tris + n_curve) << 3));
    std::vector<int32_t> new_index(out.qtree.old_index.size());
    for (size_t i = 0; i < new_index.size(); ++i) new_index[size_t(out.qtree.old_index[i])] = int32_t(i);
    for (CutBox &b : out.cut) if (b.link >= 0) b.link = new_index[size_t(b.link)];
}

}  // namespace tgb
