// C ABI of libtgb200.so (include/tgb200.h): device upload of a prepared scene (tgb_scene.cuh), wavefront render loop.
// Host logic mirrors the reference's PathTraceIntegrator (tile dicing, sample stepping); all rendering arithmetic runs in the
// CUDA kernels of tgb_wavefront.cuh.  There is NO CPU fallback: without a CUDA device every entry point fails with
// TGB_ERR_NO_DEVICE (tgb200_create once the desc has passed its checks).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "tgb_wavefront.cuh"
#include "tgb_probe.cuh"
#include "tgb_scene.cuh"


using namespace tgb;

#include <thread>
#include <map>

namespace {

// A device array (Pinned: a page-locked host array) that frees itself; move-only.  ensure(n) re-allocates only when n exceeds
// the capacity, and frees the old array first.  cudaFree waits for the device, so a kernel still queued that reads the old
// array (k_resolve reading R) finishes before it goes.  After a failed allocation the buffer is empty.  upload(src, n, st):
// ensure(n), then the host-to-device copy of n elements queued on st.
template <typename T, bool Pinned = false>
struct Buffer {
    T *p = nullptr;
    size_t cap = 0;
    Buffer() = default;
    Buffer(Buffer &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    ~Buffer() { release(); }
    void release() {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr; cap = 0;
    }
    cudaError_t ensure(size_t n) {
        if (n <= cap) return cudaSuccess;
        release();
        void *q = nullptr;
        const cudaError_t e = Pinned ? cudaMallocHost(&q, n*sizeof(T)) : cudaMalloc(&q, n*sizeof(T));
        if (e == cudaSuccess) { p = static_cast<T *>(q); cap = n; }
        return e;
    }
    cudaError_t upload(const T *src, size_t n, cudaStream_t st) {
        const cudaError_t e = ensure(n);
        return e != cudaSuccess || n == 0 ? e : cudaMemcpyAsync(p, src, n*sizeof(T), cudaMemcpyHostToDevice, st);
    }
};

// One wavefront: the loop state of its share of a (sub)step's camera paths.  A context runs two of them, each on its own stream,
// so that one wavefront's traversal kernels (ALU bound) run alongside the other's streaming kernels (HBM bound).
struct Wavefront {
    uint32_t capacity = 0;          // path slots: half of the context's capacity
    PathBuf pb[2]{};                // persistent path state, double buffered (k_accum compacts from one into the other)
    Scratch sr{};                   // per-bounce scratch records; sr.R is the context's result buffer, shared by both wavefronts
    uint32_t *order = nullptr, *squeue = nullptr, *squeue2 = nullptr;   // ray-coherence visiting order of k_trace; shadow-query queues (emitted / left after the analytic pass)
    uint32_t *squeue_cl = nullptr;  // ... the closest-hit (mesh-light) queries left after the analytic pass
    uint32_t *bin_keys = nullptr, *bin_hist = nullptr;
    Ctl *ctl = nullptr;             // device-resident loop control block
    Buffer<Ctl, true> h_ctl;        // [0..3] snapshot ring (read one iteration late), [4] initial value
    cudaEvent_t ev_ring[4]{};
    cudaEvent_t ev_k[4][8]{};       // profiling: boundaries between the kernels of an iteration (regen|trace|shade|prep|shadow|accum|sort)
};

// The instantiations of the scene-dependent kernels a context runs (select_kernels), for renders and test hooks alike
struct Kernels {
    decltype(&k_trace<false>) trace = nullptr;
    decltype(&k_shade<false, false>) shade = nullptr;
    unsigned shade_block = 0, shade_paths = 0;      // k_shade's block size and paths per block
    decltype(&k_shadow_prep<false>) shadow_prep = nullptr;
    decltype(&k_shadow_bvh<false, false>) shadow_bvh = nullptr;
    decltype(&k_hook_persist<false>) hook_persist = nullptr;
    uint32_t variant[4] = {};       // what tgb200_shade_variant reports: curves, material-sorted, Lambert-only, quad emitters
};

}  // namespace

struct tgb_ctx;
// Multi-GPU (tgb_settings::devices): held by the root context; what it holds lives on the root's device
struct Group {
    explicit Group(std::vector<tgb_ctx *> m) : members(std::move(m)) {
        for (cudaEvent_t &e : ev_gather) if (created == cudaSuccess) created = cudaEventCreate(&e);
    }
    ~Group() { for (cudaEvent_t e : ev_gather) if (e) cudaEventDestroy(e); }
    std::vector<tgb_ctx *> members;                     // members[0] = root
    std::vector<tgb_tile> deal_key;                      // tile list the cached deal belongs to
    std::vector<std::vector<tgb_tile>> shares;           // per member
    std::vector<Buffer<uint32_t>> root_pix;              // per member k >= 1: its share's pixel ids
    std::vector<uint32_t> share_pixels;
    Buffer<float4> recv;                                 // one member's packed share at a time
    cudaEvent_t ev_gather[2] = {};
    cudaError_t created = cudaSuccess;                   // the first error of the constructor's event creation
    double gather_ms = 0.0;
};

struct tgb_ctx {
    explicit tgb_ctx(int dev);      // on the current device, dev: the streams and events (created: the first error)
    ~tgb_ctx();
    int device = 0;
    cudaError_t created = cudaSuccess;
    cudaStream_t stream = nullptr;  // the caller's stream (tgb200_set_stream) or own_stream: wavefront 0, k_resolve, the hooks
    cudaStream_t stream1 = nullptr; // wavefront 1
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    std::string error;
    std::atomic<int> abort_flag{0};
    std::vector<Buffer<uint8_t>> arena;   // the allocations made once by tgb200_create (dev_alloc): scene, wavefronts, framebuffer
    DScene sc{};
    uint32_t res_x = 0, res_y = 0;
    // wavefront storage
    uint32_t capacity = 0;          // paths in flight, both wavefronts together
    Wavefront wf[2];                // the hooks run on wf[0]'s buffers
    uint32_t persist_blocks = 0;    // grid of the persistent traversal kernels (per wavefront)
    uint32_t regen_blocks = 0, prep_blocks = 0, scatter_blocks = 0;   // largest grids of the grid-stride kernels (resident blocks)
    bool has_curves = false;        // the probes pick their instantiations with the curve-segment test and per-hit epsilon
    Kernels ks;                     // the instantiations select_kernels chose for the scene
    int n_bsdfs = 0; std::vector<uint32_t> prim_types; std::vector<int> light_ids;   // host copies for the test hooks' argument checks
    Buffer<float4> R;               // finished radiance per path of the (sub)step
    cudaStream_t own_stream = nullptr;
    std::unique_ptr<Group> group;   // multi-GPU: set on the root context (devices[0]); members[0] == the root itself
    Buffer<float4> send;            // multi-GPU member: its share's pixels packed for the gather on the root
    Counters *ctr = nullptr; Buffer<Counters, true> h_ctr;
    float *fb = nullptr; uint32_t *fb_count = nullptr;
    Buffer<float, true> h_fb; Buffer<uint32_t, true> h_fb_count;   // staging
    // cached pixel list
    std::vector<tgb_tile> tiles_cached; Buffer<uint32_t> pix_id, pix_seed; uint32_t n_pix = 0;
    std::vector<uint32_t> h_pix_id;                  // host copy of the pixel list (adaptive steps build per-pixel sample ranges from it)
    // adaptive sampling: per-pixel result-slot offsets / first sample index, pixel -> list index map, the 4x4 blocks' SampleRecords
    Buffer<uint32_t> pix_first, pix_base, pix_slot; bool pix_slot_valid = false;
    Buffer<SampleRecordD> rec_dev;
    tgb_stats stats{};
    bool profiling = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint32_t bvh_depth = 0; uint32_t n_tris = 0; double bvh_sah = 0.0; size_t geom_bytes = 0;
};

tgb_ctx::tgb_ctx(int dev) : device(dev) {
    cudaError_t &e = created;
    for (cudaStream_t *s : {&own_stream, &stream1}) if (e == cudaSuccess) e = cudaStreamCreateWithFlags(s, cudaStreamNonBlocking);
    for (cudaEvent_t *v : {&ev0, &ev1}) if (e == cudaSuccess) e = cudaEventCreate(v);
    for (cudaEvent_t *v : {&ev_fork, &ev_join}) if (e == cudaSuccess) e = cudaEventCreateWithFlags(v, cudaEventDisableTiming);
    for (Wavefront &w : wf)
        for (int k = 0; k < 4; ++k) {
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&w.ev_ring[k], cudaEventDisableTiming);
            for (cudaEvent_t &v : w.ev_k[k]) if (e == cudaSuccess) e = cudaEventCreate(&v);
        }
    stream = own_stream;
}

tgb_ctx::~tgb_ctx() {
    for (cudaEvent_t v : {ev0, ev1, ev_fork, ev_join}) if (v) cudaEventDestroy(v);
    for (Wavefront &w : wf)
        for (int k = 0; k < 4; ++k) { if (w.ev_ring[k]) cudaEventDestroy(w.ev_ring[k]); for (cudaEvent_t v : w.ev_k[k]) if (v) cudaEventDestroy(v); }
    for (cudaStream_t s : {stream1, own_stream}) if (s) cudaStreamDestroy(s);
}

namespace {

int fail(tgb_ctx *c, int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    if (c) c->error = buf; else g_create_error = buf;
    return code;
}

#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return fail(c, e_ == cudaErrorMemoryAllocation ? TGB_ERR_OOM : TGB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

template <typename T>
int dev_alloc(tgb_ctx *c, T **out, size_t n) {
    c->arena.emplace_back();
    CU(c->arena.back().ensure(std::max<size_t>(n, 1)*sizeof(T)));
    *out = reinterpret_cast<T *>(c->arena.back().p);
    return TGB_OK;
}
template <typename T>
int dev_upload(tgb_ctx *c, const T **out, const std::vector<T> &v) {
    T *p = nullptr;
    int rc = dev_alloc(c, &p, v.size());
    if (rc) return rc;
    if (!v.empty()) CU(cudaMemcpy(p, v.data(), v.size()*sizeof(T), cudaMemcpyHostToDevice));
    *out = p;
    return TGB_OK;
}

// The kernel instantiations of a scene.  k_shade: material-sorted (>= 2 lobe models in use, or TGB_SORT_MATERIALS=1; =0 never),
// then with curves, then the emitter set, then Lambert-only (TGB_LOBE_SET=0 turns the last two off), then the generic one.
Kernels select_kernels(const SceneKind &s) {
    const bool cv = s.has_curves;
    // every surface Lambert (lights: null BSDF): k_shade's lobe-set-1 instantiation (same arithmetic, a fraction of the code)
    const char *ls = getenv("TGB_LOBE_SET"), *sm = getenv("TGB_SORT_MATERIALS");
    const bool diffuse_only = (s.bsdf_types & ~(1u << TGB_BSDF_LAMBERT)) == 0 && !cv && !(ls && ls[0] == '0');
    const bool sort_materials = !diffuse_only && (sm ? sm[0] == '1' : __builtin_popcount(s.bsdf_types) >= 2);
    // ... and every light a quad, no infinite emitter, every BSDF albedo and emission texture constant: the emitter-set-1
    // instantiation of it (k_shade<false, false, 1, 1>: the same arithmetic without the other emitters' and textures' code)
    const bool quad_emitters = diffuse_only && s.quad_lights && TGB_QUAD_EMITTERS;
    Kernels k;
    k.trace = cv ? k_trace<true> : k_trace<false>;
    if (sort_materials) {
        k.shade = cv ? k_shade<true, true> : k_shade<false, true>;
        k.shade_block = kShadeSortBlock; k.shade_paths = kShadeSortBlock*kShadeSortItems;
    } else {
        k.shade = cv ? k_shade<true, false> : quad_emitters ? k_shade<false, false, 1, 1> : diffuse_only ? k_shade<false, false, 1> : k_shade<false, false>;
        k.shade_block = 128; k.shade_paths = 128;
    }
    k.shadow_prep = cv ? k_shadow_prep<true> : k_shadow_prep<false>;
    k.shadow_bvh = cv ? (s.mesh_lights ? k_shadow_bvh<true, true> : k_shadow_bvh<true, false>)
                      : (s.mesh_lights ? k_shadow_bvh<false, true> : k_shadow_bvh<false, false>);
    k.hook_persist = cv ? k_hook_persist<true> : k_hook_persist<false>;
    k.variant[0] = cv; k.variant[1] = sort_materials; k.variant[2] = diffuse_only; k.variant[3] = quad_emitters;
    return k;
}

// The only function that puts scene data on the device: a prepared scene's arrays, and the records that point to them
int upload_scene(tgb_ctx *c, const HostScene &hs, const Kernels &ks) {
    DScene &sc = c->sc;
    sc = hs.sc;
    int rc;
    std::vector<DTex> dtex(hs.tex.size());
    for (size_t i = 0; i < hs.tex.size(); ++i) {
        const HostTex &t = hs.tex[i]; DTex &o = dtex[i] = t.d;
        if (o.type == TGB_TEX_BITMAP && (rc = dev_upload(c, &o.texels, t.texels))) return rc;
        if (t.has_dist) {
            if ((rc = dev_upload(c, &o.marg_pdf, t.marg_pdf))) return rc;
            if ((rc = dev_upload(c, &o.marg_cdf, t.marg_cdf))) return rc;
            if ((rc = dev_upload(c, &o.pdf, t.pdf))) return rc;
            if ((rc = dev_upload(c, &o.cdf, t.cdf))) return rc;
        }
    }
    std::vector<DBsdf> bsdfs = hs.bsdfs;
    for (size_t i = 0; i < bsdfs.size(); ++i) {
        if (bsdfs[i].type != TGB_BSDF_HAIR) continue;
        for (int p = 0; p < 3; ++p) {
            const HairLobeTables &l = hs.hair[i].lobe[p];
            if ((rc = dev_upload(c, &bsdfs[i].hair_table[p], l.table))) return rc;
            if ((rc = dev_upload(c, &bsdfs[i].hair_pdfs[p], l.pdfs))) return rc;
            if ((rc = dev_upload(c, &bsdfs[i].hair_cdfs[p], l.cdfs))) return rc;
            if ((rc = dev_upload(c, &bsdfs[i].hair_sums[p], l.sums))) return rc;
        }
    }
    std::vector<DPrim> prims = hs.prims;
    for (const MeshLight &m : hs.mesh_lights) {
        DPrim &o = prims[m.prim];
        if ((rc = dev_upload(c, &o.tri_pdf, m.pdf))) return rc;
        if ((rc = dev_upload(c, &o.tri_cdf, m.cdf))) return rc;
        if ((rc = dev_upload(c, &o.light_verts, m.verts))) return rc;
    }
    if ((rc = dev_upload(c, &sc.prims, prims))) return rc;
    if ((rc = dev_upload(c, &sc.bsdfs, bsdfs))) return rc;
    if ((rc = dev_upload(c, &sc.slots, hs.slots))) return rc;
    if ((rc = dev_upload(c, &sc.tex, dtex))) return rc;
    if ((rc = dev_upload(c, &sc.lights, hs.lights))) return rc;
    if ((rc = dev_upload(c, &sc.inf_lights, hs.inf_lights))) return rc;
    if ((rc = dev_upload(c, &sc.analytic, hs.analytic))) return rc;
    if ((rc = dev_upload(c, &sc.tri_global, hs.bvh.tree.order))) return rc;
    if ((rc = dev_upload(c, &sc.tri_prim, hs.tri_prim))) return rc;
    if ((rc = dev_upload(c, &sc.tri_shade, hs.tri_shade))) return rc;
    static_assert(sizeof(IsectRecord) == 3*sizeof(float4), "intersection record layout");
    const IsectRecord *ir = nullptr;
    if ((rc = dev_upload(c, &ir, hs.bvh.isect))) return rc;
    sc.tri_isect = reinterpret_cast<const float4 *>(ir);
    const QNode4 *qn = nullptr;
    if ((rc = dev_upload(c, &qn, hs.bvh.qtree.nodes))) return rc;
    sc.qnodes = reinterpret_cast<const uint4 *>(qn);
    if ((rc = dev_upload(c, &sc.sobol, hs.sobol))) return rc;
    if (ks.variant[3]) {    // the emitter-set k_shade reads its BSDFs as 16-byte records: constant albedo, type | lobes << 16 (lambert_rec)
        std::vector<float4> lam(bsdfs.size());
        for (size_t i = 0; i < bsdfs.size(); ++i) {
            const DBsdf &b = bsdfs[i];
            const V3 a = dtex[size_t(b.albedo_tex)].value;
            const uint32_t w = (b.type & 0xFFFFu) | (b.lobes << 16);
            float wf; std::memcpy(&wf, &w, 4);
            lam[i] = make_float4(a.x, a.y, a.z, wf);
        }
        if ((rc = dev_upload(c, &sc.lambert, lam))) return rc;
    }
    // host copies for the test hooks and tgb200_scene_info
    c->res_x = sc.cam.res_x; c->res_y = sc.cam.res_y;
    c->has_curves = hs.kind.has_curves;
    c->n_bsdfs = int(bsdfs.size());
    c->prim_types.resize(prims.size());
    for (size_t i = 0; i < prims.size(); ++i) c->prim_types[i] = prims[i].type;
    c->light_ids = hs.lights;
    const Bvh4 &bvh = hs.bvh.tree;
    c->bvh_depth = bvh.max_depth; c->n_tris = sc.n_tris; c->bvh_sah = bvh.sah_cost;
    c->geom_bytes = hs.bvh.qtree.nodes.size()*sizeof(QNode4) + hs.bvh.isect.size()*sizeof(IsectRecord) + hs.tri_shade.size()*16 + bvh.order.size()*8;
    return TGB_OK;
}

int alloc_wavefront(tgb_ctx *c, uint32_t capacity) {
    c->capacity = capacity;
    int rc;
    for (int h = 0; h < 2; ++h) {
        Wavefront &w = c->wf[h];
        const uint32_t cap = w.capacity = capacity/2 + (h == 0 ? capacity % 2 : 0);
        for (int k = 0; k < 2; ++k) {
            for (float4 **p : {&w.pb[k].T0, &w.pb[k].T1, &w.pb[k].T2, &w.pb[k].T3}) if ((rc = dev_alloc(c, p, cap))) return rc;
            if ((rc = dev_alloc(c, &w.pb[k].E, cap))) return rc;
            if ((rc = dev_alloc(c, &w.pb[k].pcg, cap))) return rc;
        }
        for (float4 **p : {&w.sr.P, &w.sr.N0, &w.sr.N1, &w.sr.M0, &w.sr.M1, &w.sr.D0, &w.sr.D1})
            if ((rc = dev_alloc(c, p, cap))) return rc;
        if ((rc = dev_alloc(c, &w.sr.vis, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.sr.SH, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.sr.cut_mask, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.squeue, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.squeue2, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.squeue_cl, size_t(cap)*2))) return rc;
        if ((rc = dev_alloc(c, &w.order, cap))) return rc;
        if ((rc = dev_alloc(c, &w.bin_keys, cap))) return rc;
        if ((rc = dev_alloc(c, &w.bin_hist, size_t(kBins) + 4))) return rc;
        if ((rc = dev_alloc(c, &w.ctl, 1))) return rc;
        CU(cudaMemset(w.ctl, 0, sizeof(Ctl)));
        CU(w.h_ctl.ensure(5));
    }
    if ((rc = dev_alloc(c, &c->ctr, 1))) return rc;
    CU(cudaMemset(c->ctr, 0, sizeof(Counters)));
    CU(c->h_ctr.ensure(1));
    size_t npx = size_t(c->res_x)*c->res_y;
    if ((rc = dev_alloc(c, &c->fb, npx*3))) return rc;
    if ((rc = dev_alloc(c, &c->fb_count, npx))) return rc;
    CU(cudaMemset(c->fb, 0, npx*3*sizeof(float)));
    CU(cudaMemset(c->fb_count, 0, npx*sizeof(uint32_t)));
    CU(c->h_fb.ensure(npx*3));
    CU(c->h_fb_count.ensure(npx));
    return TGB_OK;
}

// The tile list of a render call: the caller's or, when n_tiles == 0, the reference's (PathTraceIntegrator::diceTiles + the
// sampler seeding of prepareForRender, PathTraceIntegrator.cpp:27-42,187)
std::vector<tgb_tile> call_tiles(const tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed) {
    if (n_tiles) return std::vector<tgb_tile>(tiles, tiles + n_tiles);
    const uint32_t TileSize = 16, w = c->res_x, h = c->res_y;
    uint64_t st = uint64_t(hash32(seed));
    std::vector<tgb_tile> out;
    for (uint32_t y = 0; y < h; y += TileSize)
        for (uint32_t x = 0; x < w; x += TileSize) {
            tgb_tile t; t.x = x; t.y = y; t.w = std::min(TileSize, w - x); t.h = std::min(TileSize, h - y);
            t.sampler_seed = hash32(pcg_next(st));
            out.push_back(t);
        }
    return out;
}

// a tile list equal to the one whose pixel list is already built
bool same_tiles(const std::vector<tgb_tile> &a, const std::vector<tgb_tile> &b) {
    return !a.empty() && a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size()*sizeof(tgb_tile)) == 0;
}

// The pixel ids of a tile list, tile-major, and (pseed) each pixel's tile seed.  The tiles must lie inside the image and be
// disjoint: k_resolve, k_unpack_tiles and k_unpack_share own one pixel per thread, and a multi-GPU context would render a pixel
// of two tiles on two GPUs.
int tile_pixels(tgb_ctx *c, const std::vector<tgb_tile> &tiles, std::vector<uint32_t> &pid, std::vector<uint32_t> *pseed = nullptr) {
    pid.clear();
    if (pseed) pseed->clear();
    for (size_t t = 0; t < tiles.size(); ++t) {
        const tgb_tile &tl = tiles[t];
        if (tl.x >= c->res_x || tl.w > c->res_x - tl.x || tl.y >= c->res_y || tl.h > c->res_y - tl.y) return fail(c, TGB_ERR_INVALID, "tile %zu lies outside the image", t);
        for (uint32_t y = 0; y < tl.h; ++y) for (uint32_t x = 0; x < tl.w; ++x) pid.push_back((tl.x + x) + (tl.y + y)*c->res_x);
        if (pseed) pseed->resize(pid.size(), tl.sampler_seed);
    }
    std::vector<bool> seen(size_t(c->res_x)*c->res_y, false);
    for (uint32_t q : pid) { if (seen[q]) return fail(c, TGB_ERR_INVALID, "tile list covers pixel %u twice", q); seen[q] = true; }
    return TGB_OK;
}

int set_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed) {
    std::vector<tgb_tile> list = call_tiles(c, tiles, n_tiles, seed);
    if (same_tiles(list, c->tiles_cached)) return TGB_OK;
    std::vector<uint32_t> pid, pseed;
    if (int rc = tile_pixels(c, list, pid, &pseed)) return rc;
    c->tiles_cached.clear();                                    // (until the new list is on the device)
    c->n_pix = uint32_t(pid.size());
    c->h_pix_id = pid; c->pix_slot_valid = false;
    CU(c->pix_id.upload(pid.data(), pid.size(), c->stream));
    CU(c->pix_seed.upload(pseed.data(), pseed.size(), c->stream));
    CU(cudaStreamSynchronize(c->stream));
    c->tiles_cached = std::move(list);
    return TGB_OK;
}

inline unsigned blocks(uint32_t n, unsigned bs) { return n ? (n + bs - 1)/bs : 1; }
// Grid of a grid-stride loop kernel (k_regen, k_shadow_prep, k_bin_scatter: 256 threads) for at most `bound` items: the blocks
// they need, at most `resident` (the context's regen_blocks, prep_blocks or scatter_blocks).  Renders and probes alike.
inline unsigned loop_grid(uint32_t resident, uint32_t bound) { return std::min(blocks(bound, 256), resident); }

// The wavefront loop: the GPU analogue of renderTile over (pixels of the tiles) x (sample range), with path
// regeneration: whenever paths finish, their slots are refilled with the next camera paths of the step, so every
// iteration traces a full batch until the step's paths run out (one drain tail per step instead of one per batch).
int ensure_results(tgb_ctx *c, size_t n_paths) {
    const cudaError_t e = c->R.ensure(n_paths);
    for (Wavefront &w : c->wf) w.sr.R = c->R.p;               // (null after a failed allocation)
    CU(e);
    return TGB_OK;
}

// One bounce of wavefront w's paths in pb on stream st: k_trace -> k_shade -> k_shadow_prep -> k_shadow_bvh -> k_accum (survivors
// into nxt), as a render and tgb200_bounce_probe run it.  `bound` >= ctl.n: grids are upper bounds, the kernels read the real
// sizes from the device-resident control block (k_shadow_prep loops over them with at most the resident blocks).  ev (profiling):
// events recorded after each of the five kernels.  Returns the number of kernels launched.
uint32_t enqueue_bounce(tgb_ctx *c, Wavefront &w, const PathBuf &pb, const PathBuf &nxt, cudaStream_t st, const BatchInfo &bi,
                        uint32_t bound, const cudaEvent_t *ev) {
    const DScene &sc = c->sc; const Kernels &ks = c->ks;
    const bool has_bvh = sc.n_nodes != 0;
    if (has_bvh) ks.trace<<<std::min(blocks(bound, kTraceBlock), c->persist_blocks), kTraceBlock, 0, st>>>(sc, pb, w.order, w.ctl);
    if (ev) cudaEventRecord(ev[0], st);
    ks.shade<<<blocks(bound, ks.shade_paths), ks.shade_block, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
    if (ev) cudaEventRecord(ev[1], st);
    ks.shadow_prep<<<loop_grid(c->prep_blocks, 2*bound), 256, 0, st>>>(sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
    if (ev) cudaEventRecord(ev[2], st);
    // the any-hit queue and (scenes with mesh lights) the closest-hit queue
    if (has_bvh) ks.shadow_bvh<<<std::min(blocks(2*bound, kTraceBlock), c->persist_blocks), kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
    if (ev) cudaEventRecord(ev[3], st);
    k_accum<<<blocks(bound, 256), 256, 0, st>>>(sc, pb, nxt, w.sr, bi, w.ctl, w.bin_keys, w.bin_hist);
    if (ev) cudaEventRecord(ev[4], st);
    return has_bvh ? 5 : 3;
}

// One iteration's kernels of wavefront w on stream st: k_regen, a bounce, and the ray-coherence binning of the survivors
void enqueue_iteration(tgb_ctx *c, Wavefront &w, cudaStream_t st, const BatchInfo &bi, int cur, uint32_t bound, int slot, uint64_t &launches) {
    const DScene &sc = c->sc;
    const bool has_bvh = sc.n_nodes != 0;
    PathBuf &pb = w.pb[cur], &nxt = w.pb[cur ^ 1];
    const bool prof = c->profiling;
    if (prof) cudaEventRecord(w.ev_k[slot][0], st);
    k_regen<<<loop_grid(c->regen_blocks, bound), 256, 0, st>>>(sc, pb, bi, w.ctl, w.order, w.bin_hist); launches++;
    if (prof) cudaEventRecord(w.ev_k[slot][1], st);
    launches += enqueue_bounce(c, w, pb, nxt, st, bi, bound, prof ? &w.ev_k[slot][2] : nullptr);
    k_iter_end<<<1, 1024, 0, st>>>(w.bin_hist, w.ctl, has_bvh ? 1 : 0); launches++;
    if (has_bvh) { k_bin_scatter<<<loop_grid(c->scatter_blocks, bound), 256, 0, st>>>(w.bin_keys, w.bin_hist, w.ctl, w.order); launches++; }
    if (prof) cudaEventRecord(w.ev_k[slot][7], st);
}

// A step's finished radiances are kept per path (16 B each) until k_resolve folds them in sample order.  A pass holds at
// most this many paths, so that buffer stays within 8 GiB.
constexpr uint64_t kPassPaths = 512ull << 20;
// bits of an index into a list of n pixels: a path id is (sample within the pass << index_bits) | pixel index
inline uint32_t index_bits(uint64_t n) { uint32_t b = 0; while (b < 32 && (uint64_t(1) << b) < n) ++b; return b; }

// `run`: one run of an adaptive step (single_render_adaptive): its pixels, their result-slot offsets and first sample indices,
// `run_total` paths in one pass.  Else every pixel of the call renders samples [spp_begin, spp_begin + spp_count).
int render_device(tgb_ctx *c, uint32_t spp_begin, uint32_t spp_count, const BatchInfo *run = nullptr, uint32_t run_total = 0) {
    const uint32_t n_pix = run ? run->n_pix : c->n_pix;
    if (n_pix == 0 || (!run && spp_count == 0) || (run && run_total == 0)) return TGB_OK;
    CU(cudaEventRecord(c->ev0, c->stream));
    uint64_t launches = 0;
    float trace_ms = 0.0f, shadow_ms = 0.0f; uint64_t trace_launches = 0, shadow_launches = 0, traversed = 0, shadow_traversed = 0;
    double kms[7] = {0, 0, 0, 0, 0, 0, 0}; uint64_t iterations = 0;
    // split the sample range into passes of at most kPassPaths paths whose (sample within the pass, pixel) fits 32 bits
    const uint32_t pix_bits = index_bits(n_pix);
    const uint64_t max_k = uint64_t(1) << (32 - pix_bits);
    uint32_t spp_sub = run ? 1u : uint32_t(std::max<uint64_t>(1, std::min<uint64_t>(std::min<uint64_t>(spp_count, max_k), kPassPaths/n_pix)));
    if (uint64_t(n_pix)*spp_sub > 0xFFFFFFFFull) return fail(c, TGB_ERR_UNSUPPORTED, "tile list too large");
    if (run) spp_count = 1;                                    // one pass over the per-pixel ranges
    const bool trace_bounces = getenv("TGB_TRACE_BOUNCES") != nullptr;
    uint64_t samples_done = 0;
    for (uint32_t s0 = 0; s0 < spp_count; s0 += spp_sub) {
        uint32_t ns = std::min(spp_sub, spp_count - s0);
        uint32_t total = run ? run_total : n_pix*ns;
        samples_done += total;
        int rc = ensure_results(c, total);
        if (rc) return rc;
        BatchInfo bi;
        if (run) bi = *run;
        else { bi.pix_id = c->pix_id.p; bi.pix_seed = c->pix_seed.p; bi.n_pix = n_pix; bi.pix_first = nullptr; bi.pix_base = nullptr; bi.pix_bits = pix_bits; }
        bi.spp_begin = spp_begin + s0;
        // fork: wavefront 1 starts behind what the caller's stream holds so far (the previous sub-step's k_resolve reads R)
        const cudaStream_t st[2] = {c->stream, c->stream1};
        CU(cudaEventRecord(c->ev_fork, st[0]));
        CU(cudaStreamWaitEvent(st[1], c->ev_fork, 0));
        // The (sub)step's path ids (result slots) are split statically: wavefront h issues the camera paths [base, end).  The
        // image cannot depend on the split (every path seeds its own RNG and writes R[path id], DESIGN.md section 3).
        const uint32_t half = total - total/2;
        uint32_t bound[2] = {0, 0};                           // upper bound of ctl.n for the iteration about to be queued
        int cur[2] = {0, 0};
        bool live[2] = {false, false};
        for (int h = 0; h < 2; ++h) {
            Wavefront &w = c->wf[h];
            const uint32_t base = h ? half : 0, end = h ? total : half;
            if (end == base) continue;
            // control block of the first iteration; from then on k_iter_end keeps it
            Ctl &init = w.h_ctl.p[4];
            std::memset(&init, 0, sizeof(Ctl));
            init.capacity = w.capacity; init.total = end; init.first_path = base;
            init.n_new = std::min(w.capacity, end - base); init.n = init.n_new; init.issued = base + init.n_new;
            CU(cudaMemcpyAsync(w.ctl, &init, sizeof(Ctl), cudaMemcpyHostToDevice, st[h]));
            bound[h] = init.n; live[h] = true;
        }
        // The host runs one iteration ahead of the device: after enqueueing iteration i of both wavefronts it waits for their
        // snapshots taken after iteration i-1 (normally long complete), which bound the grids of iteration i+1 and tell when a
        // wavefront has drained; a drained wavefront is no longer enqueued.
        for (uint32_t iter = 0; live[0] || live[1]; ++iter) {
            if (c->abort_flag.load()) { cudaStreamSynchronize(st[1]); cudaStreamSynchronize(st[0]); c->abort_flag.store(0); return fail(c, TGB_ERR_ABORTED, "render aborted"); }
            const int slot = int(iter & 3u);
            for (int h = 0; h < 2; ++h) {
                if (!live[h]) continue;
                Wavefront &w = c->wf[h];
                enqueue_iteration(c, w, st[h], bi, cur[h], bound[h], slot, launches);
                cur[h] ^= 1;
                CU(cudaMemcpyAsync(&w.h_ctl.p[slot], w.ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, st[h]));
                CU(cudaEventRecord(w.ev_ring[slot], st[h]));
            }
            if (iter == 0) continue;                          // nothing known yet about iteration 1: its bound stays the first one
            const int p = int((iter - 1) & 3u);
            for (int h = 0; h < 2; ++h) {
                if (!live[h]) continue;
                Wavefront &w = c->wf[h];
                CU(cudaEventSynchronize(w.ev_ring[p]));
                const Ctl S = w.h_ctl.p[p];                   // state after iteration iter-1 = the sizes of iteration iter
                if (c->profiling) {
                    for (int k = 0; k < 7; ++k) { float ms = 0.0f; cudaEventElapsedTime(&ms, w.ev_k[p][k], w.ev_k[p][k + 1]); kms[k] += ms; }
                    trace_launches++; shadow_launches++;       // one k_trace and one k_shadow_bvh per timed iteration
                }
                if (trace_bounces) fprintf(stderr, "wavefront %d after iter %u: next n %u (survivors %u, new %u, to traverse %u) issued %u/%u\n", h, iter - 1, S.n, S.n_surv, S.n_new, S.n_sorted, S.issued, S.total);
                if (S.n == 0) { traversed += S.traversed; shadow_traversed += S.shadow_traversed; iterations += S.iterations; live[h] = false; continue; }   // iteration `iter`, already queued, is empty
                // n(iter+1) <= n(iter) + the camera paths not yet issued after iteration iter's refill
                bound[h] = uint32_t(std::min<uint64_t>(w.capacity, uint64_t(S.n) + (S.total - S.issued)));
            }
            if (iter > (1u << 24)) return fail(c, TGB_ERR_INVALID, "wavefront loop did not terminate");
        }
        // join: k_resolve, and whatever the caller queues on its stream after this call, wait for wavefront 1
        CU(cudaEventRecord(c->ev_join, st[1]));
        CU(cudaStreamWaitEvent(st[0], c->ev_join, 0));
        k_resolve<<<blocks(n_pix, 256), 256, 0, st[0]>>>(c->R.p, bi, ns, c->fb, c->fb_count); launches++;
    }
    CU(cudaEventRecord(c->ev1, c->stream));
    CU(cudaMemcpyAsync(c->h_ctr.p, c->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
    float ms = 0.0f; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
    c->stats.samples += samples_done;
    c->stats.path_rays = c->h_ctr.p->rays; c->stats.shadow_rays = c->h_ctr.p->shadow_rays;
    c->stats.rays = c->h_ctr.p->rays + c->h_ctr.p->shadow_rays; c->stats.hits = c->h_ctr.p->hits + c->h_ctr.p->shadow_hits;
    trace_ms = float(kms[1]); shadow_ms = float(kms[4]);
    c->stats.regen_ms += kms[0]; c->stats.shade_ms += kms[2]; c->stats.prep_ms += kms[3]; c->stats.accum_ms += kms[5]; c->stats.sort_ms += kms[6];
    c->stats.iterations += iterations;
    c->stats.shadow_ms += shadow_ms; c->stats.shadow_launches += shadow_launches;
    c->stats.kernel_launches += launches;
    c->stats.path_rays_traversed += traversed; c->stats.shadow_rays_traversed += shadow_traversed;
    c->stats.total_ms += ms; c->stats.trace_ms += trace_ms; c->stats.trace_launches += trace_launches;
    return TGB_OK;
}

int single_render_resident(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count) {
    CU(cudaSetDevice(c->device));
    int rc = set_tiles(c, tiles, n_tiles, seed);
    if (rc) return rc;
    return render_device(c, spp_begin, spp_count);
}

int single_render_adaptive(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, tgb_sample_record *records) {
    static_assert(sizeof(tgb_sample_record) == sizeof(SampleRecordD), "record layout");
    CU(cudaSetDevice(c->device));
    int rc = set_tiles(c, tiles, n_tiles, seed);
    if (rc) return rc;
    const uint32_t var_w = (c->res_x + 3)/4, var_h = (c->res_y + 3)/4, n_blocks = var_w*var_h;
    if (c->n_pix == 0) return TGB_OK;
    std::vector<uint32_t> cnt(c->n_pix), base(size_t(c->n_pix) + 1, 0);
    for (uint32_t i = 0; i < c->n_pix; ++i) {
        const uint32_t px = c->h_pix_id[i] % c->res_x, py = c->h_pix_id[i]/c->res_x;
        const tgb_sample_record &r = records[px/4 + (py/4)*var_w];
        cnt[i] = r.next_sample_count; base[i] = r.sample_index;
    }
    // The step renders in runs of consecutive tiles of the list (the list is tile-major: a run is a range of c->pix_id), one
    // pass each: at most kPassPaths paths, and every pixel's count fits the run's path ids.  A 4x4 block lies inside one
    // tile, so its samples fold in one run, in renderTile's order, and the image and records do not depend on the runs.
    struct Run { uint32_t p0, n, max_cnt; uint64_t total; };
    const auto one_pass = [](uint32_t n, uint64_t total, uint32_t max_cnt) {
        return total <= kPassPaths && uint64_t(max_cnt) <= (uint64_t(1) << (32 - index_bits(n)));
    };
    std::vector<Run> runs;
    uint64_t step_total = 0;
    for (uint32_t t = 0, p = 0; t < c->tiles_cached.size(); ++t) {
        const tgb_tile &tl = c->tiles_cached[t];
        const uint32_t n = tl.w*tl.h;
        if (n == 0) continue;
        uint64_t total = 0; uint32_t max_cnt = 0;
        for (uint32_t i = p; i < p + n; ++i) { total += cnt[i]; max_cnt = std::max(max_cnt, cnt[i]); }
        if (!one_pass(n, total, max_cnt))
            return fail(c, TGB_ERR_UNSUPPORTED, "adaptive step: tile %u at (%u, %u) renders %llu paths, %u for one pixel: more than one pass holds",
                        t, tl.x, tl.y, (unsigned long long)total, max_cnt);
        if (runs.empty() || !one_pass(runs.back().n + n, runs.back().total + total, std::max(runs.back().max_cnt, max_cnt))) runs.push_back(Run{p, 0, 0, 0});
        Run &r = runs.back();
        r.n += n; r.total += total; r.max_cnt = std::max(r.max_cnt, max_cnt);
        p += n; step_total += total;
    }
    // run k's result-slot offsets (n + 1 of them, from 0) start at pix_first[p0 + k]
    std::vector<uint32_t> first(size_t(c->n_pix) + runs.size());
    for (size_t k = 0; k < runs.size(); ++k) {
        uint32_t *f = first.data() + runs[k].p0 + k, slot = 0;
        for (uint32_t i = 0; i < runs[k].n; ++i) { f[i] = slot; slot += cnt[runs[k].p0 + i]; }
        f[runs[k].n] = slot;
    }
    if (!c->pix_slot_valid) {
        std::vector<uint32_t> slot(size_t(c->res_x)*c->res_y, 0xFFFFFFFFu);
        for (uint32_t i = 0; i < c->n_pix; ++i) slot[c->h_pix_id[i]] = i;
        CU(c->pix_slot.upload(slot.data(), slot.size(), c->stream));
        CU(cudaStreamSynchronize(c->stream));
        c->pix_slot_valid = true;
    }
    CU(c->pix_first.upload(first.data(), first.size(), c->stream));
    CU(c->pix_base.upload(base.data(), base.size(), c->stream));
    CU(c->rec_dev.upload(reinterpret_cast<const SampleRecordD *>(records), n_blocks, c->stream));
    CU(cudaStreamSynchronize(c->stream));                       // (the host vectors go out of scope)
    if (step_total == 0) return TGB_OK;
    for (size_t k = 0; k < runs.size(); ++k) {
        const Run &r = runs[k];
        if (r.total == 0) continue;
        BatchInfo bi; bi.pix_id = c->pix_id.p + r.p0; bi.pix_seed = c->pix_seed.p + r.p0; bi.n_pix = r.n; bi.spp_begin = 0;
        bi.pix_first = c->pix_first.p + r.p0 + k; bi.pix_base = c->pix_base.p + r.p0; bi.pix_bits = index_bits(r.n);
        if ((rc = render_device(c, 0, 0, &bi, uint32_t(r.total)))) return rc;
        k_block_stats<<<blocks(n_blocks, 128), 128, 0, c->stream>>>(c->R.p, bi, c->pix_slot.p, r.p0, c->res_x, c->res_y, var_w, n_blocks, c->rec_dev.p);
        c->stats.kernel_launches++;
    }
    CU(cudaMemcpyAsync(records, c->rec_dev.p, size_t(n_blocks)*sizeof(SampleRecordD), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
    return TGB_OK;
}

// apply f to every member of a multi-GPU context (the root last, so that the current device ends up being the root's)
template <class F> int for_members(tgb_ctx *c, F f) {
    if (!c->group) return TGB_OK;
    Group *g = c->group.get();
    for (size_t k = g->members.size(); k-- > 1;) { int rc = f(g->members[k]); if (rc) { c->error = g->members[k]->error; return rc; } }
    return TGB_OK;
}

// ---- multi-GPU group (tgb_settings::devices) ----------------------------------------------------------------------
uint32_t morton2(uint32_t x, uint32_t y) {
    auto part = [](uint32_t v) { v &= 0xFFFFu; v = (v | (v << 8)) & 0x00FF00FFu; v = (v | (v << 4)) & 0x0F0F0F0Fu; v = (v | (v << 2)) & 0x33333333u; v = (v | (v << 1)) & 0x55555555u; return v; };
    return part(x) | (part(y) << 1);
}
void shard_order(const tgb_tile *tiles, uint32_t n, std::vector<uint32_t> &order) {
    order.resize(n);
    for (uint32_t i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return morton2(tiles[a].x/16u, tiles[a].y/16u) < morton2(tiles[b].x/16u, tiles[b].y/16u); });
}

// Deal the call's tiles to the members (Morton order, round-robin) and make sure the root knows every share's pixel list.
int group_deal(tgb_ctx *root, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed) {
    tgb_ctx *c = root; Group &g = *root->group;
    std::vector<tgb_tile> list = call_tiles(root, tiles, n_tiles, seed);
    if (same_tiles(list, g.deal_key)) return TGB_OK;
    g.deal_key.clear();                                         // (until the new deal is complete)
    std::vector<uint32_t> pid;
    if (int rc = tile_pixels(root, list, pid)) return rc;     // the whole list: no pixel is rendered by two members
    const size_t N = g.members.size();
    std::vector<uint32_t> order; shard_order(list.data(), uint32_t(list.size()), order);
    g.shares.assign(N, {});
    for (uint32_t i = 0; i < list.size(); ++i) g.shares[i % N].push_back(list[order[i]]);
    CU(cudaSetDevice(root->device));
    g.root_pix.resize(N); g.share_pixels.assign(N, 0);
    size_t max_share = 0;
    for (size_t k = 0; k < N; ++k) {
        if (int rc = tile_pixels(root, g.shares[k], pid)) return rc;
        g.share_pixels[k] = uint32_t(pid.size());
        max_share = std::max(max_share, pid.size());
        if (k >= 1) {
            CU(g.root_pix[k].upload(pid.data(), pid.size(), root->stream));
            CU(cudaStreamSynchronize(root->stream));
        }
    }
    CU(g.recv.ensure(max_share));
    for (size_t k = 1; k < N; ++k) {
        tgb_ctx *m = g.members[k];
        if (cudaSetDevice(m->device) != cudaSuccess) return fail(c, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", m->device);
        CU(m->send.ensure(g.share_pixels[k]));
    }
    g.deal_key = std::move(list);
    return TGB_OK;
}

// Every member renders its share concurrently (one host thread per GPU), then the shares travel to the root over NVLink.
int group_render(tgb_ctx *root, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count, tgb_sample_record *records) {
    tgb_ctx *c = root; Group &g = *root->group;
    int rc = group_deal(root, tiles, n_tiles, seed);
    if (rc) return rc;
    const size_t N = g.members.size();
    const uint32_t var_w = (root->res_x + 3)/4, var_h = (root->res_y + 3)/4; const size_t n_blocks = size_t(var_w)*var_h;
    std::vector<int> rcs(N, TGB_OK);
    std::vector<std::vector<tgb_sample_record>> recs(records ? N : 0);
    std::vector<std::thread> th;
    for (size_t k = 0; k < N; ++k) {
        if (records) recs[k].assign(records, records + n_blocks);
        th.emplace_back([&, k] {
            tgb_ctx *m = g.members[k];
            if (g.shares[k].empty()) return;
            rcs[k] = records ? single_render_adaptive(m, g.shares[k].data(), uint32_t(g.shares[k].size()), seed, recs[k].data())
                             : single_render_resident(m, g.shares[k].data(), uint32_t(g.shares[k].size()), seed, spp_begin, spp_count);
        });
    }
    for (std::thread &t : th) t.join();
    for (size_t k = 0; k < N; ++k) if (rcs[k]) { root->error = "device " + std::to_string(g.members[k]->device) + ": " + g.members[k]->error; return rcs[k]; }
    if (records) {          // a 4x4 block lies inside one 16x16 tile: its record comes back from the member that owns the tile
        for (size_t k = 0; k < N; ++k)
            for (const tgb_tile &tl : g.shares[k])
                for (uint32_t by = tl.y/4; by < (tl.y + tl.h + 3)/4; ++by)
                    for (uint32_t bx = tl.x/4; bx < (tl.x + tl.w + 3)/4; ++bx)
                        records[bx + size_t(by)*var_w] = recs[k][bx + size_t(by)*var_w];
    }
    // gather: pack on the member, one peer copy, de-tile on the root
    CU(cudaSetDevice(root->device));
    CU(cudaEventRecord(g.ev_gather[0], root->stream));
    for (size_t k = 1; k < N; ++k) {
        tgb_ctx *m = g.members[k];
        const uint32_t np = g.share_pixels[k];
        if (!np) continue;
        if (cudaSetDevice(m->device) != cudaSuccess) return fail(c, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", m->device);
        k_pack_share<<<blocks(np, 256), 256, 0, m->stream>>>(m->pix_id.p, np, m->fb, m->fb_count, m->send.p);
        m->stats.kernel_launches++;
        cudaError_t e = cudaStreamSynchronize(m->stream);
        if (e != cudaSuccess) return fail(c, TGB_ERR_CUDA, "pack on device %d failed: %s", m->device, cudaGetErrorString(e));
        CU(cudaSetDevice(root->device));
        CU(cudaMemcpyPeerAsync(g.recv.p, root->device, m->send.p, m->device, size_t(np)*sizeof(float4), root->stream));
        k_unpack_share<<<blocks(np, 256), 256, 0, root->stream>>>(g.root_pix[k].p, np, g.recv.p, root->fb, root->fb_count);
        root->stats.kernel_launches++;
    }
    CU(cudaSetDevice(root->device));
    CU(cudaEventRecord(g.ev_gather[1], root->stream));
    CU(cudaStreamSynchronize(root->stream));
    float ms = 0.0f; cudaEventElapsedTime(&ms, g.ev_gather[0], g.ev_gather[1]); g.gather_ms += ms;
    CU(cudaGetLastError());
    return TGB_OK;
}

// The settings a scene is refused for before it is prepared
int check_settings(const tgb_scene_desc *d) {
    if (d->abi_version != TGB200_ABI_VERSION) return fail(nullptr, TGB_ERR_INVALID, "ABI version mismatch (got %u, library is %u)", d->abi_version, TGB200_ABI_VERSION);
    if (!d->settings.use_sobol) return fail(nullptr, TGB_ERR_UNSUPPORTED, "only the Sobol sampler (renderer.stratified_sampler = true) is on the hot path");
    if (d->settings.supplemental_mode != 0) return fail(nullptr, TGB_ERR_UNSUPPORTED, "supplemental_mode %u: the per-tile serial PCG stream cannot be reproduced by a wavefront renderer (DESIGN.md section 3)", d->settings.supplemental_mode);
    if (d->camera.res_x == 0 || d->camera.res_y == 0) return fail(nullptr, TGB_ERR_INVALID, "empty image");
    // max_bounces 0: PathTracer::traceSample's loop never runs and every sample is black; the wavefront's first shade would add
    // bounce-0 emission, so the setting is refused rather than rendered differently
    if (d->settings.max_bounces > 255 || d->settings.max_bounces < 1) return fail(nullptr, TGB_ERR_UNSUPPORTED, "max_bounces must be in [1, 255]");
    return TGB_OK;
}

// A context for a prepared scene on device dev (< 0: the current device)
int create_single(const HostScene &hs, int dev, tgb_ctx **out) {
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(nullptr, TGB_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU fallback)"); }
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    if (dev >= ndev) return fail(nullptr, TGB_ERR_NO_DEVICE, "CUDA device %d not present (%d devices)", dev, ndev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return fail(nullptr, TGB_ERR_NO_DEVICE, "cannot query device %d", dev);
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, TGB_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major, prop.minor);
    if (cudaSetDevice(dev) != cudaSuccess) return fail(nullptr, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", dev);
    tgb_ctx *c = new tgb_ctx(dev);
    int rc = TGB_OK;
    do {
        if (c->created != cudaSuccess) { rc = fail(c, TGB_ERR_CUDA, "stream or event creation failed: %s", cudaGetErrorString(c->created)); break; }
        c->ks = select_kernels(hs.kind);
        if ((rc = upload_scene(c, hs, c->ks))) break;
        // default: 2 x 4 Mi paths in flight (H100, C1: 2 x 2 Mi measured 3 % slower)
        const uint32_t max_paths = hs.sc.set.max_paths_in_flight;
        uint32_t cap = max_paths ? max_paths : (1u << 23);
        cap = std::max(cap, 1024u);
        if ((rc = alloc_wavefront(c, cap))) break;
        {   // persistent traversal grid of one wavefront: what is resident at once (blocks per SM x SMs, smaller of the two
            // kernels), or TGB_TRAVERSAL_BLOCKS per SM.  H100, C1: 6 (resident) > 4 > 12 (twice resident) > 3 blocks per SM.
            int sms = 0, b1 = 0, b2 = 0;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b1, c->ks.trace, kTraceBlock, 0);
            if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b2, c->ks.shadow_bvh, kTraceBlock, 0);
            if (e != cudaSuccess || sms <= 0 || b1 <= 0 || b2 <= 0) { rc = fail(c, TGB_ERR_CUDA, "traversal kernels cannot be resident (%s)", cudaGetErrorString(e)); break; }
            const char *per_sm = getenv("TGB_TRAVERSAL_BLOCKS");
            c->persist_blocks = uint32_t(sms)*uint32_t(per_sm ? std::max(1, atoi(per_sm)) : std::min(b1, b2));
            // k_regen, k_shadow_prep and k_bin_scatter loop over the device-side counts: a grid of what is resident at once
            // instead of one sized for the worst case, whose blocks past the real count would only read ctl and exit
            int br = 0, bp = 0, bs = 0;
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&br, k_regen, 256, 0);
            if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bp, c->ks.shadow_prep, 256, 0);
            if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bs, k_bin_scatter, 256, 0);
            if (e != cudaSuccess || br <= 0 || bp <= 0 || bs <= 0) { rc = fail(c, TGB_ERR_CUDA, "loop kernels cannot be resident (%s)", cudaGetErrorString(e)); break; }
            c->regen_blocks = uint32_t(sms)*uint32_t(br); c->prep_blocks = uint32_t(sms)*uint32_t(bp); c->scatter_blocks = uint32_t(sms)*uint32_t(bs);
            // TGB_LOOP_BLOCKS: at most that many blocks in the whole grid (not per SM), so that a test knows each trip's size
            if (const char *lb = getenv("TGB_LOOP_BLOCKS")) {
                const int v = atoi(lb);
                if (v >= 1) for (uint32_t *g : {&c->regen_blocks, &c->prep_blocks, &c->scatter_blocks}) *g = std::min(*g, uint32_t(v));
            }
        }
    } while (0);
    if (rc) { g_create_error = c->error; tgb200_destroy(c); return rc; }
    *out = c;
    return TGB_OK;
}

// Closest hits of n device rays through the analytic pass and the renderer's traversal kernels (into device Hit records)
// As in a render, rays that miss the BVH's top-level cut before their analytic hit skip the traversal (TGB_HOOK_CUT=0: every ray
// is traversed).  list: the traversal list, [count | indices of the rays to traverse], which the caller keeps until its stream
// has run the kernels.
cudaError_t hook_closest(tgb_ctx *c, const tgb_ray *dr, Hit *dx, uint32_t n, Buffer<uint32_t> &list) {
    const char *cut_env = getenv("TGB_HOOK_CUT");
    const int cut = (cut_env && cut_env[0] == '0') ? 0 : 1;
    cudaError_t e = list.ensure(size_t(n) + 1);
    if (e == cudaSuccess) e = cudaMemsetAsync(list.p, 0, sizeof(uint32_t), c->stream);
    if (e == cudaSuccess) {
        k_hook_analytic<<<blocks(n, 256), 256, 0, c->stream>>>(c->sc, dr, dx, n, cut, list.p + 1, list.p);
        c->stats.kernel_launches++;
    }
    if (e == cudaSuccess && c->sc.n_nodes) {
        // the renderer's own persistent kernel body (lane refill)
        uint32_t *cursor = &c->wf[0].ctl->cursor_trace;
        e = cudaMemsetAsync(cursor, 0, sizeof(uint32_t), c->stream);
        uint32_t grid = std::min(blocks(n, kTraceBlock), c->persist_blocks);
        if (e == cudaSuccess) c->ks.hook_persist<<<grid, kTraceBlock, 0, c->stream>>>(c->sc, dr, dx, list.p + 1, list.p, n, cursor);
        c->stats.kernel_launches++;
    }
    return e;
}

// The pixel list of tgb200_pack_tiles / tgb200_unpack_tiles on the device: the last render's when the tile list is the same,
// else a copy in `own`
int device_tile_pixels(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, Buffer<uint32_t> &own, const uint32_t **dev, uint32_t *n_out) {
    const std::vector<tgb_tile> list(tiles, tiles + n_tiles);
    if (same_tiles(list, c->tiles_cached)) { *dev = c->pix_id.p; *n_out = c->n_pix; return TGB_OK; }
    std::vector<uint32_t> pid;
    if (int rc = tile_pixels(c, list, pid)) return rc;
    CU(own.upload(pid.data(), pid.size(), c->stream));
    CU(cudaStreamSynchronize(c->stream));
    *dev = own.p; *n_out = uint32_t(pid.size());
    return TGB_OK;
}

// UniformSampler (sampling/UniformSampler.hpp:40-52): the integrator's own PCG32 stream (tile seeds, adaptive distribution)
inline float pcg_next1d(uint64_t &state) { return normalized_uint(pcg_next(state)); }
// Tungsten's min / max (math/MathUtil.hpp:10-26): a < b ? a : b and a > b ? a : b.  They agree with std::min / std::max on
// numbers but not on NaN: a block whose mean overflowed to Inf has a NaN error estimate, and min(NaN, maxError) = maxError
// gives it the largest weight, where std::min would carry the NaN into the dilation and the sample budget.
inline float tungsten_min(float a, float b) { return a < b ? a : b; }
inline float tungsten_max(float a, float b) { return a > b ? a : b; }

// The tree tgb200_create builds for a scene of n triangles (9 floats each: v0 v1 v2) and nothing else.  extent = the largest
// coordinate magnitude in play besides the triangles' (tgb200_create: the camera position's).
void build_triangle_scene_bvh(const float *tri_verts, uint32_t n, float extent, SceneBvh &sb) {
    std::vector<BuildTri> tris(n);
    for (uint32_t i = 0; i < n; ++i) std::memcpy(&tris[i], tri_verts + 9*size_t(i), sizeof(BuildTri));
    SceneBvhInput in;
    in.tris = tris.data(); in.n_tris = n; in.extent = extent;
    build_scene_bvh(in, bvh_options(), sb);
}
// 1/d as the kernels compute it: components no larger than 1e-30 in magnitude are replaced by +-1e-30
void host_inv_dir(const V3 &d, float inv[3]) {
    const float ooeps = 1e-30f;
    inv[0] = 1.0f/(std::fabs(d.x) > ooeps ? d.x : std::copysign(ooeps, d.x));
    inv[1] = 1.0f/(std::fabs(d.y) > ooeps ? d.y : std::copysign(ooeps, d.y));
    inv[2] = 1.0f/(std::fabs(d.z) > ooeps ? d.z : std::copysign(ooeps, d.z));
}
// Traversal::triangle on the host, on the intersection record the kernels read: best = t when the triangle is hit in (tnear, best)
bool host_triangle(const IsectRecord &rec, const V3 &o, const V3 &d, float tnear, float &best) {
    const V3 v0 = f3(rec.f), e1 = f3(rec.f + 3), e2 = f3(rec.f + 6), ng = f3(rec.f + 9);
    V3 C = v0 - o, R = cross(d, C);
    auto edot = [](V3 a, V3 b) { return a.x*b.x + (a.y*b.y + a.z*b.z); };
    float den = edot(ng, d), absDen = std::fabs(den);
    auto xs = [&](float a) { return den < 0.0f || (den == 0.0f && std::signbit(den)) ? -a : a; };
    float U = xs(edot(R, e2)), V = xs(edot(R, e1));
    if (!(den != 0.0f && U >= 0.0f && V >= 0.0f && U + V <= absDen)) return false;
    float T = xs(edot(ng, C));
    if (!(T > absDen*tnear && T < absDen*best)) return false;
    best = T/absDen;
    return true;
}

// ---- test hooks: host arrays in, one probe kernel on the context's stream, host arrays out ----
// A probe's end: the restore of the state it saved, then the synchronise after which its arrays (Buffers declared in the probe)
// may be freed
struct ProbeBufs {
    tgb_ctx *c;
    Buffer<Ctl> ctl_saved; Buffer<Counters> ctr_saved; bool saved = false;
    explicit ProbeBufs(tgb_ctx *ctx) : c(ctx) {}
    // Snapshot of wavefront 0's control block and the context's counters, which a probe that runs the renderer's kernels uses:
    // its launches must not show in them or in the next render's statistics.  finish() queues the restore.
    cudaError_t save_state() {
        cudaError_t e = ctl_saved.ensure(1);
        if (e == cudaSuccess) e = ctr_saved.ensure(1);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctl_saved.p, c->wf[0].ctl, sizeof(Ctl), cudaMemcpyDeviceToDevice, c->stream);
        if (e == cudaSuccess) e = cudaMemcpyAsync(ctr_saved.p, c->ctr, sizeof(Counters), cudaMemcpyDeviceToDevice, c->stream);
        saved = e == cudaSuccess;
        return e;
    }
    int finish(cudaError_t e, const char *what) {
        if (saved) {        // also when a launch failed: the copies are queued after whatever was queued
            const cudaError_t r1 = cudaMemcpyAsync(c->wf[0].ctl, ctl_saved.p, sizeof(Ctl), cudaMemcpyDeviceToDevice, c->stream);
            const cudaError_t r2 = cudaMemcpyAsync(c->ctr, ctr_saved.p, sizeof(Counters), cudaMemcpyDeviceToDevice, c->stream);
            if (e == cudaSuccess) e = r1 != cudaSuccess ? r1 : r2;
        }
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        return e == cudaSuccess ? TGB_OK : fail(c, TGB_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
    }
};
template <typename T> cudaError_t download(tgb_ctx *c, T *dst, const T *src, size_t n) {
    return cudaMemcpyAsync(dst, src, n*sizeof(T), cudaMemcpyDeviceToHost, c->stream);
}
// lobe_set 1 (the Lambert-only instantiation) exists only without curves, as in k_shade
int probe_check(tgb_ctx *c, int lobe_set) {
    if (lobe_set != 0 && lobe_set != 1) return fail(c, TGB_ERR_INVALID, "lobe_set must be 0 or 1");
    if (lobe_set == 1 && c->has_curves) return fail(c, TGB_ERR_INVALID, "lobe_set 1 has no instantiation with curves");
    return TGB_OK;
}
}  // namespace

extern "C" {

uint32_t tgb200_abi_version(void) { return TGB200_ABI_VERSION; }

const char *tgb200_last_error(const tgb_ctx *ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

void tgb200_destroy(tgb_ctx *c) {
    if (!c) return;
    if (c->group) for (size_t k = 1; k < c->group->members.size(); ++k) tgb200_destroy(c->group->members[k]);
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->stream1) cudaStreamSynchronize(c->stream1);
    delete c;               // with its group, which lives on this device
}

int tgb200_create(const tgb_scene_desc *d, tgb_ctx **out) {
    if (!d || !out) return fail(nullptr, TGB_ERR_INVALID, "null argument");
    *out = nullptr;
    const uint32_t N = d->settings.n_devices;
    if (N > 8) return fail(nullptr, TGB_ERR_INVALID, "at most 8 devices");
    for (uint32_t i = 0; i < N; ++i) for (uint32_t j = 0; j < i; ++j)
        if (d->settings.devices[i] == d->settings.devices[j]) return fail(nullptr, TGB_ERR_INVALID, "device %d listed twice", d->settings.devices[i]);
    // the scene is checked and prepared once, before any device is touched
    if (int rc = check_settings(d)) return rc;
    HostScene hs;
    if (int rc = prepare_scene(d, hs)) return rc;
    if (N <= 1) return create_single(hs, N == 1 ? d->settings.devices[0] : d->settings.device, out);
    // one context per GPU, created concurrently, each uploading the same prepared scene
    std::vector<tgb_ctx *> members(N, nullptr); std::vector<int> rcs(N, TGB_OK); std::vector<std::string> errs(N);
    std::vector<std::thread> th;
    for (uint32_t k = 0; k < N; ++k) th.emplace_back([&, k] {
        rcs[k] = create_single(hs, d->settings.devices[k], &members[k]);
        if (rcs[k]) errs[k] = g_create_error;
    });
    for (std::thread &t : th) t.join();
    for (uint32_t k = 0; k < N; ++k) if (rcs[k]) {
        for (tgb_ctx *m : members) if (m) tgb200_destroy(m);
        return fail(nullptr, rcs[k], "device %d: %s", d->settings.devices[k], errs[k].c_str());
    }
    tgb_ctx *root = members[0];
    for (uint32_t k = 1; k < N; ++k) {             // NVLink peer access root <-> member (without it the copies stage through the host)
        int can = 0;
        cudaDeviceCanAccessPeer(&can, root->device, members[k]->device);
        if (can) { cudaSetDevice(root->device); cudaDeviceEnablePeerAccess(members[k]->device, 0); cudaSetDevice(members[k]->device); cudaDeviceEnablePeerAccess(root->device, 0); }
        cudaGetLastError();
    }
    cudaSetDevice(root->device);
    root->group = std::make_unique<Group>(members);
    if (const cudaError_t e = root->group->created; e != cudaSuccess) {
        tgb200_destroy(root);
        return fail(nullptr, TGB_ERR_CUDA, "cudaEventCreate failed: %s", cudaGetErrorString(e));
    }
    *out = root;
    return TGB_OK;
}

int tgb200_clear_framebuffer(tgb_ctx *c) {
    if (!c) return TGB_ERR_INVALID;
    { int rc = for_members(c, [](tgb_ctx *m) { return tgb200_clear_framebuffer(m); }); if (rc) return rc; }
    CU(cudaSetDevice(c->device));
    size_t npx = size_t(c->res_x)*c->res_y;
    CU(cudaMemsetAsync(c->fb, 0, npx*3*sizeof(float), c->stream));
    CU(cudaMemsetAsync(c->fb_count, 0, npx*sizeof(uint32_t), c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return TGB_OK;
}

int tgb200_render_resident(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count) {
    if (!c) return TGB_ERR_INVALID;
    if (n_tiles && !tiles) return fail(c, TGB_ERR_INVALID, "null tile list");
    if (c->group) return group_render(c, tiles, n_tiles, seed, spp_begin, spp_count, nullptr);
    return single_render_resident(c, tiles, n_tiles, seed, spp_begin, spp_count);
}

int tgb200_read_framebuffer(tgb_ctx *c, float *rgb_mean, uint32_t *count) {
    if (!c || !rgb_mean) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    size_t npx = size_t(c->res_x)*c->res_y;
    CU(cudaMemcpyAsync(c->h_fb.p, c->fb, npx*3*sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    if (count) CU(cudaMemcpyAsync(c->h_fb_count.p, c->fb_count, npx*sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    std::memcpy(rgb_mean, c->h_fb.p, npx*3*sizeof(float));
    if (count) std::memcpy(count, c->h_fb_count.p, npx*sizeof(uint32_t));
    return TGB_OK;
}

int tgb200_render_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count,
                        float *rgb_mean, uint32_t *count) {
    if (!c || !rgb_mean) return c ? fail(c, TGB_ERR_INVALID, "null framebuffer") : TGB_ERR_INVALID;
    if (n_tiles && !tiles) return fail(c, TGB_ERR_INVALID, "null tile list");
    // the caller's running mean and counts are the input state (of every member of a multi-GPU context, for its own pixels);
    // without counts the running mean restarts from the sample index range's start
    std::vector<uint32_t> base;
    if (!count) base.assign(size_t(c->res_x)*c->res_y, spp_begin);
    int rc = tgb200_write_framebuffer(c, rgb_mean, count ? count : base.data());
    if (rc) return rc;
    if ((rc = tgb200_render_resident(c, tiles, n_tiles, seed, spp_begin, spp_count))) return rc;
    return tgb200_read_framebuffer(c, rgb_mean, count);
}

int tgb200_framebuffer_device_ptr(tgb_ctx *c, void **rgb_mean_dev, uint64_t *n_bytes) {
    if (!c || !rgb_mean_dev) return TGB_ERR_INVALID;
    *rgb_mean_dev = c->fb;
    if (n_bytes) *n_bytes = uint64_t(c->res_x)*c->res_y*3*sizeof(float);
    return TGB_OK;
}

int tgb200_trace_closest(tgb_ctx *c, const tgb_ray *rays, tgb_hit *hits, uint32_t n) {
    if (!c || (n && (!rays || !hits))) return TGB_ERR_INVALID;
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    Buffer<tgb_ray> dr; Buffer<tgb_hit> dh; Buffer<Hit> dx; Buffer<uint32_t> list;
    CU(dr.ensure(n)); CU(dh.ensure(n)); CU(dx.ensure(n));
    cudaError_t e = cudaMemcpyAsync(dr.p, rays, size_t(n)*sizeof(tgb_ray), cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = hook_closest(c, dr.p, dx.p, n, list);
    if (e == cudaSuccess) {
        k_hook_finish<<<blocks(n, 256), 256, 0, c->stream>>>(c->sc, dr.p, dx.p, dh.p, n);
        c->stats.kernel_launches++;
        e = cudaMemcpyAsync(hits, dh.p, size_t(n)*sizeof(tgb_hit), cudaMemcpyDeviceToHost, c->stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e == cudaSuccess) e = cudaGetLastError();
    return e == cudaSuccess ? TGB_OK : fail(c, TGB_ERR_CUDA, "trace_closest failed: %s", cudaGetErrorString(e));
}

int tgb200_get_stats(tgb_ctx *c, tgb_stats *out) {
    if (!c || !out) return TGB_ERR_INVALID;
    *out = c->stats;
    if (c->group) {         // counts add up over the GPUs, times are those of the slowest GPU
        for (size_t k = 1; k < c->group->members.size(); ++k) {
            const tgb_stats &m = c->group->members[k]->stats;
            out->samples += m.samples; out->rays += m.rays; out->hits += m.hits; out->kernel_launches += m.kernel_launches;
            out->path_rays += m.path_rays; out->shadow_rays += m.shadow_rays; out->trace_launches += m.trace_launches;
            out->shadow_launches += m.shadow_launches; out->path_rays_traversed += m.path_rays_traversed;
            out->shadow_rays_traversed += m.shadow_rays_traversed; out->iterations += m.iterations;
            out->trace_ms = std::max(out->trace_ms, m.trace_ms); out->total_ms = std::max(out->total_ms, m.total_ms);
            out->shadow_ms = std::max(out->shadow_ms, m.shadow_ms); out->regen_ms = std::max(out->regen_ms, m.regen_ms);
            out->shade_ms = std::max(out->shade_ms, m.shade_ms); out->prep_ms = std::max(out->prep_ms, m.prep_ms);
            out->accum_ms = std::max(out->accum_ms, m.accum_ms); out->sort_ms = std::max(out->sort_ms, m.sort_ms);
        }
        out->sort_ms += c->group->gather_ms;            // (the gather is accounted with the loop's bookkeeping time)
    }
    return TGB_OK;
}

int tgb200_reset_stats(tgb_ctx *c) {
    if (!c) return TGB_ERR_INVALID;
    { int rc = for_members(c, [](tgb_ctx *m) { return tgb200_reset_stats(m); }); if (rc) return rc; if (c->group) c->group->gather_ms = 0.0; }
    CU(cudaSetDevice(c->device));
    c->stats = tgb_stats{};
    CU(cudaMemsetAsync(c->ctr, 0, sizeof(Counters), c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return TGB_OK;
}

int tgb200_set_stream(tgb_ctx *c, void *cuda_stream) {
    if (!c) return TGB_ERR_INVALID;
    if (c->group && cuda_stream) return fail(c, TGB_ERR_UNSUPPORTED, "a multi-GPU context runs every GPU on its own stream");
    CU(cudaSetDevice(c->device));
    CU(cudaStreamSynchronize(c->stream));
    c->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : c->own_stream;
    return TGB_OK;
}

int tgb200_set_profiling(tgb_ctx *c, int enable) {
    if (!c) return TGB_ERR_INVALID;
    for_members(c, [enable](tgb_ctx *m) { return tgb200_set_profiling(m, enable); });
    c->profiling = enable != 0;
    return TGB_OK;
}

int tgb200_scene_info(tgb_ctx *c, uint32_t *n_tris, uint32_t *n_nodes, uint32_t *bvh_depth, uint64_t *geom_bytes, uint32_t *capacity) {
    if (!c) return TGB_ERR_INVALID;
    if (n_tris) *n_tris = c->n_tris;
    if (n_nodes) *n_nodes = c->sc.n_nodes;
    if (bvh_depth) *bvh_depth = c->bvh_depth;
    if (geom_bytes) *geom_bytes = c->geom_bytes;
    if (capacity) *capacity = c->capacity;
    return TGB_OK;
}

int tgb200_pack_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, void *rgb_out_dev) {
    if (!c || !tiles || !rgb_out_dev) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    Buffer<uint32_t> own; const uint32_t *pid = nullptr; uint32_t n = 0;
    int rc = device_tile_pixels(c, tiles, n_tiles, own, &pid, &n);
    if (rc || !n) return rc;
    k_pack_tiles<<<blocks(n, 256), 256, 0, c->stream>>>(pid, n, c->fb, static_cast<float *>(rgb_out_dev));
    c->stats.kernel_launches++;
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return fail(c, TGB_ERR_CUDA, "pack_tiles failed: %s", cudaGetErrorString(e));
    return TGB_OK;
}

int tgb200_unpack_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, const void *rgb_in_dev, uint32_t sample_count) {
    if (!c || !tiles || !rgb_in_dev) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    Buffer<uint32_t> own; const uint32_t *pid = nullptr; uint32_t n = 0;
    int rc = device_tile_pixels(c, tiles, n_tiles, own, &pid, &n);
    if (rc || !n) return rc;
    k_unpack_tiles<<<blocks(n, 256), 256, 0, c->stream>>>(pid, n, static_cast<const float *>(rgb_in_dev), c->fb, c->fb_count, sample_count);
    c->stats.kernel_launches++;
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) return fail(c, TGB_ERR_CUDA, "unpack_tiles failed: %s", cudaGetErrorString(e));
    return TGB_OK;
}

// Host-only: the hair BCSDF tables tgb200_create would upload for one material (no GPU needed).
// tables = 3 lobes (R, TT, TRT) x 64 x 64 x RGB, sums = 3 x 64 row sums, v = the three longitudinal variances.
int tgb200_hair_selftest(float roughness, float scale_angle_deg, const float *sigma_a, float *tables, float *sums, float *v) {
    if (!sigma_a || !tables || !sums || !v) return TGB_ERR_INVALID;
    HairTables ht;
    hair_precompute(roughness, scale_angle_deg, sigma_a, ht);
    for (int p = 0; p < 3; ++p) {
        std::memcpy(tables + size_t(p)*64*64*3, ht.lobe[p].table.data(), sizeof(float)*64*64*3);
        std::memcpy(sums + p*64, ht.lobe[p].sums.data(), sizeof(float)*64);
        v[p] = ht.v[p];
    }
    return TGB_OK;
}

// Host-only self-check of the BVH builder (no GPU needed): builds the 4-ary BVH over n triangles (9 floats each) and
// verifies that every triangle is referenced by exactly one leaf and lies inside every box on its root-to-leaf chain.
int tgb200_bvh_selftest(const float *tri_verts, uint32_t n, uint32_t *n_nodes, uint32_t *depth, uint32_t *max_leaf) {
    if (n && !tri_verts) return TGB_ERR_INVALID;
    std::vector<BuildTri> tris(n);
    for (uint32_t i = 0; i < n; ++i) std::memcpy(&tris[i], tri_verts + 9*size_t(i), sizeof(BuildTri));
    Bvh4 bvh;
    build_bvh4(tris.data(), n, bvh, 0, 0.0f);
    if (n_nodes) *n_nodes = uint32_t(bvh.nodes.size());
    if (depth) *depth = bvh.max_depth;
    if (n == 0) return bvh.nodes.empty() ? TGB_OK : TGB_ERR_INVALID;
    if (bvh.order.size() != n) return TGB_ERR_INVALID;
    std::vector<uint32_t> seen(n, 0);
    uint32_t worst_leaf = 0;
    struct It { int32_t node; float lo[3], hi[3]; };
    std::vector<It> stack;
    It root; root.node = 0;
    for (int a = 0; a < 3; ++a) { root.lo[a] = bvh.lo[a]; root.hi[a] = bvh.hi[a]; }
    stack.push_back(root);
    while (!stack.empty()) {
        It it = stack.back(); stack.pop_back();
        if (it.node < 0 || size_t(it.node) >= bvh.nodes.size()) return TGB_ERR_INVALID;
        const Node4 &nd = bvh.nodes[size_t(it.node)];
        for (int k = 0; k < 4; ++k) {
            if (nd.link[k] == kEmptyLink) continue;
            It ch; ch.node = nd.link[k];
            ch.lo[0] = nd.f[k]; ch.hi[0] = nd.f[4 + k]; ch.lo[1] = nd.f[8 + k]; ch.hi[1] = nd.f[12 + k]; ch.lo[2] = nd.f[16 + k]; ch.hi[2] = nd.f[20 + k];
            for (int a = 0; a < 3; ++a) if (ch.lo[a] < it.lo[a] || ch.hi[a] > it.hi[a]) return TGB_ERR_INVALID;   // child box inside parent box
            if (nd.link[k] >= 0) { stack.push_back(ch); continue; }
            int code = ~nd.link[k]; uint32_t first = uint32_t(code >> 3), count = uint32_t(code & 7) + 1;
            worst_leaf = std::max(worst_leaf, count);
            for (uint32_t i = 0; i < count; ++i) {
                if (first + i >= n) return TGB_ERR_INVALID;
                uint32_t t = bvh.order[first + i];
                if (t >= n) return TGB_ERR_INVALID;
                seen[t]++;
                const float *v[3] = {tris[t].v0, tris[t].v1, tris[t].v2};
                for (int q = 0; q < 3; ++q) for (int a = 0; a < 3; ++a)
                    if (v[q][a] < ch.lo[a] || v[q][a] > ch.hi[a]) return TGB_ERR_INVALID;                          // triangle inside its leaf box
            }
        }
    }
    for (uint32_t i = 0; i < n; ++i) if (seen[i] != 1) return TGB_ERR_INVALID;
    if (max_leaf) *max_leaf = worst_leaf;
    return TGB_OK;
}

int tgb200_write_framebuffer(tgb_ctx *c, const float *rgb_mean, const uint32_t *count) {
    if (!c || !rgb_mean || !count) return TGB_ERR_INVALID;
    { int rc = for_members(c, [=](tgb_ctx *m) { return tgb200_write_framebuffer(m, rgb_mean, count); }); if (rc) return rc; }
    CU(cudaSetDevice(c->device));
    size_t npx = size_t(c->res_x)*c->res_y;
    std::memcpy(c->h_fb.p, rgb_mean, npx*3*sizeof(float)); std::memcpy(c->h_fb_count.p, count, npx*sizeof(uint32_t));
    CU(cudaMemcpyAsync(c->fb, c->h_fb.p, npx*3*sizeof(float), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->fb_count, c->h_fb_count.p, npx*sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    return TGB_OK;
}

// One adaptive step (PathTraceIntegrator::renderTile with per-block sample counts, PathTraceIntegrator.cpp:136-156): every pixel
// of 4x4 block b renders records[b].next_sample_count samples starting at sample index records[b].sample_index; the resident
// framebuffer takes them in sample order and the records' Welford statistics are updated in the reference's order.
int tgb200_render_adaptive(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, tgb_sample_record *records) {
    if (!c || !records) return c ? fail(c, TGB_ERR_INVALID, "null records") : TGB_ERR_INVALID;
    if (n_tiles && !tiles) return fail(c, TGB_ERR_INVALID, "null tile list");
    if (c->group) return group_render(c, tiles, n_tiles, seed, 0, 0, records);
    return single_render_adaptive(c, tiles, n_tiles, seed, records);
}

int tgb200_shard_tiles(const tgb_tile *tiles, uint32_t n_tiles, uint32_t *order) {
    if ((n_tiles && !tiles) || !order) return TGB_ERR_INVALID;
    std::vector<uint32_t> o; shard_order(tiles, n_tiles, o);
    std::memcpy(order, o.data(), size_t(n_tiles)*4);
    return TGB_OK;
}

// PathTraceIntegrator::generateWork (PathTraceIntegrator.cpp:44-134), host only: advances every block's sample index, then
// either gives every block spp_count samples or -- adaptive sampling on and current_spp >= 16 -- distributes the step's
// budget by the blocks' clamped, dilated error estimates.  sampler_state = the integrator's UniformSampler state (it already
// produced the tile seeds); returns 1 when there is work, 0 when the error estimate is zero everywhere (the reference
// then skips the step), negative on bad arguments.
int tgb200_generate_work(tgb_sample_record *records, uint32_t res_x, uint32_t res_y, uint32_t current_spp, uint32_t next_spp,
                         int adaptive_sampling, uint64_t *sampler_state) {
    if (!records || !sampler_state || !res_x || !res_y || next_spp < current_spp) return TGB_ERR_INVALID;
    const uint32_t var_w = (res_x + 3)/4, var_h = (res_y + 3)/4; const size_t n = size_t(var_w)*var_h;
    for (size_t i = 0; i < n; ++i) records[i].sample_index += records[i].next_sample_count;
    const int spp_count = int(next_spp - current_spp);
    if (adaptive_sampling && current_spp >= 16) {                                        // AdaptiveThreshold (PathTraceIntegrator.hpp)
        // errorPercentile95 (:44-59)
        std::vector<float> errors; errors.reserve(n);
        for (size_t i = 0; i < n; ++i) {
            tgb_sample_record &r = records[i];
            float variance = r.running_variance/float(r.sample_count - 1u);              // SampleRecord::variance (uint32 arithmetic, then float)
            r.adaptive_weight = variance/(float(r.sample_count)*tungsten_max(r.mean*r.mean, 1e-3f));
            if (r.adaptive_weight > 0.0f) errors.push_back(r.adaptive_weight);
        }
        if (errors.empty()) return 0;
        std::sort(errors.begin(), errors.end());
        const float max_error = errors[(errors.size()*95)/100];
        if (max_error == 0.0f) return 0;
        for (size_t i = 0; i < n; ++i) records[i].adaptive_weight = tungsten_min(records[i].adaptive_weight, max_error);
        // dilateAdaptiveWeights (:61-88)
        for (uint32_t y = 0; y < var_h; ++y) for (uint32_t x = 0; x < var_w; ++x) {
            size_t idx = x + size_t(y)*var_w;
            if (y < var_h - 1) records[idx].adaptive_weight = tungsten_max(records[idx].adaptive_weight, records[idx + var_w].adaptive_weight);
            if (x < var_w - 1) records[idx].adaptive_weight = tungsten_max(records[idx].adaptive_weight, records[idx + 1].adaptive_weight);
        }
        for (int y = int(var_h) - 1; y >= 0; --y) for (int x = int(var_w) - 1; x >= 0; --x) {
            size_t idx = size_t(x) + size_t(y)*var_w;
            if (y > 0) records[idx].adaptive_weight = tungsten_max(records[idx].adaptive_weight, records[idx - var_w].adaptive_weight);
            if (x > 0) records[idx].adaptive_weight = tungsten_max(records[idx].adaptive_weight, records[idx - 1].adaptive_weight);
        }
        // distributeAdaptiveSamples (:90-112)
        double total_weight = 0.0;
        for (size_t i = 0; i < n; ++i) total_weight += records[i].adaptive_weight;
        const int adaptive_budget = (spp_count - 1)*int(res_x)*int(res_y);
        const int budget_per_tile = adaptive_budget/16;
        const float weight_to_sample = float(double(budget_per_tile)/total_weight);
        float pixel_pdf = 0.0f;
        for (size_t i = 0; i < n; ++i) {
            float fractional = records[i].adaptive_weight*weight_to_sample;
            int adaptive = int(fractional);
            pixel_pdf += fractional - float(adaptive);
            if (pcg_next1d(*sampler_state) < pixel_pdf) { adaptive++; pixel_pdf -= 1.0f; }
            records[i].next_sample_count = uint32_t(adaptive + 1);
        }
    } else {
        for (size_t i = 0; i < n; ++i) records[i].next_sample_count = uint32_t(spp_count);
    }
    return 1;
}

// Host-only check of the quantised device BVH (no GPU needed): builds the tree tgb200_create builds for a scene of n triangles
// (the rays' origins take the camera's part in the padding) and walks it on the HOST with the kernels' node arithmetic
// (qnode_slab_host mirrors Traversal::visit) and their triangle test on the uploaded records for every ray (8 floats: o, d,
// tmin, tmax).  The closest t must equal the brute-force closest t over all triangles bit for bit (ids may differ only on exact
// ties).  Returns the number of rays whose t differs in *mismatches; also verifies the link remap.
int tgb200_qbvh_selftest(const float *tri_verts, uint32_t n, const float *rays, uint32_t n_rays,
                         uint32_t *mismatches, uint32_t *n_nodes, uint64_t *node_visits) {
    if ((n && !tri_verts) || (n_rays && !rays) || !mismatches) return TGB_ERR_INVALID;
    float extent = 0.0f;
    for (uint32_t r = 0; r < n_rays; ++r) for (int k = 0; k < 3; ++k) extent = std::max(extent, std::fabs(rays[8*size_t(r) + k]));
    SceneBvh sb;
    build_triangle_scene_bvh(tri_verts, n, extent, sb);
    const Bvh4 &bvh = sb.tree; const QBvh4 &qb = sb.qtree;
    const int32_t empty_link = ~int32_t(n << 3);                       // the leaf of the all-zero record behind the last triangle
    if (n_nodes) *n_nodes = uint32_t(qb.nodes.size());
    if (qb.nodes.size() != bvh.nodes.size()) return TGB_ERR_INVALID;
    for (size_t i = 0; i < qb.nodes.size(); ++i) {                      // links: same leaves, children remapped consistently
        const Node4 &src = bvh.nodes[size_t(qb.old_index[i])];
        for (int k = 0; k < 4; ++k) {
            int32_t l = qb.nodes[i].link[k];
            if (src.link[k] < 0) { if (l != (src.link[k] == kEmptyLink ? empty_link : src.link[k])) return TGB_ERR_INVALID; }
            else if (l < 0 || size_t(l) >= qb.nodes.size() || qb.old_index[size_t(l)] != src.link[k]) return TGB_ERR_INVALID;
        }
    }
    uint32_t bad = 0; uint64_t visits = 0;
    std::vector<int32_t> stack;
    for (uint32_t r = 0; r < n_rays; ++r) {
        const float *ry = rays + 8*size_t(r);
        V3 o = f3(ry), d = f3(ry + 3); float tnear = ry[6], tfar = ry[7];
        float brute = tfar;
        for (uint32_t k = 0; k < n; ++k) host_triangle(sb.isect[k], o, d, tnear, brute);
        float best = tfar;
        if (!qb.nodes.empty()) {
            float inv[3]; host_inv_dir(d, inv);
            float oo[3] = {o.x, o.y, o.z};
            stack.clear(); stack.push_back(0);
            while (!stack.empty()) {
                int32_t cur = stack.back(); stack.pop_back();
                if (cur >= 0) {
                    float t4[4]; visits++;
                    qnode_slab_host(qb.nodes[size_t(cur)], oo, inv, tnear, best, t4);
                    for (int k = 0; k < 4; ++k) if (t4[k] != INFINITY) stack.push_back(qb.nodes[size_t(cur)].link[k]);
                } else {
                    int code = ~cur; uint32_t first = uint32_t(code >> 3), count = uint32_t(code & 3) + 1;
                    for (uint32_t i = 0; i < count; ++i) host_triangle(sb.isect[first + i], o, d, tnear, best);
                }
            }
        }
        if (std::memcmp(&best, &brute, 4) != 0) bad++;
    }
    *mismatches = bad;
    if (node_visits) *node_visits = visits;
    return TGB_OK;
}

// Host-only count of the any-hit shadow walk's work (no GPU).  Builds the tree, top-level cut and records tgb200_create builds for
// a scene of n triangles seen from camera_pos, and walks every query (8 floats: o, d, tnear, t_light) with the kernels' node and
// triangle arithmetic twice: as k_shadow_bvh walked any-hit queries before (children sorted near-to-far, from the root) and as it
// walks them now (nearest child entered, the others pushed unsorted, from the cut boxes the segment enters).  A query that enters no cut box is not walked: k_shadow_prep settles it.
// out = 11 uint32 per query: cut mask, deepest stack of the walk from the cut, then per walk (root, cut): occluded, node visits,
// LEAF trips, triangle tests; last, the deepest stack of the walk from the root.  For a query that meets no triangle the root walk
// is the closest-hit walk of k_trace (same order, same culling: its t_max never shrinks), so that column is k_trace's stack too.  *stack_need = the bound tgb200_create checks; TGB_ERR_UNSUPPORTED when it exceeds stack_size (0: the
// traversal's stack), before any walk.
int tgb200_shadow_walk_count(const float *tri_verts, uint32_t n, const float *camera_pos, const float *queries, uint32_t n_queries,
                             uint32_t stack_size, uint32_t *stack_need, uint32_t *out) {
    if (!tri_verts || n == 0 || !camera_pos || (n_queries && (!queries || !out))) return TGB_ERR_INVALID;
    SceneBvh sb;
    build_triangle_scene_bvh(tri_verts, n, std::max(std::max(std::fabs(camera_pos[0]), std::fabs(camera_pos[1])), std::fabs(camera_pos[2])), sb);
    if (stack_need) *stack_need = sb.stack_need;
    if (sb.stack_need > (stack_size ? stack_size : uint32_t(kStackSize))) return TGB_ERR_UNSUPPORTED;
    const std::vector<CutBox> &cut = sb.cut; const QBvh4 &qb = sb.qtree;
    std::vector<int32_t> stack;
    for (uint32_t r = 0; r < n_queries; ++r) {
        const float *q = queries + 8*size_t(r);
        const V3 o = f3(q), d = f3(q + 3); const float tnear = q[6], tfar = q[7];
        float inv[3]; host_inv_dir(d, inv);
        const float oo[3] = {o.x, o.y, o.z}, ood[3] = {o.x*inv[0], o.y*inv[1], o.z*inv[2]};
        uint32_t mask = 0;                                                  // mesh_cut_test<true>
        for (size_t k = 0; k < cut.size(); ++k) {
            float tmn = tnear, tmx = tfar;
            for (int a = 0; a < 3; ++a) {
                const float ta = std::fmaf(cut[k].lo[a], inv[a], -ood[a]), tb = std::fmaf(cut[k].hi[a], inv[a], -ood[a]);
                tmn = std::fmax(tmn, std::fmin(ta, tb)); tmx = std::fmin(tmx, std::fmax(ta, tb));
            }
            if (tmn <= tmx) mask |= 1u << k;
        }
        uint32_t *o10 = out + 11*size_t(r);
        std::memset(o10, 0, 11*sizeof(uint32_t));
        o10[0] = mask;
        if (!mask) continue;
        for (int from_cut = 0; from_cut < 2; ++from_cut) {
            uint32_t *c4 = o10 + 2 + 4*from_cut;
            stack.clear();
            if (from_cut) { for (int k = int(cut.size()) - 1; k >= 0; --k) if (mask & (1u << k)) stack.push_back(cut[size_t(k)].link); }
            else stack.push_back(0);
            bool occluded = false;
            int32_t cur = stack.back(); stack.pop_back();
            size_t deepest = stack.size();
            for (;;) {
                if (cur >= 0) {
                    float t[4]; c4[1]++;
                    qnode_slab_host(qb.nodes[size_t(cur)], oo, inv, tnear, tfar, t);
                    int32_t l[4] = {qb.nodes[size_t(cur)].link[0], qb.nodes[size_t(cur)].link[1], qb.nodes[size_t(cur)].link[2], qb.nodes[size_t(cur)].link[3]};
                    auto cswap = [&](int a, int b) { if (t[b] < t[a]) { std::swap(t[a], t[b]); std::swap(l[a], l[b]); } };
                    cswap(0, 1); cswap(2, 3); cswap(0, 2);
                    if (!from_cut) { cswap(1, 3); cswap(1, 2); }
                    if (t[0] != INFINITY) {
                        for (int k = 3; k >= 1; --k) if (t[k] != INFINITY) stack.push_back(l[k]);
                        deepest = std::max(deepest, stack.size());
                        cur = l[0];
                        continue;
                    }
                } else {
                    const int code = ~cur; const uint32_t first = uint32_t(code >> 3), count = uint32_t(code & 3) + 1;
                    c4[2]++;
                    for (uint32_t i = 0; i < count && !occluded; ++i) {
                        c4[3]++;
                        float best = tfar;
                        occluded = host_triangle(sb.isect[first + i], o, d, tnear, best);
                    }
                    if (occluded) break;
                }
                if (stack.empty()) break;
                cur = stack.back(); stack.pop_back();
            }
            c4[0] = occluded ? 1u : 0u;
            o10[from_cut ? 1 : 10] = uint32_t(deepest);
        }
    }
    return TGB_OK;
}


int tgb200_bsdf_probe(tgb_ctx *c, int bsdf, float u, float v, uint32_t requested, int lobe_set, uint32_t n, const float *wi_wo,
                      float *out) {
    if (!c || (n && (!wi_wo || !out))) return TGB_ERR_INVALID;
    if (int rc = probe_check(c, lobe_set)) return rc;
    if (bsdf < 0 || bsdf >= c->n_bsdfs) return fail(c, TGB_ERR_INVALID, "bsdf %d out of range", bsdf);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<float> dw, dout;
    cudaError_t e = dw.upload(wi_wo, 6*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(4*size_t(n));
    if (e == cudaSuccess) {
        const uint32_t g = blocks(n, 128);
        if (c->has_curves) k_probe_bsdf<true, 0><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw.p, dout.p, n);
        else if (lobe_set == 1) k_probe_bsdf<false, 1><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw.p, dout.p, n);
        else k_probe_bsdf<false, 0><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw.p, dout.p, n);
        e = download(c, out, dout.p, 4*size_t(n));
    }
    return b.finish(e, "bsdf_probe");
}

int tgb200_bsdf_sample_probe(tgb_ctx *c, uint32_t seed, uint32_t n, const int *bsdf, const uint32_t *pixel_id, uint32_t sample,
                             float u, float v, uint32_t requested, int lobe_set, const float *wi, float *out, uint32_t *lobes) {
    if (!c || (n && (!bsdf || !pixel_id || !wi || !out || !lobes))) return TGB_ERR_INVALID;
    if (int rc = probe_check(c, lobe_set)) return rc;
    for (uint32_t i = 0; i < n; ++i)
        if (bsdf[i] < 0 || bsdf[i] >= c->n_bsdfs) return fail(c, TGB_ERR_INVALID, "bsdf %d out of range", bsdf[i]);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<int> db; Buffer<uint32_t> dpix, dl; Buffer<float> dwi, dout;
    cudaError_t e = db.upload(bsdf, n, c->stream);
    if (e == cudaSuccess) e = dpix.upload(pixel_id, n, c->stream);
    if (e == cudaSuccess) e = dwi.upload(wi, 3*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(8*size_t(n));
    if (e == cudaSuccess) e = dl.ensure(n);
    if (e == cudaSuccess) {
        const uint32_t g = blocks(n, 128);
        if (c->has_curves) k_probe_bsdf_sample<true, 0><<<g, 128, 0, c->stream>>>(c->sc, seed, db.p, dpix.p, sample, u, v, requested, dwi.p, dout.p, dl.p, n);
        else if (lobe_set == 1) k_probe_bsdf_sample<false, 1><<<g, 128, 0, c->stream>>>(c->sc, seed, db.p, dpix.p, sample, u, v, requested, dwi.p, dout.p, dl.p, n);
        else k_probe_bsdf_sample<false, 0><<<g, 128, 0, c->stream>>>(c->sc, seed, db.p, dpix.p, sample, u, v, requested, dwi.p, dout.p, dl.p, n);
        e = download(c, out, dout.p, 8*size_t(n));
        if (e == cudaSuccess) e = download(c, lobes, dl.p, n);
    }
    return b.finish(e, "bsdf_sample_probe");
}

int tgb200_light_probe(tgb_ctx *c, int prim, uint32_t seed, uint32_t n, uint32_t sample, const float *p, float *out) {
    if (!c || (n && (!p || !out))) return TGB_ERR_INVALID;
    if (prim < 0 || uint32_t(prim) >= c->sc.n_prims) return fail(c, TGB_ERR_INVALID, "primitive %d out of range", prim);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<float> dp, dout; Buffer<tgb_ray> dr; Buffer<Hit> dx; Buffer<uint32_t> list;
    cudaError_t e = dp.upload(p, 3*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(12*size_t(n));
    if (e == cudaSuccess) e = dr.ensure(n);
    if (e == cudaSuccess) e = dx.ensure(n);
    if (e == cudaSuccess) {
        k_probe_light<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, prim, seed, sample, dp.p, dout.p, dr.p, n);
        if (c->prim_types[size_t(prim)] == TGB_PRIM_MESH && (e = hook_closest(c, dr.p, dx.p, n, list)) == cudaSuccess)
            k_probe_light_mesh<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, prim, dr.p, dx.p, dout.p, n);
        if (e == cudaSuccess) e = download(c, out, dout.p, 12*size_t(n));
    }
    return b.finish(e, "light_probe");
}

int tgb200_choose_light_probe(tgb_ctx *c, uint32_t seed, uint32_t n, const uint32_t *pixel_id, uint32_t sample, const float *p,
                              float *out) {
    if (!c || (n && (!pixel_id || !p || !out))) return TGB_ERR_INVALID;
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<uint32_t> dpix; Buffer<float> dp, dout;
    cudaError_t e = dpix.upload(pixel_id, n, c->stream);
    if (e == cudaSuccess) e = dp.upload(p, 3*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(2*size_t(n));
    if (e == cudaSuccess) {
        k_probe_choose_light<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, seed, dpix.p, sample, dp.p, dout.p, n);
        e = download(c, out, dout.p, 2*size_t(n));
    }
    return b.finish(e, "choose_light_probe");
}

int tgb200_shadow_probe(tgb_ctx *c, uint32_t n, const float *query, const int *light_mis, float *out) {
    if (!c || (n && (!query || !light_mis || !out))) return TGB_ERR_INVALID;
    for (uint32_t i = 0; i < n; ++i)
        if (std::find(c->light_ids.begin(), c->light_ids.end(), light_mis[2*size_t(i)]) == c->light_ids.end())
            return fail(c, TGB_ERR_INVALID, "query %u: primitive %d is not a samplable light", i, light_mis[2*size_t(i)]);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<float> dq, dout; Buffer<int> dl;
    cudaError_t e = dq.upload(query, 8*size_t(n), c->stream);
    if (e == cudaSuccess) e = dl.upload(light_mis, 2*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(8*size_t(n));
    if (e == cudaSuccess) e = b.save_state();
    const Wavefront &w = c->wf[0];
    const DScene &sc = c->sc; cudaStream_t st = c->stream;
    // one scratch slot per query: chunks of wavefront 0's capacity
    for (uint32_t off = 0; off < n && e == cudaSuccess; off += w.capacity) {
        const uint32_t m = std::min(w.capacity, n - off);
        // shadow_count, shadow_count2, cursor_trace, cursor_shadow, shadow_count_closest, cursor_closest
        e = cudaMemsetAsync(&w.ctl->shadow_count, 0, 6*sizeof(uint32_t), st);
        if (e != cudaSuccess) break;
        k_probe_shadow_setup<<<blocks(m, 128), 128, 0, st>>>(sc, w.sr, dq.p + 8*size_t(off), dl.p + 2*size_t(off), dout.p + 8*size_t(off),
                                                            w.squeue, w.ctl, m);
        c->ks.shadow_prep<<<loop_grid(c->prep_blocks, m), 256, 0, st>>>(sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
        k_probe_shadow_traversed<<<blocks(m, 256), 256, 0, st>>>(w.squeue2, w.squeue_cl, w.ctl, dout.p + 8*size_t(off));
        if (sc.n_nodes)
            c->ks.shadow_bvh<<<std::min(blocks(m, kTraceBlock), c->persist_blocks), kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
        k_probe_shadow_read<<<blocks(m, 128), 128, 0, st>>>(w.sr, dl.p + 2*size_t(off), dout.p + 8*size_t(off), m);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = download(c, out, dout.p, 8*size_t(n));
    return b.finish(e, "shadow_probe");
}

int tgb200_bounce_probe(tgb_ctx *c, uint32_t n, const uint32_t *state_in, uint32_t *state_out) {
    if (!c || (n && (!state_in || !state_out))) return TGB_ERR_INVALID;
    const uint32_t max_bounces = c->sc.set.max_bounces;
    for (uint32_t i = 0; i < n; ++i) {
        const uint32_t *r = state_in + TGB_BOUNCE_WORDS*size_t(i);
        if (r[TGB_BR_BOUNCE] >= max_bounces || r[TGB_BR_BOUNCE] > 0xFFu || r[TGB_BR_DIMENSION] > 0xFFFFu)
            return fail(c, TGB_ERR_INVALID, "state %u: bounce %u (max_bounces %u) or dimension %u out of range", i, r[TGB_BR_BOUNCE],
                        max_bounces, r[TGB_BR_DIMENSION]);
    }
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    Wavefront &w = c->wf[0];
    if (int rc = ensure_results(c, w.capacity)) return rc;
    ProbeBufs b(c);
    Buffer<uint32_t> din, dout, pix;
    cudaError_t e = din.upload(state_in, TGB_BOUNCE_WORDS*size_t(n), c->stream);
    if (e == cudaSuccess) e = dout.ensure(TGB_BOUNCE_WORDS*size_t(n));
    if (e == cudaSuccess) e = pix.ensure(4*size_t(w.capacity) + 1);
    if (e == cudaSuccess) e = b.save_state();
    const DScene &sc = c->sc; cudaStream_t st = c->stream;
    PathBuf &pb = w.pb[0], &dst = w.pb[1];
    // per chunk: one pixel per path (pix_id, pix_seed, pix_first (m + 1 offsets), pix_base), so path id = result slot = its index
    uint32_t *pix_id = pix.p, *pix_seed = pix.p + w.capacity, *pix_base = pix.p + 2*size_t(w.capacity), *pix_first = pix.p + 3*size_t(w.capacity);
    for (uint32_t off = 0; off < n && e == cudaSuccess; off += w.capacity) {
        const uint32_t m = std::min(w.capacity, n - off);
        // the states enter as m survivors k_accum has just handed over, with no camera path left to issue: k_iter_end and
        // k_bin_scatter then set up the iteration (survivor count, traversal order by ray-coherence key, culled survivors left out)
        Ctl init; std::memset(&init, 0, sizeof(Ctl));
        init.next_count = m; init.capacity = w.capacity;
        e = cudaMemcpyAsync(w.ctl, &init, sizeof(Ctl), cudaMemcpyHostToDevice, st);
        if (e == cudaSuccess) e = cudaMemsetAsync(w.bin_hist, 0, kBins*sizeof(uint32_t), st);
        if (e != cudaSuccess) break;
        BatchInfo bi; bi.pix_id = pix_id; bi.pix_seed = pix_seed; bi.n_pix = m; bi.spp_begin = 0;
        bi.pix_first = pix_first; bi.pix_base = pix_base;
        bi.pix_bits = index_bits(m);
        uint32_t *o = dout.p + TGB_BOUNCE_WORDS*size_t(off);
        k_probe_bounce_setup<<<blocks(m, 256), 256, 0, st>>>(sc, pb, din.p + TGB_BOUNCE_WORDS*size_t(off), pix_id, pix_seed, pix_first,
                                                            pix_base, w.bin_keys, w.bin_hist, o, m);
        k_iter_end<<<1, 1024, 0, st>>>(w.bin_hist, w.ctl, sc.n_nodes ? 1 : 0);
        if (sc.n_nodes) k_bin_scatter<<<loop_grid(c->scatter_blocks, m), 256, 0, st>>>(w.bin_keys, w.bin_hist, w.ctl, w.order);
        enqueue_bounce(c, w, pb, dst, st, bi, m, nullptr);
        k_probe_bounce_alive<<<blocks(m, 256), 256, 0, st>>>(dst, w.ctl, o);
        k_probe_bounce_finished<<<blocks(m, 256), 256, 0, st>>>(pb, c->R.p, o, m);
        e = cudaGetLastError();
        // (the next chunk's control block is copied from this host variable: wait until this one is consumed)
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e == cudaSuccess) e = download(c, state_out, dout.p, TGB_BOUNCE_WORDS*size_t(n));
    return b.finish(e, "bounce_probe");
}

int tgb200_bin_probe(tgb_ctx *c, uint32_t n, const uint32_t *keys, uint32_t *order, uint32_t *cursors, uint32_t *n_sorted) {
    if (!c || !cursors || !n_sorted || (n && (!keys || !order))) return TGB_ERR_INVALID;
    Wavefront &w = c->wf[0];
    if (n > w.capacity) return fail(c, TGB_ERR_INVALID, "%u survivors: wavefront 0 holds %u", n, w.capacity);
    for (uint32_t i = 0; i < n; ++i)
        if (keys[i] > kBins) return fail(c, TGB_ERR_INVALID, "survivor %u: key %u is past kBins (%u)", i, keys[i], kBins);
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    Buffer<uint32_t> dkeys;
    cudaError_t e = dkeys.upload(keys, n, c->stream);
    if (e == cudaSuccess) e = b.save_state();
    const cudaStream_t st = c->stream;
    // n survivors just handed over by k_accum, with no camera path left to issue (as tgb200_bounce_probe stages them)
    Ctl init; std::memset(&init, 0, sizeof(Ctl));
    init.next_count = n; init.capacity = w.capacity;
    if (e == cudaSuccess) e = cudaMemcpyAsync(w.ctl, &init, sizeof(Ctl), cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(w.bin_hist, 0, kBins*sizeof(uint32_t), st);
    if (e == cudaSuccess) {
        k_probe_bin_setup<<<blocks(n, 256), 256, 0, st>>>(dkeys.p, w.bin_keys, w.bin_hist, n);
        k_iter_end<<<1, 1024, 0, st>>>(w.bin_hist, w.ctl, 1);
        k_bin_scatter<<<loop_grid(c->scatter_blocks, n), 256, 0, st>>>(w.bin_keys, w.bin_hist, w.ctl, w.order);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = download(c, n_sorted, &w.ctl->n_sorted, 1);
    if (e == cudaSuccess) e = download(c, cursors, w.bin_hist, kBins);
    // (init and n_sorted are host variables the stream reads and writes: wait before reading n_sorted or leaving)
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e == cudaSuccess && *n_sorted) e = download(c, order, w.order, std::min(*n_sorted, n));
    return b.finish(e, "bin_probe");
}

int tgb200_shade_variant(const tgb_ctx *c, uint32_t *variant) {
    if (!c || !variant) return TGB_ERR_INVALID;
    std::memcpy(variant, c->ks.variant, sizeof(c->ks.variant));
    return TGB_OK;
}

int tgb200_clear_abort(tgb_ctx *c) {
    if (!c) return TGB_ERR_INVALID;
    for_members(c, [](tgb_ctx *m) { return tgb200_clear_abort(m); });
    c->abort_flag.store(0);
    return TGB_OK;
}

int tgb200_abort(tgb_ctx *c) {
    if (!c) return TGB_ERR_INVALID;
    for_members(c, [](tgb_ctx *m) { return tgb200_abort(m); });
    c->abort_flag.store(1);
    return TGB_OK;
}

}  // extern "C"