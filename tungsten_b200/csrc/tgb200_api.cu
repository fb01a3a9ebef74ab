// C ABI of libtgb200.so (include/tgb200.h): scene preparation, device upload, wavefront render loop.
// Host logic mirrors the reference's TraceableScene constructor + PathTraceIntegrator (prepare, tile
// dicing, sample stepping); all rendering arithmetic runs in the CUDA kernels of tgb_wavefront.cuh.
// There is NO CPU fallback: without a CUDA device every entry point fails with TGB_ERR_NO_DEVICE.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "bvh_build.h"
#include "hair_tables.h"
#include "tgb_wavefront.cuh"
#include "tgb_probe.cuh"

extern "C" const unsigned char tgb_sobol_blob[];      // sobol_blob.cpp (.incbin of data/sobol_1024x32.u32)

using namespace tgb;

#include <thread>
#include <map>

struct tgb_ctx;
struct Group {
    std::vector<tgb_ctx *> members;                     // members[0] = root
    std::vector<tgb_tile> deal_key; uint32_t deal_seed = 0;      // tile list the cached deal belongs to
    std::vector<std::vector<tgb_tile>> shares;           // per member
    std::vector<uint32_t *> root_pix;                    // per member k >= 1: its share's pixel ids on the ROOT device
    std::vector<uint32_t> share_pixels;
    std::vector<float4 *> send;                          // per member k >= 1: pack buffer on ITS device
    float4 *recv = nullptr; size_t recv_capacity = 0;    // on the root device
    std::vector<size_t> send_capacity;
    double gather_ms = 0.0;
};

namespace {

thread_local std::string g_create_error;

struct DeviceBuf {
    void *p = nullptr; size_t bytes = 0;
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
    Ctl *h_ctl = nullptr;           // pinned: [0..3] snapshot ring (read one iteration late), [4] initial value
    cudaEvent_t ev_ring[4]{};
    cudaEvent_t ev_k[4][8]{};       // profiling: boundaries between the kernels of an iteration (regen|trace|shade|prep|shadow|accum|sort)
};

}  // namespace

struct tgb_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;  // the caller's stream (tgb200_set_stream) or own_stream: wavefront 0, k_resolve, the hooks
    cudaStream_t stream1 = nullptr; // wavefront 1
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    std::string error;
    std::atomic<int> abort_flag{0};
    std::vector<void *> allocs;
    DScene sc{};
    uint32_t res_x = 0, res_y = 0;
    // wavefront storage
    uint32_t capacity = 0;          // paths in flight, both wavefronts together
    Wavefront wf[2];                // the hooks run on wf[0]'s buffers
    bool mesh_lights = false;       // a mesh is a light: closest-hit shadow queries exist, k_shadow_bvh<., false> runs
    uint32_t persist_blocks = 0;    // grid of the persistent traversal kernels (per wavefront)
    bool diffuse_only = false;      // all surfaces Lambert / null: k_shade<.., .., 1>
    bool sort_materials = false;    // >= 2 lobe models in use: k_shade deals the paths of a block to its threads by BSDF type
    bool has_curves = false;        // selects the kernel instantiations with the curve-segment test and per-hit epsilon
    int n_bsdfs = 0; std::vector<uint32_t> prim_types; std::vector<int> light_ids;   // host copies for the test hooks' argument checks
    float4 *R = nullptr; size_t res_capacity = 0;   // finished radiance per path of the (sub)step
    cudaStream_t own_stream = nullptr;
    struct Group *group = nullptr;  // multi-GPU: set on the root context (devices[0]); members[0] == the root itself
    Counters *ctr = nullptr; Counters *h_ctr = nullptr;
    float *fb = nullptr; uint32_t *fb_count = nullptr;
    float *h_fb = nullptr; uint32_t *h_fb_count = nullptr;   // pinned staging
    // cached pixel list
    std::vector<tgb_tile> tiles_cached; uint32_t *pix_id = nullptr, *pix_seed = nullptr; uint32_t n_pix = 0, pix_capacity = 0;
    std::vector<uint32_t> h_pix_id;                  // host copy of the pixel list (adaptive steps build per-pixel sample ranges from it)
    // adaptive sampling: per-pixel result-slot offsets / first sample index, pixel -> list index map, the 4x4 blocks' SampleRecords
    uint32_t *pix_first = nullptr, *pix_base = nullptr, *pix_slot = nullptr; uint32_t adaptive_capacity = 0; bool pix_slot_valid = false;
    SampleRecordD *rec_dev = nullptr;
    tgb_stats stats{};
    bool profiling = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    uint32_t bvh_depth = 0; uint32_t n_tris = 0; double bvh_sah = 0.0; size_t geom_bytes = 0;
};

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
    void *p = nullptr;
    CU(cudaMalloc(&p, std::max<size_t>(n, 1)*sizeof(T)));
    c->allocs.push_back(p);
    *out = static_cast<T *>(p);
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

V3 f3(const float *p) { return v3(p[0], p[1], p[2]); }
void transpose3(const float *m, float *t) {
    t[0] = m[0]; t[1] = m[3]; t[2] = m[6]; t[3] = m[1]; t[4] = m[4]; t[5] = m[7]; t[6] = m[2]; t[7] = m[5]; t[8] = m[8];
}

// ---- host-side "prepareForRender" pieces (fp32, reference operation order; compiled with -fmad=false) ----
float filter_width(uint32_t f) {
    switch (f) { case TGB_FILTER_DIRAC: return 0.0f; case TGB_FILTER_BOX: return 0.5f; case TGB_FILTER_TENT: return 1.0f; default: return 2.0f; }
}
float filter_eval(uint32_t f, float x) {                        // cameras/ReconstructionFilter.hpp:171-193
    switch (f) {
    case TGB_FILTER_BOX: return (x >= -0.5f && x <= 0.5f) ? 1.0f : 0.0f;
    case TGB_FILTER_TENT: return 1.0f - std::fabs(x);
    case TGB_FILTER_GAUSSIAN: { const float Alpha = 2.0f; return std::max(std::exp(-Alpha*x*x) - std::exp(-Alpha*4.0f), 0.0f); }
    case TGB_FILTER_MITCHELL: { x = std::fabs(x); const float B = 1.0f/3.0f, C = 1.0f/3.0f;
        if (x < 1.0f) return 1.0f/6.0f*((12.0f - 9.0f*B - 6.0f*C)*x*x*x + (-18.0f + 12.0f*B + 6.0f*C)*x*x + (6.0f - 2.0f*B));
        else if (x < 2.0f) return 1.0f/6.0f*((-B - 6.0f*C)*x*x*x + (6.0f*B + 30.0f*C)*x*x + (-12.0f*B - 48.0f*C)*x + (8.0f*B + 24.0f*C));
        return 0.0f; }
    case TGB_FILTER_CATMULL_ROM: { x = std::fabs(x);
        if (x < 1.0f) return 1.0f/6.0f*((12.0f - 3.0f)*x*x*x + (-18.0f + 3.0f)*x*x + 6.0f);
        else if (x < 2.0f) return 1.0f/6.0f*(-3.0f*x*x*x + 15.0f*x*x - 24.0f*x + 12.0f);
        return 0.0f; }
    case TGB_FILTER_LANCZOS: { x = std::fabs(x);
        if (x == 0.0f) return 1.0f;
        else if (x < 2.0f) return std::sin(PI_F*x)*std::sin(PI_F*x/2.0f)/(PI_F*PI_F*x*x/2.0f);
        return 0.0f; }
    default: return 0.0f;
    }
}
void filter_precompute(DCamera &cam) {                          // cameras/ReconstructionFilter.cpp:34-58
    const int R = 31;
    float width = filter_width(cam.filter);
    cam.filter_bin = width/R;
    std::memset(cam.filter_cdf, 0, sizeof(cam.filter_cdf));
    if (cam.filter == TGB_FILTER_BOX || cam.filter == TGB_FILTER_DIRAC) return;
    float f[32], sum = 0.0f;
    for (int i = 0; i < R; ++i) { f[i] = filter_eval(cam.filter, (i*width)/R); sum += f[i]; }
    cam.filter_cdf[0] = 0.0f;
    for (int i = 1; i < R; ++i) cam.filter_cdf[i] = cam.filter_cdf[i - 1] + f[i - 1]/sum;
    cam.filter_cdf[R] = 1.0f;
}
float h_dielectric_reflectance(float eta, float cosThetaI) {    // bsdfs/Fresnel.hpp:75-92
    if (cosThetaI < 0.0f) { eta = 1.0f/eta; cosThetaI = -cosThetaI; }
    float sinThetaTSq = eta*eta*(1.0f - cosThetaI*cosThetaI);
    if (sinThetaTSq > 1.0f) return 1.0f;
    float cosThetaT = std::sqrt(std::max(1.0f - sinThetaTSq, 0.0f));
    float Rs = (eta*cosThetaI - cosThetaT)/(eta*cosThetaI + cosThetaT);
    float Rp = (eta*cosThetaT - cosThetaI)/(eta*cosThetaT + cosThetaI);
    return (Rs*Rs + Rp*Rp)*0.5f;
}
float diffuse_fresnel(float ior, int sampleCount) {             // bsdfs/Fresnel.hpp:141-153
    double acc = 0.0;
    float fb = h_dielectric_reflectance(ior, 0.0f);
    for (int i = 1; i <= sampleCount; ++i) {
        float cosThetaSq = float(i)/sampleCount;
        float fa = h_dielectric_reflectance(ior, std::min(std::sqrt(cosThetaSq), 1.0f));
        acc += double(fa + fb)*(0.5/sampleCount);
        fb = fa;
    }
    return float(acc);
}
uint32_t bsdf_lobes(const tgb_bsdf &b) {
    switch (b.type) {
    case TGB_BSDF_NULL: return 0;
    case TGB_BSDF_LAMBERT: return LOBE_DIFFUSE_R;
    case TGB_BSDF_ROUGH_CONDUCTOR: return LOBE_GLOSSY_R;
    case TGB_BSDF_ROUGH_DIELECTRIC: return b.enable_refraction ? (LOBE_GLOSSY_R | LOBE_GLOSSY_T) : LOBE_GLOSSY_R;
    case TGB_BSDF_PLASTIC: return LOBE_SPEC_R | LOBE_DIFFUSE_R;
    case TGB_BSDF_ROUGH_PLASTIC: return LOBE_GLOSSY_R | LOBE_DIFFUSE_R;
    case TGB_BSDF_MIRROR: case TGB_BSDF_CONDUCTOR: return LOBE_SPEC_R;                   // MirrorBsdf.cpp:13, ConductorBsdf.cpp:19
    case TGB_BSDF_DIELECTRIC: return b.enable_refraction ? (LOBE_SPEC_R | LOBE_SPEC_T) : LOBE_SPEC_R;   // DielectricBsdf.cpp:174-180
    case TGB_BSDF_SMOOTH_COAT: return LOBE_SPEC_R;          // | substrate lobes, added by upload_scene
    case TGB_BSDF_ROUGH_COAT: return LOBE_GLOSSY_R;         // | substrate lobes (RoughCoatBsdf.cpp:301-306)
    case TGB_BSDF_HAIR: return LOBE_GLOSSY_R | LOBE_GLOSSY_T | LOBE_ANISO;                  // bsdfs/HairBcsdf.cpp:20
    default: return 0xFFFFFFFFu;
    }
}

struct HostTex { DTex d; V3 maxv; std::vector<float> marg_pdf, marg_cdf, pdf, cdf; bool has_dist = false; };

// BitmapTexture::makeSamplable(MAP_SPHERICAL) + Distribution2D (textures/BitmapTexture.cpp:400-431,
// sampling/Distribution2D.hpp:18-46)
void build_spherical_distribution(const tgb_texture &t, HostTex &ht) {
    int w = int(t.res_u), h = int(t.res_v); bool clampm = (t.flags >> 1) & 1;
    std::vector<float> weights(size_t(w)*h);
    for (int y = 0, idx = 0; y < h; ++y) {
        float rowWeight = 1.0f;
        rowWeight *= std::sin((y*PI_F)/h);
        for (int x = 0; x < w; ++x, ++idx) {
            const float *p = t.texels + 3*size_t(idx);
            weights[idx] = max_comp(v3(p[0], p[1], p[2]))*rowWeight;
        }
    }
    // in-place max dilation, x then y, wrapping unless the texture clamps (BitmapTexture.cpp:411-428)
    for (int y = 0; y < h; ++y) {
        for (int x = 0; x < w - 1; ++x) weights[x + y*w] = std::max(weights[x + y*w], weights[x + 1 + y*w]);
        if (!clampm) weights[y*w] = weights[w - 1 + y*w] = std::max(weights[w - 1 + y*w], weights[y*w]);
        for (int x = w - 1; x > 0; --x) weights[x + y*w] = std::max(weights[x + y*w], weights[x - 1 + y*w]);
    }
    for (int x = 0; x < w; ++x) {
        for (int y = 0; y < h - 1; ++y) weights[x + y*w] = std::max(weights[x + y*w], weights[x + (y + 1)*w]);
        if (!clampm) weights[x] = weights[x + (h - 1)*w] = std::max(weights[x], weights[x + (h - 1)*w]);
        for (int y = h - 1; y > 0; --y) weights[x + y*w] = std::max(weights[x + y*w], weights[x + (y - 1)*w]);
    }
    // Distribution2D (sampling/Distribution2D.hpp:18-60)
    ht.pdf = weights; ht.cdf.assign(size_t(w + 1)*h, 0.0f); ht.marg_pdf.assign(h, 0.0f); ht.marg_cdf.assign(h + 1, 0.0f);
    for (int y = 0; y < h; ++y) {
        int idxP = y*w, idxC = y*(w + 1);
        ht.cdf[idxC] = 0.0f;
        for (int x = 0; x < w; ++x, ++idxP, ++idxC) { ht.marg_pdf[y] += ht.pdf[idxP]; ht.cdf[idxC + 1] = ht.cdf[idxC] + ht.pdf[idxP]; }
        ht.marg_cdf[y + 1] = ht.marg_cdf[y] + ht.marg_pdf[y];
    }
    for (int y = 0; y < h; ++y) {
        int idxP = y*w, idxC = y*(w + 1), idxTail = idxC + w;
        float rowWeight = ht.cdf[idxTail];
        if (rowWeight < 1e-4f) { for (int x = 0; x < w; ++x, ++idxP, ++idxC) { ht.pdf[idxP] = 1.0f/w; ht.cdf[idxC] = x/float(w); } }
        else { for (int x = 0; x < w; ++x, ++idxP, ++idxC) { ht.pdf[idxP] /= rowWeight; ht.cdf[idxC] /= rowWeight; } }
        ht.cdf[idxTail] = 1.0f;
    }
    float totalWeight = ht.marg_cdf[h];
    for (float &p : ht.marg_pdf) p /= totalWeight;
    for (float &cc : ht.marg_cdf) cc /= totalWeight;
    ht.marg_cdf[h] = 1.0f;
    ht.has_dist = true;
}

// The BVH build switches: BvhOptions' defaults, overridden from the environment (DESIGN.md section 6).  tgb200_create and the
// host-only BVH checks read them alike, so the checks walk the tree tgb200_create builds.
BvhOptions bvh_options() {
    BvhOptions o;
    if (const char *e = getenv("TGB_TRI_LEAF")) o.tri_leaf = uint32_t(atoi(e));
    if (const char *e = getenv("TGB_TRI_COST")) o.tri_cost = float(atof(e));
    if (const char *e = getenv("TGB_CURVE_LEAF")) o.curve_leaf = uint32_t(atoi(e));
    if (const char *e = getenv("TGB_CURVE_COST")) o.curve_cost = float(atof(e));
    if (const char *e = getenv("TGB_CUT_BOXES")) o.max_cut = size_t(std::min(16, std::max(4, atoi(e))));
    return o;
}

// World bounds of a quad's four corners or a cube's eight
Aabb analytic_bounds(const DPrim &p) {
    Aabb b = {{INFINITY, INFINITY, INFINITY}, {-INFINITY, -INFINITY, -INFINITY}};
    auto grow = [&](V3 q) { float v[3] = {q.x, q.y, q.z}; for (int a = 0; a < 3; ++a) { b.lo[a] = std::min(b.lo[a], v[a]); b.hi[a] = std::max(b.hi[a], v[a]); } };
    if (p.type == TGB_PRIM_QUAD) { grow(p.base); grow(p.base + p.edge0); grow(p.base + p.edge1); grow(p.base + p.edge0 + p.edge1); }
    else for (int j = 0; j < 8; ++j) grow(p.pos + m3mul(p.rot, v3((j & 1 ? p.scale.x : -p.scale.x), (j & 2 ? p.scale.y : -p.scale.y), (j & 4 ? p.scale.z : -p.scale.z))));
    return b;
}

int upload_scene(tgb_ctx *c, const tgb_scene_desc *d) {
    const tgb_camera &cam = d->camera;
    DScene &sc = c->sc;
    sc.set = d->settings;
    // camera precompute (cameras/PinholeCamera.cpp:28-35, Camera.cpp:37-42)
    sc.cam.pos = f3(cam.pos); std::memcpy(sc.cam.m, cam.xform, sizeof(sc.cam.m));
    float fovRad = cam.fov_deg*(PI_F/180.0f);
    sc.cam.plane_dist = 1.0f/std::tan(fovRad*0.5f);
    sc.cam.ratio = cam.res_y/float(cam.res_x);
    sc.cam.pixel_size_x = 1.0f/cam.res_x;
    sc.cam.res_x = cam.res_x; sc.cam.res_y = cam.res_y; sc.cam.filter = cam.filter;
    filter_precompute(sc.cam);
    c->res_x = cam.res_x; c->res_y = cam.res_y;

    // ---- textures
    std::vector<HostTex> tex(d->n_textures + 1);
    for (uint32_t i = 0; i < d->n_textures; ++i) {
        const tgb_texture &t = d->textures[i]; DTex &o = tex[i].d;
        std::memset(&o, 0, sizeof(o));
        o.type = t.type; o.value = f3(t.value); o.value2 = f3(t.value2); o.res_u = int(t.res_u); o.res_v = int(t.res_v); o.flags = t.flags;
        if (t.type == TGB_TEX_BITMAP) {
            if (!t.texels || !t.res_u || !t.res_v) return fail(c, TGB_ERR_INVALID, "bitmap texture %u has no texels", i);
            size_t n = size_t(t.res_u)*t.res_v;
            V3 acc = v3s(0.0f), mx = v3s(0.0f);
            for (size_t k = 0; k < n; ++k) { V3 cc = f3(t.texels + 3*k); acc = acc + cc/float(n); mx = v3(std::max(mx.x, cc.x), std::max(mx.y, cc.y), std::max(mx.z, cc.z)); }
            o.avg = acc; tex[i].maxv = mx;
            std::vector<float> tx(t.texels, t.texels + 3*n);
            int rc = dev_upload(c, &o.texels, tx); if (rc) return rc;
        } else if (t.type == TGB_TEX_CHECKER) {
            o.avg = (o.value + o.value2)*0.5f;
            tex[i].maxv = v3(std::max(o.value.x, o.value2.x), std::max(o.value.y, o.value2.y), std::max(o.value.z, o.value2.z));
        } else if (t.type == TGB_TEX_CONSTANT) { o.avg = o.value; tex[i].maxv = o.value; }
        else return fail(c, TGB_ERR_UNSUPPORTED, "texture type %u is outside the hot path", t.type);
    }
    { DTex &o = tex[d->n_textures].d; std::memset(&o, 0, sizeof(o)); o.type = TGB_TEX_CONSTANT; o.value = v3s(1.0f); o.avg = o.value; tex[d->n_textures].maxv = o.value; }

    // ---- bsdfs
    std::vector<DBsdf> bsdfs(d->n_bsdfs);
    for (uint32_t i = 0; i < d->n_bsdfs; ++i) {
        const tgb_bsdf &b = d->bsdfs[i]; DBsdf &o = bsdfs[i];
        std::memset(&o, 0, sizeof(o));
        o.type = b.type; o.lobes = bsdf_lobes(b);
        if (o.lobes == 0xFFFFFFFFu) return fail(c, TGB_ERR_UNSUPPORTED, "bsdf type %u is outside the hot path", b.type);
        if (b.albedo_tex < 0 || uint32_t(b.albedo_tex) >= d->n_textures) return fail(c, TGB_ERR_INVALID, "bsdf %u: bad albedo texture", i);
        bool rough = b.type == TGB_BSDF_ROUGH_CONDUCTOR || b.type == TGB_BSDF_ROUGH_DIELECTRIC || b.type == TGB_BSDF_ROUGH_PLASTIC || b.type == TGB_BSDF_ROUGH_COAT;
        if (rough && (b.roughness_tex < 0 || uint32_t(b.roughness_tex) >= d->n_textures)) return fail(c, TGB_ERR_INVALID, "bsdf %u: bad roughness texture", i);
        o.dist = b.distribution; o.albedo_tex = b.albedo_tex; o.rough_tex = b.roughness_tex;
        o.ior = b.ior; o.inv_ior = 1.0f/b.ior; o.eta = f3(b.eta); o.k = f3(b.k); o.enable_t = b.enable_refraction; o.substrate = b.substrate;
        if (b.type == TGB_BSDF_SMOOTH_COAT || b.type == TGB_BSDF_ROUGH_COAT) {             // SmoothCoatBsdf.cpp:218-223, RoughCoatBsdf.cpp:301-306
            if (b.substrate < 0 || uint32_t(b.substrate) >= d->n_bsdfs || d->bsdfs[b.substrate].type == TGB_BSDF_SMOOTH_COAT ||
                d->bsdfs[b.substrate].type == TGB_BSDF_ROUGH_COAT || d->bsdfs[b.substrate].type == TGB_BSDF_HAIR)
                return fail(c, TGB_ERR_UNSUPPORTED, "bsdf %u: a coat needs a substrate that is neither a coat nor the hair BCSDF", i);
            o.scaled_sigma_a = f3(b.sigma_a)*b.thickness;
            o.avg_transmittance = std::exp(-2.0f*avg(o.scaled_sigma_a));
            o.lobes = (b.type == TGB_BSDF_SMOOTH_COAT ? LOBE_SPEC_R : LOBE_GLOSSY_R) | bsdf_lobes(d->bsdfs[b.substrate]);
        }
        if (b.type == TGB_BSDF_HAIR) {                                                    // bsdfs/HairBcsdf.cpp:422-446
            HairTables ht;
            hair_precompute(b.hair_roughness, b.hair_scale_angle_deg, b.sigma_a, ht);
            for (int p = 0; p < 3; ++p) {
                o.hair_v[p] = ht.v[p];
                int rc = dev_upload(c, &o.hair_table[p], ht.lobe[p].table); if (rc) return rc;
                rc = dev_upload(c, &o.hair_pdfs[p], ht.lobe[p].pdfs); if (rc) return rc;
                rc = dev_upload(c, &o.hair_cdfs[p], ht.lobe[p].cdfs); if (rc) return rc;
                rc = dev_upload(c, &o.hair_sums[p], ht.lobe[p].sums); if (rc) return rc;
            }
            o.hair_scale_rad = ht.scale_angle_rad;
        }
        if (b.type == TGB_BSDF_PLASTIC || b.type == TGB_BSDF_ROUGH_PLASTIC) {             // bsdfs/PlasticBsdf.cpp:179-185
            o.scaled_sigma_a = f3(b.sigma_a)*b.thickness;
            o.avg_transmittance = std::exp(-2.0f*avg(o.scaled_sigma_a));
            o.diffuse_fresnel = diffuse_fresnel(b.ior, 1000000);
            o.substrate_weight = avg(tex[b.albedo_tex].d.avg);                             // RoughPlasticBsdf.cpp:215-222
        }
    }

    // ---- primitives, lights, triangles
    std::vector<DPrim> prims(d->n_primitives);
    std::vector<int> lights, inf_lights, analytic;
    std::vector<BuildTri> btris; std::vector<uint32_t> tri_prim; std::vector<float4> tri_shade;
    std::vector<BuildBox> cboxes; std::vector<IsectRecord> crecs; std::vector<uint32_t> cseg_prim;   // curve BVH primitives (kCurvePieces per segment) of all primitives
    int lightCount = 0;
    for (uint32_t i = 0; i < d->n_primitives; ++i) {
        const tgb_primitive &p = d->primitives[i]; DPrim &o = prims[i];
        std::memset(&o, 0, sizeof(o));
        o.type = p.type; o.emission_tex = p.emission_tex; o.bsdf_first = p.bsdf_first; o.bsdf_count = p.bsdf_count;
        if (p.emission_tex >= int(d->n_textures)) return fail(c, TGB_ERR_INVALID, "primitive %u: bad emission texture", i);
        bool emissive = p.emission_tex >= 0 && max_comp(tex[p.emission_tex].maxv) > 0.0f;  // primitives/Primitive.hpp:111-115
        bool samplable = true, infinite = false;
        if (p.type != TGB_PRIM_INFINITE_SPHERE && p.type != TGB_PRIM_INFINITE_SPHERE_CAP && p.type != TGB_PRIM_SKYDOME) {
            if (p.bsdf_count == 0 || p.bsdf_first + p.bsdf_count > d->n_bsdf_slots) return fail(c, TGB_ERR_INVALID, "primitive %u: bad bsdf range", i);
            for (uint32_t k = 0; k < p.bsdf_count; ++k) if (d->bsdf_slots[p.bsdf_first + k] >= d->n_bsdfs) return fail(c, TGB_ERR_INVALID, "primitive %u: bad bsdf index", i);
            // the hair BCSDF is evaluated in the curve's tangent space (Curves::tangentSpace): on any other primitive the kernels
            // compiled for curve-free scenes would not know the lobe at all
            if (p.type != TGB_PRIM_CURVES)
                for (uint32_t k = 0; k < p.bsdf_count; ++k) {
                    const tgb_bsdf *b = &d->bsdfs[d->bsdf_slots[p.bsdf_first + k]];
                    for (int hop = 0; hop < 4 && b; ++hop) {
                        if (b->type == TGB_BSDF_HAIR) return fail(c, TGB_ERR_UNSUPPORTED, "primitive %u: the hair BCSDF on a primitive that is not `curves` is outside the hot path", i);
                        b = ((b->type == TGB_BSDF_SMOOTH_COAT || b->type == TGB_BSDF_ROUGH_COAT) && b->substrate >= 0 && uint32_t(b->substrate) < d->n_bsdfs) ? &d->bsdfs[b->substrate] : nullptr;
                    }
                }
        }
        switch (p.type) {
        case TGB_PRIM_MESH: {
            if (p.n_tris && (!p.verts || !p.tris)) return fail(c, TGB_ERR_INVALID, "mesh %u has null buffers", i);
            o.tri_first = uint32_t(btris.size()); o.n_tris = p.n_tris;
            if (p.smooth) o.flags |= PF_SMOOTH;
            std::vector<float> areas(p.n_tris), lverts;
            float total = 0.0f;
            for (uint32_t k = 0; k < p.n_tris; ++k) {
                const tgb_triangle &t = p.tris[k];
                if (t.v0 >= p.n_verts || t.v1 >= p.n_verts || t.v2 >= p.n_verts) return fail(c, TGB_ERR_INVALID, "mesh %u: vertex index out of range", i);
                const tgb_vertex &a = p.verts[t.v0], &b = p.verts[t.v1], &cc = p.verts[t.v2];
                BuildTri bt; std::memcpy(bt.v0, a.pos, 12); std::memcpy(bt.v1, b.pos, 12); std::memcpy(bt.v2, cc.pos, 12);
                btris.push_back(bt); tri_prim.push_back(i);
                int mat = std::min(std::max(t.material, 0), int(p.bsdf_count) - 1);      // TriangleMesh.cpp:539
                float4 s0 = make_float4(a.normal[0], a.normal[1], a.normal[2], b.normal[0]);
                float4 s1 = make_float4(b.normal[1], b.normal[2], cc.normal[0], cc.normal[1]);
                float4 s2 = make_float4(cc.normal[2], a.uv[0], a.uv[1], b.uv[0]);
                float4 s3 = make_float4(b.uv[1], cc.uv[0], cc.uv[1], 0.0f);
                if (mat > 1023 || i >= (1u << 22)) return fail(c, TGB_ERR_UNSUPPORTED, "mesh %u: more than 1024 materials in one mesh or more than 4 Mi primitives", i);
                uint32_t packed = uint32_t(mat) | (i << 10);            // material | primitive << 10 (make_surface)
                std::memcpy(&s3.w, &packed, 4);
                tri_shade.push_back(s0); tri_shade.push_back(s1); tri_shade.push_back(s2); tri_shade.push_back(s3);
                V3 p0 = f3(a.pos), p1 = f3(b.pos), p2 = f3(cc.pos);
                areas[k] = length(cross(p1 - p0, p2 - p0))*0.5f;                           // MathUtil::triangleArea
                total += areas[k];                                                         // TriangleMesh.cpp:556-562
                if (emissive) { const float *pp[3] = {a.pos, b.pos, cc.pos}; for (int q = 0; q < 3; ++q) for (int r = 0; r < 3; ++r) lverts.push_back(pp[q][r]); }
            }
            o.total_area = total;
            if (p.n_tris == 0 || p.n_verts == 0) emissive = false;                         // isDirac(): not traced, not a light
            if (emissive) {
                // Distribution1D over triangle areas (TriangleMesh.cpp:389-403; sampling/Distribution1D.hpp:16-35)
                std::vector<float> pdf = areas, cdf(p.n_tris + 1);
                cdf[0] = 0.0f;
                for (uint32_t k = 0; k < p.n_tris; ++k) cdf[k + 1] = cdf[k] + pdf[k];
                float tw = cdf[p.n_tris];
                for (float &x : pdf) x /= tw;
                for (float &x : cdf) x /= tw;
                cdf[p.n_tris] = 1.0f;
                int rc = dev_upload(c, &o.tri_pdf, pdf); if (rc) return rc;
                rc = dev_upload(c, &o.tri_cdf, cdf); if (rc) return rc;
                rc = dev_upload(c, &o.light_verts, lverts); if (rc) return rc;
            }
            break; }
        case TGB_PRIM_QUAD: {                                                             // primitives/Quad.cpp:298-316
            o.base = f3(p.base); o.edge0 = f3(p.edge0); o.edge1 = f3(p.edge1);
            V3 n = cross(o.edge1, o.edge0);
            o.area = length(n);
            o.normal = n/o.area;
            o.inv_uv_sq0 = 1.0f/length_sq(o.edge0); o.inv_uv_sq1 = 1.0f/length_sq(o.edge1);
            analytic.push_back(int(i));
            break; }
        case TGB_PRIM_CUBE: {                                                             // primitives/Cube.cpp:351-367
            o.pos = f3(p.pos); o.scale = f3(p.scale);
            std::memcpy(o.rot, p.rot, sizeof(o.rot)); transpose3(o.rot, o.inv_rot);
            if (emissive) return fail(c, TGB_ERR_UNSUPPORTED, "emissive cubes are outside the hot path");
            analytic.push_back(int(i));
            break; }
        case TGB_PRIM_INFINITE_SPHERE_CAP: {                                              // primitives/InfiniteSphereCap.cpp:231-247
            o.normal = f3(p.cap_dir); o.area = p.cap_cos;
            if (!(p.cap_cos < 1.0f)) return fail(c, TGB_ERR_INVALID, "infinite_sphere_cap %u: cap angle must be positive", i);
            samplable = p.do_sample != 0; infinite = true;
            break; }
        case TGB_PRIM_SKYDOME:                                                            // primitives/Skydome.cpp: an environment sphere with its own prepared image
            if (p.emission_tex < 0 || tex[p.emission_tex].d.type != TGB_TEX_BITMAP) return fail(c, TGB_ERR_INVALID, "skydome %u: pass the prepared sky image (Skydome::prepareForRender) as a bitmap emission texture", i);
            o.type = TGB_PRIM_INFINITE_SPHERE; o.flags |= PF_SKYDOME;
            /* fall through: lookup without rotation (Skydome::directionToUV, Skydome.cpp:29-38) = identity matrices from the caller */
        case TGB_PRIM_INFINITE_SPHERE: {                                                  // primitives/InfiniteSphere.cpp prepareForRender
            std::memcpy(o.rot, p.rot, sizeof(o.rot)); transpose3(o.rot, o.inv_rot);
            if (p.type == TGB_PRIM_SKYDOME) { const float id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; std::memcpy(o.rot, id, sizeof(id)); std::memcpy(o.inv_rot, id, sizeof(id)); }
            samplable = p.do_sample != 0; infinite = true;
            if (emissive && tex[p.emission_tex].d.type == TGB_TEX_CHECKER) return fail(c, TGB_ERR_UNSUPPORTED, "checker environment maps are outside the hot path");
            break; }
        case TGB_PRIM_CURVES: {                                                           // primitives/Curves.cpp:572-613 (nodes arrive prepared)
            if (p.curve_mode > TGB_CURVE_BCSDF_CYLINDER) return fail(c, TGB_ERR_UNSUPPORTED, "curves %u: mode outside the hot path", i);
            if (emissive) return fail(c, TGB_ERR_UNSUPPORTED, "emissive curves are outside the hot path");
            if (p.n_curve_segments && (!p.curve_nodes || !p.curve_segments)) return fail(c, TGB_ERR_INVALID, "curves %u has null buffers", i);
            if (tex[d->bsdfs[d->bsdf_slots[p.bsdf_first]].albedo_tex].d.type != TGB_TEX_CONSTANT)
                return fail(c, TGB_ERR_UNSUPPORTED, "curves %u: textured materials on curves are outside the hot path", i);
            o.curve_mode = p.curve_mode; o.tri_first = uint32_t(cboxes.size()); o.n_tris = p.n_curve_segments*kCurvePieces;   // rebased below
            for (uint32_t k = 0; k < p.n_curve_segments; ++k) {
                uint32_t t = p.curve_segments[k];
                if (t < 2 || t >= p.n_curve_nodes) return fail(c, TGB_ERR_INVALID, "curves %u: segment index out of range", i);
                const float *n0 = p.curve_nodes + 4*size_t(t - 2), *n1 = n0 + 4, *n2 = n0 + 8;
                // One BVH primitive per quarter of the segment's parameter range (the reference bounds the whole segment,
                // curveBox, Curves.cpp:231-243): bounds of the quadratic on [ta, tb] = its end values + the interior extremum,
                // grown by the largest node width (the width spline is a convex combination of the node widths).
                float maxW = std::max(std::max(n0[3], n1[3]), n2[3]);
                for (int piece = 0; piece < kCurvePieces; ++piece) {
                    BuildBox bb;
                    float ta = float(piece)/kCurvePieces, tb = float(piece + 1)/kCurvePieces;
                    for (int a = 0; a < 3; ++a) {
                        float qa = 0.5f*n0[a] - n1[a] + 0.5f*n2[a], qb = n1[a] - n0[a], qc = 0.5f*(n0[a] + n1[a]);
                        float fa = (qa*ta + qb)*ta + qc, fb = (qa*tb + qb)*tb + qc;
                        float lo = std::min(fa, fb), hi = std::max(fa, fb);
                        float tFlat = -qb/(2.0f*qa);
                        if (tFlat > ta && tFlat < tb) { float f = (qa*tFlat + qb)*tFlat + qc; lo = std::min(lo, f); hi = std::max(hi, f); }
                        float slack = 4e-7f*std::max(std::fabs(lo), std::fabs(hi));            // Horner vs the kernel's expanded form
                        bb.lo[a] = lo - maxW - slack; bb.hi[a] = hi + maxW + slack;
                        bb.centroid[a] = 0.5f*(lo + hi);
                    }
                    cboxes.push_back(bb); cseg_prim.push_back(i);
                    IsectRecord rec; std::memcpy(rec.f, n0, sizeof(rec.f));        // n0, n1, n2
                    crecs.push_back(rec);
                }
            }
            break; }
        default: return fail(c, TGB_ERR_UNSUPPORTED, "primitive type %u is outside the hot path", p.type);
        }
        if (emissive) {                                                                   // renderer/TraceableScene.hpp:89-96
            o.flags |= PF_EMISSIVE; lightCount++;
            if (samplable) lights.push_back(int(i));
            if (infinite) inf_lights.push_back(int(i));
        }
        if (samplable) o.flags |= PF_SAMPLABLE;
        if (infinite) o.flags |= PF_INFINITE;
    }
    if (lightCount == 0) {                                                                // renderer/TraceableScene.hpp:97-102
        DPrim o; std::memset(&o, 0, sizeof(o));
        o.type = TGB_PRIM_INFINITE_SPHERE; o.emission_tex = int(d->n_textures);
        o.flags = PF_EMISSIVE | PF_SAMPLABLE | PF_INFINITE;
        const float id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        std::memcpy(o.rot, id, sizeof(id)); std::memcpy(o.inv_rot, id, sizeof(id));
        lights.push_back(int(prims.size())); inf_lights.push_back(int(prims.size()));
        prims.push_back(o);
    }
    for (int li : lights) {
        DPrim &l = prims[li];
        if (l.type == TGB_PRIM_INFINITE_SPHERE_CAP && tex[l.emission_tex].d.type == TGB_TEX_BITMAP)
            return fail(c, TGB_ERR_UNSUPPORTED, "bitmap emission on an infinite_sphere_cap is outside the hot path");
        if (l.type == TGB_PRIM_INFINITE_SPHERE && tex[l.emission_tex].d.type == TGB_TEX_BITMAP && !tex[l.emission_tex].has_dist)
            build_spherical_distribution(d->textures[l.emission_tex], tex[l.emission_tex]);
    }
    std::vector<DTex> dtex(tex.size());
    for (size_t i = 0; i < tex.size(); ++i) {
        if (tex[i].has_dist) {
            int rc = dev_upload(c, &tex[i].d.marg_pdf, tex[i].marg_pdf); if (rc) return rc;
            rc = dev_upload(c, &tex[i].d.marg_cdf, tex[i].marg_cdf); if (rc) return rc;
            rc = dev_upload(c, &tex[i].d.pdf, tex[i].pdf); if (rc) return rc;
            rc = dev_upload(c, &tex[i].d.cdf, tex[i].cdf); if (rc) return rc;
        }
        dtex[i] = tex[i].d;
    }

    // ---- BVH over every mesh triangle, curve piece and -- only when they are many -- analytic primitive.
    // Analytic quads/cubes are few in most scenes and are then tested coherently by the kernel that creates a ray; from
    // TGB_ANALYTIC_BVH_MIN (24) primitives on they get a third SAH tree instead (the reference keeps them in Embree's top-level
    // user-geometry BVH, renderer/TraceableScene.hpp:112-134), so a ray's cost no longer grows with their number.
    size_t analytic_bvh_min = 24;
    if (const char *e = getenv("TGB_ANALYTIC_BVH_MIN")) analytic_bvh_min = size_t(std::max(1, atoi(e)));
    const bool analytic_in_bvh = analytic.size() >= analytic_bvh_min;
    std::vector<Aabb> abounds(analytic.size());
    for (size_t k = 0; k < analytic.size(); ++k) abounds[k] = analytic_bounds(prims[size_t(analytic[k])]);
    SceneBvhInput in;
    in.tris = btris.data(); in.n_tris = uint32_t(btris.size());
    in.curve_boxes = cboxes.data(); in.curve_recs = crecs.data(); in.n_curve = uint32_t(cboxes.size());
    if (analytic_in_bvh) { in.analytic = abounds.data(); in.n_analytic = uint32_t(abounds.size()); }
    in.extent = std::max(std::max(std::fabs(sc.cam.pos.x), std::fabs(sc.cam.pos.y)), std::fabs(sc.cam.pos.z));
    SceneBvh sb;
    build_scene_bvh(in, bvh_options(), sb);
    const Bvh4 &bvh = sb.tree;
    if (!cboxes.empty()) {
        for (uint32_t pi : cseg_prim) tri_prim.push_back(pi);
        for (DPrim &p : prims) if (p.type == TGB_PRIM_CURVES) p.tri_first += uint32_t(btris.size());
    }
    std::vector<int> analytic_loop = analytic;           // what the ray-creating kernels loop over
    if (analytic_in_bvh)                                  // ... nothing: the list goes into BVH leaf order instead
        for (size_t k = 0; k < sb.analytic_order.size(); ++k) analytic_loop[k] = analytic[sb.analytic_order[k]];
    {   // ray-binning grid: bounds of every finite primitive (TraceableScene::_sceneBounds, TraceableScene.hpp:104-110)
        float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
        auto grow = [&](const float *p) { for (int a = 0; a < 3; ++a) { lo[a] = std::min(lo[a], p[a]); hi[a] = std::max(hi[a], p[a]); } };
        if (!bvh.nodes.empty()) { grow(bvh.lo); grow(bvh.hi); }
        for (const Aabb &b : abounds) { grow(b.lo); grow(b.hi); }
        for (int a = 0; a < 3; ++a) if (!(hi[a] > lo[a])) { lo[a] = -1.0f; hi[a] = 1.0f; }
        sc.bin_lo = v3(lo[0], lo[1], lo[2]);
        sc.bin_inv = v3(16.0f/(hi[0] - lo[0]), 16.0f/(hi[1] - lo[1]), 16.0f/(hi[2] - lo[2]));
    }
    sc.n_cut = int(sb.cut.size());
    for (int i = 0; i < sc.n_cut; ++i) {
        for (int a = 0; a < 3; ++a) { sc.cut[2*a][i] = sb.cut[size_t(i)].lo[a]; sc.cut[2*a + 1][i] = sb.cut[size_t(i)].hi[a]; }
        sc.cut_link[i] = sb.cut[size_t(i)].link;
    }
    {
        const char *e = getenv("TGB_SHADOW_CUT_ENTRY");
        sc.cut_entry = (e && e[0] == '0') ? 0 : 1;
    }
    if (sb.stack_need > uint32_t(kStackSize)) return fail(c, TGB_ERR_UNSUPPORTED, "BVH depth %u (%u stack entries) exceeds the traversal stack", bvh.max_depth, sb.stack_need);
    c->bvh_depth = bvh.max_depth; c->n_tris = uint32_t(btris.size()); c->bvh_sah = bvh.sah_cost;
    c->geom_bytes = sb.qtree.nodes.size()*sizeof(QNode4) + sb.isect.size()*sizeof(IsectRecord) + tri_shade.size()*16 + bvh.order.size()*8;

    int rc;
    if ((rc = dev_upload(c, &sc.prims, prims))) return rc;
    if ((rc = dev_upload(c, &sc.bsdfs, bsdfs))) return rc;
    c->n_bsdfs = int(bsdfs.size());
    c->prim_types.resize(prims.size());
    for (size_t i = 0; i < prims.size(); ++i) c->prim_types[i] = prims[i].type;
    c->light_ids = lights;
    for (int li : lights) c->mesh_lights = c->mesh_lights || prims[size_t(li)].type == TGB_PRIM_MESH;
    std::vector<uint32_t> slots(d->bsdf_slots, d->bsdf_slots + d->n_bsdf_slots);
    if ((rc = dev_upload(c, &sc.slots, slots))) return rc;
    if ((rc = dev_upload(c, &sc.tex, dtex))) return rc;
    if ((rc = dev_upload(c, &sc.lights, lights))) return rc;
    if ((rc = dev_upload(c, &sc.inf_lights, inf_lights))) return rc;
    if ((rc = dev_upload(c, &sc.analytic, analytic_loop))) return rc;
    if ((rc = dev_upload(c, &sc.tri_global, bvh.order))) return rc;
    if ((rc = dev_upload(c, &sc.tri_prim, tri_prim))) return rc;
    {   // shading records follow the intersection records into BVH leaf order (one hop from a hit id)
        std::vector<float4> shade_leaf(tri_shade.size());
        for (size_t k = 0; k < btris.size(); ++k) std::memcpy(&shade_leaf[4*k], &tri_shade[4*size_t(bvh.order[k])], 4*sizeof(float4));
        if ((rc = dev_upload(c, &sc.tri_shade, shade_leaf))) return rc;
    }
    {
        static_assert(sizeof(IsectRecord) == 3*sizeof(float4), "intersection record layout");
        const IsectRecord *ir = nullptr;
        if ((rc = dev_upload(c, &ir, sb.isect))) return rc;
        sc.tri_isect = reinterpret_cast<const float4 *>(ir);
    }
    {
        const QNode4 *qn = nullptr;
        if ((rc = dev_upload(c, &qn, sb.qtree.nodes))) return rc;
        sc.qnodes = reinterpret_cast<const uint4 *>(qn); sc.qy = 0x3F80u;
    }
    std::vector<uint32_t> sobol(1024*32);
    std::memcpy(sobol.data(), tgb_sobol_blob, sobol.size()*4);
    if ((rc = dev_upload(c, &sc.sobol, sobol))) return rc;
    sc.n_prims = uint32_t(prims.size()); sc.n_lights = int(lights.size()); sc.n_inf_lights = int(inf_lights.size());
    sc.n_analytic = analytic_in_bvh ? 0 : int(analytic.size()); sc.analytic_base = analytic_in_bvh ? int(sb.isect.size()) : 0x7fffffff;
    sc.n_nodes = uint32_t(bvh.nodes.size()); sc.n_tris = uint32_t(btris.size());
    sc.n_curve_segs = uint32_t(cboxes.size()); c->has_curves = !cboxes.empty();
    {
        uint32_t types = 0;
        for (uint32_t i = 0; i < d->n_primitives; ++i) {
            const tgb_primitive &p = d->primitives[i];
            if (p.type == TGB_PRIM_INFINITE_SPHERE || p.type == TGB_PRIM_INFINITE_SPHERE_CAP || p.type == TGB_PRIM_SKYDOME) continue;
            for (uint32_t k = 0; k < p.bsdf_count; ++k) {
                uint32_t t = d->bsdfs[d->bsdf_slots[p.bsdf_first + k]].type;
                if (t != TGB_BSDF_NULL) types |= 1u << std::min(t, 31u);
            }
        }
        const char *env = getenv("TGB_SORT_MATERIALS");
        c->sort_materials = env ? env[0] == '1' : __builtin_popcount(types) >= 2;
        // every surface Lambert (lights: null BSDF): k_shade's lobe-set-1 instantiation (same arithmetic, a fraction of the code)
        const char *ls = getenv("TGB_LOBE_SET");
        c->diffuse_only = (types & ~(1u << TGB_BSDF_LAMBERT)) == 0 && !c->has_curves && !(ls && ls[0] == '0');
        if (c->diffuse_only) c->sort_materials = false;
    }
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
        CU(cudaMallocHost(reinterpret_cast<void **>(&w.h_ctl), 5*sizeof(Ctl)));
    }
    if ((rc = dev_alloc(c, &c->ctr, 1))) return rc;
    CU(cudaMemset(c->ctr, 0, sizeof(Counters)));
    CU(cudaMallocHost(reinterpret_cast<void **>(&c->h_ctr), sizeof(Counters)));
    size_t npx = size_t(c->res_x)*c->res_y;
    if ((rc = dev_alloc(c, &c->fb, npx*3))) return rc;
    if ((rc = dev_alloc(c, &c->fb_count, npx))) return rc;
    CU(cudaMemset(c->fb, 0, npx*3*sizeof(float)));
    CU(cudaMemset(c->fb_count, 0, npx*sizeof(uint32_t)));
    CU(cudaMallocHost(reinterpret_cast<void **>(&c->h_fb), npx*3*sizeof(float)));
    CU(cudaMallocHost(reinterpret_cast<void **>(&c->h_fb_count), npx*sizeof(uint32_t)));
    return TGB_OK;
}

// PathTraceIntegrator::diceTiles + the sampler seeding of prepareForRender (PathTraceIntegrator.cpp:27-42,187)
void dice_tiles(uint32_t w, uint32_t h, uint32_t seed, std::vector<tgb_tile> &out) {
    const uint32_t TileSize = 16;
    uint64_t st = uint64_t(hash32(seed));
    out.clear();
    for (uint32_t y = 0; y < h; y += TileSize)
        for (uint32_t x = 0; x < w; x += TileSize) {
            tgb_tile t; t.x = x; t.y = y; t.w = std::min(TileSize, w - x); t.h = std::min(TileSize, h - y);
            t.sampler_seed = hash32(pcg_next(st));
            out.push_back(t);
        }
}

int set_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed) {
    std::vector<tgb_tile> own;
    if (n_tiles == 0) { dice_tiles(c->res_x, c->res_y, seed, own); tiles = own.data(); n_tiles = uint32_t(own.size()); }
    if (c->tiles_cached.size() == n_tiles && n_tiles && std::memcmp(c->tiles_cached.data(), tiles, n_tiles*sizeof(tgb_tile)) == 0) return TGB_OK;
    std::vector<uint32_t> pid, pseed;
    for (uint32_t t = 0; t < n_tiles; ++t) {
        const tgb_tile &tl = tiles[t];
        if (tl.x >= c->res_x || tl.w > c->res_x - tl.x || tl.y >= c->res_y || tl.h > c->res_y - tl.y) return fail(c, TGB_ERR_INVALID, "tile %u lies outside the image", t);
        for (uint32_t y = 0; y < tl.h; ++y) for (uint32_t x = 0; x < tl.w; ++x) { pid.push_back((tl.x + x) + (tl.y + y)*c->res_x); pseed.push_back(tl.sampler_seed); }
    }
    {   // tiles must be disjoint: k_resolve owns one pixel per thread
        std::vector<bool> seen(size_t(c->res_x)*c->res_y, false);
        for (uint32_t q : pid) { if (seen[q]) return fail(c, TGB_ERR_INVALID, "tile list covers pixel %u twice", q); seen[q] = true; }
    }
    if (pid.size() > c->pix_capacity) {
        int rc;
        if ((rc = dev_alloc(c, &c->pix_id, pid.size()))) return rc;
        if ((rc = dev_alloc(c, &c->pix_seed, pid.size()))) return rc;
        c->pix_capacity = uint32_t(pid.size());
    }
    c->n_pix = uint32_t(pid.size());
    c->h_pix_id = pid; c->pix_slot_valid = false;
    if (c->n_pix) {
        CU(cudaMemcpyAsync(c->pix_id, pid.data(), pid.size()*4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaMemcpyAsync(c->pix_seed, pseed.data(), pseed.size()*4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    c->tiles_cached.assign(tiles, tiles + n_tiles);
    return TGB_OK;
}

inline unsigned blocks(uint32_t n, unsigned bs) { return n ? (n + bs - 1)/bs : 1; }

// The wavefront loop: the GPU analogue of renderTile over (pixels of the tiles) x (sample range), with path
// regeneration: whenever paths finish, their slots are refilled with the next camera paths of the step, so every
// iteration traces a full batch until the step's paths run out (one drain tail per step instead of one per batch).
int ensure_results(tgb_ctx *c, size_t n_paths) {
    if (n_paths <= c->res_capacity) return TGB_OK;
    if (c->R) cudaFree(c->R);
    c->R = nullptr; c->res_capacity = 0;
    for (Wavefront &w : c->wf) w.sr.R = nullptr;
    CU(cudaMalloc(reinterpret_cast<void **>(&c->R), n_paths*sizeof(float4)));
    c->res_capacity = n_paths;
    for (Wavefront &w : c->wf) w.sr.R = c->R;
    return TGB_OK;
}

// k_shadow_bvh over the any-hit queue and (scenes with mesh lights) the closest-hit queue
void launch_shadow_bvh(tgb_ctx *c, const Wavefront &w, cudaStream_t st, uint32_t grid) {
    const DScene &sc = c->sc;
    if (c->has_curves) {
        if (c->mesh_lights) k_shadow_bvh<true, true><<<grid, kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
        else k_shadow_bvh<true, false><<<grid, kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
    } else {
        if (c->mesh_lights) k_shadow_bvh<false, true><<<grid, kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
        else k_shadow_bvh<false, false><<<grid, kTraceBlock, 0, st>>>(sc, w.sr, w.squeue2, w.squeue_cl, w.ctl, c->ctr);
    }
}

// k_trace, k_shade and k_shadow_prep of wavefront w over the paths of pb, in the instantiations the context renders with (also
// tgb200_bounce_probe's).  `bound` >= ctl.n: an upper bound of the paths.
void launch_trace(tgb_ctx *c, const Wavefront &w, const PathBuf &pb, cudaStream_t st, uint32_t bound) {
    const uint32_t grid = std::min(blocks(bound, kTraceBlock), c->persist_blocks);
    if (c->has_curves) k_trace<true><<<grid, kTraceBlock, 0, st>>>(c->sc, pb, w.order, w.ctl);
    else k_trace<false><<<grid, kTraceBlock, 0, st>>>(c->sc, pb, w.order, w.ctl);
}
void launch_shade(tgb_ctx *c, const Wavefront &w, const PathBuf &pb, cudaStream_t st, const BatchInfo &bi, uint32_t bound) {
    const DScene &sc = c->sc; const bool curves = c->has_curves;
    if (c->sort_materials) {
        if (curves) k_shade<true, true><<<blocks(bound, kShadeSortBlock*kShadeSortItems), kShadeSortBlock, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
        else k_shade<false, true><<<blocks(bound, kShadeSortBlock*kShadeSortItems), kShadeSortBlock, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
    } else {
        if (curves) k_shade<true, false><<<blocks(bound, 128), 128, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
        else if (c->diffuse_only) k_shade<false, false, 1><<<blocks(bound, 128), 128, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
        else k_shade<false, false><<<blocks(bound, 128), 128, 0, st>>>(sc, pb, w.sr, bi, w.ctl, w.squeue, c->ctr);
    }
}
void launch_shadow_prep(tgb_ctx *c, const Wavefront &w, cudaStream_t st, uint32_t bound) {
    if (c->has_curves) k_shadow_prep<true><<<blocks(2*bound, 256), 256, 0, st>>>(c->sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
    else k_shadow_prep<false><<<blocks(2*bound, 256), 256, 0, st>>>(c->sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
}

// One iteration's kernels of wavefront w on stream st.  `bound` >= the iteration's ctl.n: grids are upper bounds, the kernels
// read the real sizes from the device-resident control block.
void enqueue_iteration(tgb_ctx *c, Wavefront &w, cudaStream_t st, const BatchInfo &bi, int cur, uint32_t bound, int slot, uint64_t &launches) {
    const DScene &sc = c->sc;
    const bool has_bvh = sc.n_nodes != 0;
    PathBuf &pb = w.pb[cur], &nxt = w.pb[cur ^ 1];
    const bool prof = c->profiling;
    if (prof) cudaEventRecord(w.ev_k[slot][0], st);
    k_regen<<<blocks(bound, 256), 256, 0, st>>>(sc, pb, bi, w.ctl, w.order, w.bin_hist); launches++;
    if (prof) cudaEventRecord(w.ev_k[slot][1], st);
    if (has_bvh) { launch_trace(c, w, pb, st, bound); launches++; }
    if (prof) cudaEventRecord(w.ev_k[slot][2], st);
    launch_shade(c, w, pb, st, bi, bound); launches++;
    if (prof) cudaEventRecord(w.ev_k[slot][3], st);
    launch_shadow_prep(c, w, st, bound); launches++;
    if (prof) cudaEventRecord(w.ev_k[slot][4], st);
    if (has_bvh) { launch_shadow_bvh(c, w, st, std::min(blocks(2*bound, kTraceBlock), c->persist_blocks)); launches++; }
    if (prof) cudaEventRecord(w.ev_k[slot][5], st);
    k_accum<<<blocks(bound, 256), 256, 0, st>>>(sc, pb, nxt, w.sr, bi, w.ctl, w.bin_keys, w.bin_hist); launches++;
    if (prof) cudaEventRecord(w.ev_k[slot][6], st);
    k_iter_end<<<1, 1024, 0, st>>>(w.bin_hist, w.ctl, has_bvh ? 1 : 0); launches++;
    if (has_bvh) { k_bin_scatter<<<blocks(bound, 256), 256, 0, st>>>(w.bin_keys, w.bin_hist, w.ctl, w.order); launches++; }
    if (prof) cudaEventRecord(w.ev_k[slot][7], st);
}

// `adaptive`: per-pixel sample ranges come from c->pix_first / c->pix_base (tgb200_render_adaptive), else every pixel
// renders samples [spp_begin, spp_begin + spp_count).
int render_device(tgb_ctx *c, uint32_t spp_begin, uint32_t spp_count, bool adaptive = false, uint32_t adaptive_total = 0) {
    if (c->n_pix == 0 || (!adaptive && spp_count == 0) || (adaptive && adaptive_total == 0)) return TGB_OK;
    CU(cudaEventRecord(c->ev0, c->stream));
    uint64_t launches = 0;
    float trace_ms = 0.0f, shadow_ms = 0.0f; uint64_t trace_launches = 0, shadow_launches = 0, traversed = 0, shadow_traversed = 0;
    double kms[7] = {0, 0, 0, 0, 0, 0, 0}; uint64_t iterations = 0;
    // a step's finished radiances are kept per path (16 B each) until k_resolve folds them in sample order;
    // split the sample range so that this buffer stays below 8 GB and (sample within the call, pixel) fits 32 bits
    uint32_t pix_bits = 0; while (pix_bits < 32 && (uint64_t(1) << pix_bits) < uint64_t(c->n_pix)) ++pix_bits;
    const uint64_t max_k = uint64_t(1) << (32 - pix_bits);
    const uint64_t max_paths = 512ull << 20;
    uint32_t spp_sub = adaptive ? 1u : uint32_t(std::max<uint64_t>(1, std::min<uint64_t>(std::min<uint64_t>(spp_count, max_k), max_paths/c->n_pix)));
    if (uint64_t(c->n_pix)*spp_sub > 0xFFFFFFFFull) return fail(c, TGB_ERR_UNSUPPORTED, "tile list too large");
    if (adaptive) spp_count = 1;                               // one pass over the per-pixel ranges
    const bool trace_bounces = getenv("TGB_TRACE_BOUNCES") != nullptr;
    uint64_t samples_done = 0;
    for (uint32_t s0 = 0; s0 < spp_count; s0 += spp_sub) {
        uint32_t ns = std::min(spp_sub, spp_count - s0);
        uint32_t total = adaptive ? adaptive_total : c->n_pix*ns;
        samples_done += total;
        int rc = ensure_results(c, total);
        if (rc) return rc;
        BatchInfo bi; bi.pix_id = c->pix_id; bi.pix_seed = c->pix_seed; bi.n_pix = c->n_pix; bi.spp_begin = spp_begin + s0;
        bi.pix_first = adaptive ? c->pix_first : nullptr; bi.pix_base = adaptive ? c->pix_base : nullptr; bi.pix_bits = pix_bits;
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
            Ctl &init = w.h_ctl[4];
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
                CU(cudaMemcpyAsync(&w.h_ctl[slot], w.ctl, sizeof(Ctl), cudaMemcpyDeviceToHost, st[h]));
                CU(cudaEventRecord(w.ev_ring[slot], st[h]));
            }
            if (iter == 0) continue;                          // nothing known yet about iteration 1: its bound stays the first one
            const int p = int((iter - 1) & 3u);
            for (int h = 0; h < 2; ++h) {
                if (!live[h]) continue;
                Wavefront &w = c->wf[h];
                CU(cudaEventSynchronize(w.ev_ring[p]));
                const Ctl S = w.h_ctl[p];                     // state after iteration iter-1 = the sizes of iteration iter
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
        k_resolve<<<blocks(c->n_pix, 256), 256, 0, st[0]>>>(c->R, bi, ns, c->fb, c->fb_count); launches++;
    }
    CU(cudaEventRecord(c->ev1, c->stream));
    CU(cudaMemcpyAsync(c->h_ctr, c->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
    float ms = 0.0f; cudaEventElapsedTime(&ms, c->ev0, c->ev1);
    c->stats.samples += samples_done;
    c->stats.path_rays = c->h_ctr->rays; c->stats.shadow_rays = c->h_ctr->shadow_rays;
    c->stats.rays = c->h_ctr->rays + c->h_ctr->shadow_rays; c->stats.hits = c->h_ctr->hits + c->h_ctr->shadow_hits;
    trace_ms = float(kms[1]); shadow_ms = float(kms[4]);
    c->stats.regen_ms += kms[0]; c->stats.shade_ms += kms[2]; c->stats.prep_ms += kms[3]; c->stats.accum_ms += kms[5]; c->stats.sort_ms += kms[6];
    c->stats.iterations += iterations;
    c->stats.shadow_ms += shadow_ms; c->stats.shadow_launches += shadow_launches;
    c->stats.kernel_launches += launches;
    c->stats.path_rays_traversed += traversed; c->stats.shadow_rays_traversed += shadow_traversed;
    c->stats.total_ms += ms; c->stats.trace_ms += trace_ms; c->stats.trace_launches += trace_launches;
    return TGB_OK;
}

// apply f to every member of a multi-GPU context (the root last, so that the current device ends up being the root's)
template <class F> int for_members(tgb_ctx *c, F f) {
    if (!c->group) return TGB_OK;
    Group *g = c->group;
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

int single_render_resident(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count);
int single_render_adaptive(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, tgb_sample_record *records);

// Deal the call's tiles to the members (Morton order, round-robin) and make sure the root knows every share's pixel list.
int group_deal(tgb_ctx *root, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed) {
    tgb_ctx *c = root; Group &g = *root->group;
    std::vector<tgb_tile> own;
    if (n_tiles == 0) { dice_tiles(root->res_x, root->res_y, seed, own); tiles = own.data(); n_tiles = uint32_t(own.size()); }
    if (g.deal_key.size() == n_tiles && n_tiles && std::memcmp(g.deal_key.data(), tiles, n_tiles*sizeof(tgb_tile)) == 0) return TGB_OK;
    const size_t N = g.members.size();
    std::vector<uint32_t> order; shard_order(tiles, n_tiles, order);
    g.shares.assign(N, {});
    for (uint32_t i = 0; i < n_tiles; ++i) g.shares[i % N].push_back(tiles[order[i]]);
    CU(cudaSetDevice(root->device));
    for (uint32_t *p : g.root_pix) if (p) cudaFree(p);
    g.root_pix.assign(N, nullptr); g.share_pixels.assign(N, 0);
    size_t max_share = 0;
    for (size_t k = 0; k < N; ++k) {
        std::vector<uint32_t> pid;
        for (const tgb_tile &tl : g.shares[k]) {
            if (tl.x >= root->res_x || tl.w > root->res_x - tl.x || tl.y >= root->res_y || tl.h > root->res_y - tl.y) return fail(c, TGB_ERR_INVALID, "tile lies outside the image");
            for (uint32_t y = 0; y < tl.h; ++y) for (uint32_t x = 0; x < tl.w; ++x) pid.push_back((tl.x + x) + (tl.y + y)*root->res_x);
        }
        g.share_pixels[k] = uint32_t(pid.size());
        max_share = std::max(max_share, pid.size());
        if (k >= 1 && !pid.empty()) {
            CU(cudaMalloc(reinterpret_cast<void **>(&g.root_pix[k]), pid.size()*4));
            CU(cudaMemcpy(g.root_pix[k], pid.data(), pid.size()*4, cudaMemcpyHostToDevice));
        }
    }
    if (max_share > g.recv_capacity) {
        if (g.recv) cudaFree(g.recv);
        g.recv = nullptr; g.recv_capacity = 0;
        CU(cudaMalloc(reinterpret_cast<void **>(&g.recv), max_share*sizeof(float4)));
        g.recv_capacity = max_share;
    }
    g.send.resize(N, nullptr); g.send_capacity.resize(N, 0);
    for (size_t k = 1; k < N; ++k) {
        if (g.share_pixels[k] > g.send_capacity[k]) {
            tgb_ctx *m = g.members[k];
            if (cudaSetDevice(m->device) != cudaSuccess) return fail(c, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", m->device);
            if (g.send[k]) cudaFree(g.send[k]);
            g.send[k] = nullptr; g.send_capacity[k] = 0;
            if (cudaMalloc(reinterpret_cast<void **>(&g.send[k]), size_t(g.share_pixels[k])*sizeof(float4)) != cudaSuccess) return fail(c, TGB_ERR_OOM, "gather buffer allocation failed on device %d", m->device);
            g.send_capacity[k] = g.share_pixels[k];
        }
    }
    g.deal_key.assign(tiles, tiles + n_tiles); g.deal_seed = seed;
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
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CU(cudaEventCreate(&e0)); CU(cudaEventCreate(&e1));
    CU(cudaEventRecord(e0, root->stream));
    for (size_t k = 1; k < N; ++k) {
        tgb_ctx *m = g.members[k];
        const uint32_t np = g.share_pixels[k];
        if (!np) continue;
        if (cudaSetDevice(m->device) != cudaSuccess) return fail(c, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", m->device);
        k_pack_share<<<blocks(np, 256), 256, 0, m->stream>>>(m->pix_id, np, m->fb, m->fb_count, g.send[k]);
        m->stats.kernel_launches++;
        cudaError_t e = cudaStreamSynchronize(m->stream);
        if (e != cudaSuccess) return fail(c, TGB_ERR_CUDA, "pack on device %d failed: %s", m->device, cudaGetErrorString(e));
        CU(cudaSetDevice(root->device));
        CU(cudaMemcpyPeerAsync(g.recv, root->device, g.send[k], m->device, size_t(np)*sizeof(float4), root->stream));
        k_unpack_share<<<blocks(np, 256), 256, 0, root->stream>>>(g.root_pix[k], np, g.recv, root->fb, root->fb_count);
        root->stats.kernel_launches++;
    }
    CU(cudaSetDevice(root->device));
    CU(cudaEventRecord(e1, root->stream));
    CU(cudaStreamSynchronize(root->stream));
    float ms = 0.0f; cudaEventElapsedTime(&ms, e0, e1); g.gather_ms += ms;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    CU(cudaGetLastError());
    return TGB_OK;
}

}  // namespace

extern "C" {

uint32_t tgb200_abi_version(void) { return TGB200_ABI_VERSION; }

const char *tgb200_last_error(const tgb_ctx *ctx) { return ctx ? ctx->error.c_str() : g_create_error.c_str(); }

void tgb200_destroy(tgb_ctx *c) {
    if (!c) return;
    if (c->group) {
        Group *g = c->group; c->group = nullptr;
        cudaSetDevice(c->device);
        for (uint32_t *p : g->root_pix) if (p) cudaFree(p);
        if (g->recv) cudaFree(g->recv);
        for (size_t k = 1; k < g->members.size(); ++k) {
            cudaSetDevice(g->members[k]->device);
            if (k < g->send.size() && g->send[k]) cudaFree(g->send[k]);
            tgb200_destroy(g->members[k]);
        }
        delete g;
    }
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->stream1) cudaStreamSynchronize(c->stream1);
    for (void *p : c->allocs) cudaFree(p);
    if (c->R) cudaFree(c->R);
    if (c->h_ctr) cudaFreeHost(c->h_ctr);
    if (c->h_fb) cudaFreeHost(c->h_fb);
    if (c->h_fb_count) cudaFreeHost(c->h_fb_count);
    for (cudaEvent_t e : {c->ev0, c->ev1, c->ev_fork, c->ev_join}) if (e) cudaEventDestroy(e);
    for (Wavefront &w : c->wf) {
        if (w.h_ctl) cudaFreeHost(w.h_ctl);
        for (int k = 0; k < 4; ++k) { if (w.ev_ring[k]) cudaEventDestroy(w.ev_ring[k]); for (cudaEvent_t e : w.ev_k[k]) if (e) cudaEventDestroy(e); }
    }
    if (c->stream1) cudaStreamDestroy(c->stream1);
    if (c->own_stream) cudaStreamDestroy(c->own_stream);
    delete c;
}

static int create_single(const tgb_scene_desc *d, tgb_ctx **out);

int tgb200_create(const tgb_scene_desc *d, tgb_ctx **out) {
    if (!d || !out) return fail(nullptr, TGB_ERR_INVALID, "null argument");
    *out = nullptr;
    const uint32_t N = d->settings.n_devices;
    if (N <= 1) {
        tgb_scene_desc one = *d;
        if (N == 1) one.settings.device = d->settings.devices[0];
        one.settings.n_devices = 0;
        return create_single(&one, out);
    }
    if (N > 8) return fail(nullptr, TGB_ERR_INVALID, "at most 8 devices");
    for (uint32_t i = 0; i < N; ++i) for (uint32_t j = 0; j < i; ++j)
        if (d->settings.devices[i] == d->settings.devices[j]) return fail(nullptr, TGB_ERR_INVALID, "device %d listed twice", d->settings.devices[i]);
    // one context per GPU, created concurrently (each uploads its own replica of the scene; the host BVH build runs per member)
    std::vector<tgb_ctx *> members(N, nullptr); std::vector<int> rcs(N, TGB_OK); std::vector<std::string> errs(N);
    std::vector<std::thread> th;
    for (uint32_t k = 0; k < N; ++k) th.emplace_back([&, k] {
        tgb_scene_desc one = *d; one.settings.device = d->settings.devices[k]; one.settings.n_devices = 0;
        rcs[k] = create_single(&one, &members[k]);
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
    root->group = new Group();
    root->group->members = members;
    *out = root;
    return TGB_OK;
}

static int create_single(const tgb_scene_desc *d, tgb_ctx **out) {
    tgb_ctx *c = nullptr;
    *out = nullptr;
    if (d->abi_version != TGB200_ABI_VERSION) return fail(nullptr, TGB_ERR_INVALID, "ABI version mismatch (got %u, library is %u)", d->abi_version, TGB200_ABI_VERSION);
    if (!d->settings.use_sobol) return fail(nullptr, TGB_ERR_UNSUPPORTED, "only the Sobol sampler (renderer.stratified_sampler = true) is on the hot path");
    if (d->settings.supplemental_mode != 0) return fail(nullptr, TGB_ERR_UNSUPPORTED, "supplemental_mode %u: the per-tile serial PCG stream cannot be reproduced by a wavefront renderer (DESIGN.md section 3)", d->settings.supplemental_mode);
    if (d->camera.res_x == 0 || d->camera.res_y == 0) return fail(nullptr, TGB_ERR_INVALID, "empty image");
    // max_bounces 0: PathTracer::traceSample's loop never runs and every sample is black; the wavefront's first shade would add
    // bounce-0 emission, so the setting is refused rather than rendered differently
    if (d->settings.max_bounces > 255 || d->settings.max_bounces < 1) return fail(nullptr, TGB_ERR_UNSUPPORTED, "max_bounces must be in [1, 255]");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(nullptr, TGB_ERR_NO_DEVICE, "no CUDA device available (this library has no CPU fallback)"); }
    int dev = d->settings.device;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    if (dev >= ndev) return fail(nullptr, TGB_ERR_NO_DEVICE, "CUDA device %d not present (%d devices)", dev, ndev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return fail(nullptr, TGB_ERR_NO_DEVICE, "cannot query device %d", dev);
    if (prop.major != 9 || prop.minor != 0) return fail(nullptr, TGB_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only", dev, prop.major, prop.minor);
    c = new tgb_ctx();
    c->device = dev;
    int rc = TGB_OK;
    do {
        if (cudaSetDevice(dev) != cudaSuccess) { rc = fail(c, TGB_ERR_CUDA, "cudaSetDevice(%d) failed", dev); break; }
        if (cudaStreamCreateWithFlags(&c->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaStreamCreateWithFlags(&c->stream1, cudaStreamNonBlocking) != cudaSuccess) { rc = fail(c, TGB_ERR_CUDA, "cudaStreamCreate failed"); break; }
        c->stream = c->own_stream;
        for (cudaEvent_t *e : {&c->ev0, &c->ev1}) cudaEventCreate(e);
        for (cudaEvent_t *e : {&c->ev_fork, &c->ev_join}) cudaEventCreateWithFlags(e, cudaEventDisableTiming);
        for (Wavefront &w : c->wf)
            for (int k = 0; k < 4; ++k) {
                cudaEventCreateWithFlags(&w.ev_ring[k], cudaEventDisableTiming);
                for (cudaEvent_t &e : w.ev_k[k]) cudaEventCreate(&e);
            }
        if ((rc = upload_scene(c, d))) break;
        // default: 2 x 4 Mi paths in flight (H100, C1: 2 x 2 Mi measured 3 % slower)
        uint32_t cap = d->settings.max_paths_in_flight ? d->settings.max_paths_in_flight : (1u << 23);
        cap = std::max(cap, 1024u);
        if ((rc = alloc_wavefront(c, cap))) break;
        {   // persistent traversal grid of one wavefront: what is resident at once (blocks per SM x SMs, smaller of the two
            // kernels), or TGB_TRAVERSAL_BLOCKS per SM.  H100, C1: 6 (resident) > 4 > 12 (twice resident) > 3 blocks per SM.
            int sms = 0, b1 = 0, b2 = 0;
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
            cudaError_t e = cudaSuccess;
            auto prep = [&](auto kern, int *nb) {
                if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(nb, kern, kTraceBlock, 0);
            };
            if (c->has_curves) { prep(k_trace<true>, &b1); prep(c->mesh_lights ? k_shadow_bvh<true, true> : k_shadow_bvh<true, false>, &b2); }
            else { prep(k_trace<false>, &b1); prep(c->mesh_lights ? k_shadow_bvh<false, true> : k_shadow_bvh<false, false>, &b2); }
            if (e != cudaSuccess || sms <= 0 || b1 <= 0 || b2 <= 0) { rc = fail(c, TGB_ERR_CUDA, "traversal kernels cannot be resident (%s)", cudaGetErrorString(e)); break; }
            const char *per_sm = getenv("TGB_TRAVERSAL_BLOCKS");
            c->persist_blocks = uint32_t(sms)*uint32_t(per_sm ? std::max(1, atoi(per_sm)) : std::min(b1, b2));
        }
    } while (0);
    if (rc) { g_create_error = c->error; tgb200_destroy(c); return rc; }
    *out = c;
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
}  // extern "C"
namespace {
int single_render_resident(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count) {
    CU(cudaSetDevice(c->device));
    int rc = set_tiles(c, tiles, n_tiles, seed);
    if (rc) return rc;
    return render_device(c, spp_begin, spp_count);
}
}  // namespace
extern "C" {

int tgb200_read_framebuffer(tgb_ctx *c, float *rgb_mean, uint32_t *count) {
    if (!c || !rgb_mean) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    size_t npx = size_t(c->res_x)*c->res_y;
    CU(cudaMemcpyAsync(c->h_fb, c->fb, npx*3*sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    if (count) CU(cudaMemcpyAsync(c->h_fb_count, c->fb_count, npx*sizeof(uint32_t), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    std::memcpy(rgb_mean, c->h_fb, npx*3*sizeof(float));
    if (count) std::memcpy(count, c->h_fb_count, npx*sizeof(uint32_t));
    return TGB_OK;
}

int tgb200_render_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, uint32_t spp_begin, uint32_t spp_count,
                        float *rgb_mean, uint32_t *count) {
    if (!c || !rgb_mean) return c ? fail(c, TGB_ERR_INVALID, "null framebuffer") : TGB_ERR_INVALID;
    if (n_tiles && !tiles) return fail(c, TGB_ERR_INVALID, "null tile list");
    if (c->group) {         // every member needs the caller's running means for its own pixels
        std::vector<uint32_t> base;
        if (!count) base.assign(size_t(c->res_x)*c->res_y, spp_begin);
        int rc = tgb200_write_framebuffer(c, rgb_mean, count ? count : base.data());
        if (rc) return rc;
        if ((rc = group_render(c, tiles, n_tiles, seed, spp_begin, spp_count, nullptr))) return rc;
        return tgb200_read_framebuffer(c, rgb_mean, count);
    }
    CU(cudaSetDevice(c->device));
    size_t npx = size_t(c->res_x)*c->res_y;
    // host -> device: the caller's running mean and counts are the input state
    std::memcpy(c->h_fb, rgb_mean, npx*3*sizeof(float));
    CU(cudaMemcpyAsync(c->fb, c->h_fb, npx*3*sizeof(float), cudaMemcpyHostToDevice, c->stream));
    if (count) {
        std::memcpy(c->h_fb_count, count, npx*sizeof(uint32_t));
        CU(cudaMemcpyAsync(c->fb_count, c->h_fb_count, npx*sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    } else {
        // without counts the running mean restarts from the sample index range's start
        std::vector<uint32_t> base(npx, spp_begin);
        std::memcpy(c->h_fb_count, base.data(), npx*sizeof(uint32_t));
        CU(cudaMemcpyAsync(c->fb_count, c->h_fb_count, npx*sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
    }
    int rc = set_tiles(c, tiles, n_tiles, seed);
    if (rc) return rc;
    if ((rc = render_device(c, spp_begin, spp_count))) return rc;
    return tgb200_read_framebuffer(c, rgb_mean, count);
}

int tgb200_framebuffer_device_ptr(tgb_ctx *c, void **rgb_mean_dev, uint64_t *n_bytes) {
    if (!c || !rgb_mean_dev) return TGB_ERR_INVALID;
    *rgb_mean_dev = c->fb;
    if (n_bytes) *n_bytes = uint64_t(c->res_x)*c->res_y*3*sizeof(float);
    return TGB_OK;
}

// Closest hits of n device rays through the analytic pass and the renderer's traversal kernels (into device Hit records)
// As in a render, rays that miss the BVH's top-level cut before their analytic hit skip the traversal (TGB_HOOK_CUT=0: every ray
// is traversed).
static cudaError_t hook_closest(tgb_ctx *c, const tgb_ray *dr, Hit *dx, uint32_t n) {
    const char *cut_env = getenv("TGB_HOOK_CUT");
    const int cut = (cut_env && cut_env[0] == '0') ? 0 : 1;
    uint32_t *list = nullptr;                                   // [count | indices of the rays to traverse]
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void **>(&list), (size_t(n) + 1)*sizeof(uint32_t), c->stream);
    if (e != cudaSuccess) return e;
    e = cudaMemsetAsync(list, 0, sizeof(uint32_t), c->stream);
    if (e == cudaSuccess) {
        k_hook_analytic<<<blocks(n, 256), 256, 0, c->stream>>>(c->sc, dr, dx, n, cut, list + 1, list);
        c->stats.kernel_launches++;
    }
    if (e == cudaSuccess && c->sc.n_nodes) {
        // the renderer's own persistent kernel body (lane refill)
        uint32_t *cursor = &c->wf[0].ctl->cursor_trace;
        e = cudaMemsetAsync(cursor, 0, sizeof(uint32_t), c->stream);
        uint32_t grid = std::min(blocks(n, kTraceBlock), c->persist_blocks);
        if (e == cudaSuccess) {
            if (c->has_curves) k_hook_persist<true><<<grid, kTraceBlock, 0, c->stream>>>(c->sc, dr, dx, list + 1, list, n, cursor);
            else k_hook_persist<false><<<grid, kTraceBlock, 0, c->stream>>>(c->sc, dr, dx, list + 1, list, n, cursor);
        }
        c->stats.kernel_launches++;
    }
    const cudaError_t ef = cudaFreeAsync(list, c->stream);
    return e != cudaSuccess ? e : ef;
}

int tgb200_trace_closest(tgb_ctx *c, const tgb_ray *rays, tgb_hit *hits, uint32_t n) {
    if (!c || (n && (!rays || !hits))) return TGB_ERR_INVALID;
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    tgb_ray *dr = nullptr; tgb_hit *dh = nullptr; Hit *dx = nullptr;
    CU(cudaMalloc(reinterpret_cast<void **>(&dr), size_t(n)*sizeof(tgb_ray)));
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&dh), size_t(n)*sizeof(tgb_hit));
    if (e == cudaSuccess) e = cudaMalloc(reinterpret_cast<void **>(&dx), size_t(n)*sizeof(Hit));
    if (e != cudaSuccess) { cudaFree(dr); cudaFree(dh); return fail(c, TGB_ERR_OOM, "cudaMalloc failed: %s", cudaGetErrorString(e)); }
    int rc = TGB_OK;
    do {
        if ((e = cudaMemcpyAsync(dr, rays, size_t(n)*sizeof(tgb_ray), cudaMemcpyHostToDevice, c->stream)) != cudaSuccess) break;
        if ((e = hook_closest(c, dr, dx, n)) != cudaSuccess) break;
        k_hook_finish<<<blocks(n, 256), 256, 0, c->stream>>>(c->sc, dr, dx, dh, n);
        c->stats.kernel_launches++;
        if ((e = cudaMemcpyAsync(hits, dh, size_t(n)*sizeof(tgb_hit), cudaMemcpyDeviceToHost, c->stream)) != cudaSuccess) break;
        e = cudaStreamSynchronize(c->stream);
        if (e == cudaSuccess) e = cudaGetLastError();
    } while (0);
    if (e != cudaSuccess) rc = fail(c, TGB_ERR_CUDA, "trace_closest failed: %s", cudaGetErrorString(e));
    cudaFree(dr); cudaFree(dh); cudaFree(dx);
    return rc;
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

static int tile_pixels(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t **dev, uint32_t *n_out, bool *owned) {
    *owned = true;
    if (c->tiles_cached.size() == n_tiles && n_tiles && std::memcmp(c->tiles_cached.data(), tiles, n_tiles*sizeof(tgb_tile)) == 0) {
        *dev = c->pix_id; *n_out = c->n_pix; *owned = false;      // same tile list as the last render: reuse its pixel list
        return TGB_OK;
    }
    std::vector<uint32_t> pid;
    for (uint32_t t = 0; t < n_tiles; ++t) {
        const tgb_tile &tl = tiles[t];
        if (tl.x >= c->res_x || tl.w > c->res_x - tl.x || tl.y >= c->res_y || tl.h > c->res_y - tl.y) return fail(c, TGB_ERR_INVALID, "tile %u lies outside the image", t);
        for (uint32_t y = 0; y < tl.h; ++y) for (uint32_t x = 0; x < tl.w; ++x) pid.push_back((tl.x + x) + (tl.y + y)*c->res_x);
    }
    *n_out = uint32_t(pid.size()); *dev = nullptr;
    if (pid.empty()) return TGB_OK;
    CU(cudaMalloc(reinterpret_cast<void **>(dev), pid.size()*4));
    cudaError_t e = cudaMemcpyAsync(*dev, pid.data(), pid.size()*4, cudaMemcpyHostToDevice, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) { cudaFree(*dev); *dev = nullptr; return fail(c, TGB_ERR_CUDA, "tile upload failed: %s", cudaGetErrorString(e)); }
    return TGB_OK;
}

int tgb200_pack_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, void *rgb_out_dev) {
    if (!c || !tiles || !rgb_out_dev) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    uint32_t *pid = nullptr, n = 0; bool owned = true;
    int rc = tile_pixels(c, tiles, n_tiles, &pid, &n, &owned);
    if (rc || !n) return rc;
    k_pack_tiles<<<blocks(n, 256), 256, 0, c->stream>>>(pid, n, c->fb, static_cast<float *>(rgb_out_dev));
    c->stats.kernel_launches++;
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (owned) cudaFree(pid);
    if (e != cudaSuccess) return fail(c, TGB_ERR_CUDA, "pack_tiles failed: %s", cudaGetErrorString(e));
    return TGB_OK;
}

int tgb200_unpack_tiles(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, const void *rgb_in_dev, uint32_t sample_count) {
    if (!c || !tiles || !rgb_in_dev) return TGB_ERR_INVALID;
    CU(cudaSetDevice(c->device));
    uint32_t *pid = nullptr, n = 0; bool owned = true;
    int rc = tile_pixels(c, tiles, n_tiles, &pid, &n, &owned);
    if (rc || !n) return rc;
    k_unpack_tiles<<<blocks(n, 256), 256, 0, c->stream>>>(pid, n, static_cast<const float *>(rgb_in_dev), c->fb, c->fb_count, sample_count);
    c->stats.kernel_launches++;
    cudaError_t e = cudaStreamSynchronize(c->stream);
    if (owned) cudaFree(pid);
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
    std::memcpy(c->h_fb, rgb_mean, npx*3*sizeof(float)); std::memcpy(c->h_fb_count, count, npx*sizeof(uint32_t));
    CU(cudaMemcpyAsync(c->fb, c->h_fb, npx*3*sizeof(float), cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->fb_count, c->h_fb_count, npx*sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
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
}  // extern "C"
namespace {
int single_render_adaptive(tgb_ctx *c, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, tgb_sample_record *records) {
    static_assert(sizeof(tgb_sample_record) == sizeof(SampleRecordD), "record layout");
    CU(cudaSetDevice(c->device));
    int rc = set_tiles(c, tiles, n_tiles, seed);
    if (rc) return rc;
    const uint32_t var_w = (c->res_x + 3)/4, var_h = (c->res_y + 3)/4, n_blocks = var_w*var_h;
    if (c->n_pix == 0) return TGB_OK;
    if (c->adaptive_capacity < c->n_pix + 1 || !c->rec_dev) {
        if ((rc = dev_alloc(c, &c->pix_first, size_t(c->n_pix) + 1))) return rc;
        if ((rc = dev_alloc(c, &c->pix_base, size_t(c->n_pix) + 1))) return rc;
        if (!c->pix_slot && (rc = dev_alloc(c, &c->pix_slot, size_t(c->res_x)*c->res_y))) return rc;
        if (!c->rec_dev && (rc = dev_alloc(c, &c->rec_dev, n_blocks))) return rc;
        c->adaptive_capacity = c->n_pix + 1;
    }
    std::vector<uint32_t> first(size_t(c->n_pix) + 1), base(size_t(c->n_pix) + 1, 0);
    uint64_t total = 0; uint32_t max_cnt = 0;
    for (uint32_t i = 0; i < c->n_pix; ++i) {
        const uint32_t px = c->h_pix_id[i] % c->res_x, py = c->h_pix_id[i]/c->res_x;
        const tgb_sample_record &r = records[px/4 + (py/4)*var_w];
        first[i] = uint32_t(total); base[i] = r.sample_index;
        total += r.next_sample_count; max_cnt = std::max(max_cnt, r.next_sample_count);
        if (total > 0xFFFFFFFFull) return fail(c, TGB_ERR_UNSUPPORTED, "adaptive step too large");
    }
    first[c->n_pix] = uint32_t(total);
    uint32_t pix_bits = 0; while (pix_bits < 32 && (uint64_t(1) << pix_bits) < uint64_t(c->n_pix)) ++pix_bits;
    if (uint64_t(max_cnt) > (uint64_t(1) << (32 - pix_bits))) return fail(c, TGB_ERR_UNSUPPORTED, "adaptive step: %u samples for one pixel do not fit the path id", max_cnt);
    if (!c->pix_slot_valid) {
        std::vector<uint32_t> slot(size_t(c->res_x)*c->res_y, 0xFFFFFFFFu);
        for (uint32_t i = 0; i < c->n_pix; ++i) slot[c->h_pix_id[i]] = i;
        CU(cudaMemcpyAsync(c->pix_slot, slot.data(), slot.size()*4, cudaMemcpyHostToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
        c->pix_slot_valid = true;
    }
    CU(cudaMemcpyAsync(c->pix_first, first.data(), first.size()*4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->pix_base, base.data(), base.size()*4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(c->rec_dev, records, size_t(n_blocks)*sizeof(SampleRecordD), cudaMemcpyHostToDevice, c->stream));
    CU(cudaStreamSynchronize(c->stream));                       // (the host vectors go out of scope)
    if (total == 0) return TGB_OK;
    if ((rc = render_device(c, 0, 0, true, uint32_t(total)))) return rc;
    BatchInfo bi; bi.pix_id = c->pix_id; bi.pix_seed = c->pix_seed; bi.n_pix = c->n_pix; bi.spp_begin = 0;
    bi.pix_first = c->pix_first; bi.pix_base = c->pix_base; bi.pix_bits = pix_bits;
    k_block_stats<<<blocks(n_blocks, 128), 128, 0, c->stream>>>(c->R, bi, c->pix_slot, c->res_x, c->res_y, var_w, n_blocks, c->rec_dev);
    c->stats.kernel_launches++;
    CU(cudaMemcpyAsync(records, c->rec_dev, size_t(n_blocks)*sizeof(SampleRecordD), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    CU(cudaGetLastError());
    return TGB_OK;
}
}  // namespace
extern "C" {

int tgb200_shard_tiles(const tgb_tile *tiles, uint32_t n_tiles, uint32_t *order) {
    if ((n_tiles && !tiles) || !order) return TGB_ERR_INVALID;
    std::vector<uint32_t> o; shard_order(tiles, n_tiles, o);
    std::memcpy(order, o.data(), size_t(n_tiles)*4);
    return TGB_OK;
}

namespace {
// UniformSampler (sampling/UniformSampler.hpp:40-52): the integrator's own PCG32 stream (tile seeds, adaptive distribution)
inline float pcg_next1d(uint64_t &state) { return normalized_uint(pcg_next(state)); }
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
            r.adaptive_weight = variance/(float(r.sample_count)*std::max(r.mean*r.mean, 1e-3f));
            if (r.adaptive_weight > 0.0f) errors.push_back(r.adaptive_weight);
        }
        if (errors.empty()) return 0;
        std::sort(errors.begin(), errors.end());
        const float max_error = errors[(errors.size()*95)/100];
        if (max_error == 0.0f) return 0;
        for (size_t i = 0; i < n; ++i) records[i].adaptive_weight = std::min(records[i].adaptive_weight, max_error);
        // dilateAdaptiveWeights (:61-88)
        for (uint32_t y = 0; y < var_h; ++y) for (uint32_t x = 0; x < var_w; ++x) {
            size_t idx = x + size_t(y)*var_w;
            if (y < var_h - 1) records[idx].adaptive_weight = std::max(records[idx].adaptive_weight, records[idx + var_w].adaptive_weight);
            if (x < var_w - 1) records[idx].adaptive_weight = std::max(records[idx].adaptive_weight, records[idx + 1].adaptive_weight);
        }
        for (int y = int(var_h) - 1; y >= 0; --y) for (int x = int(var_w) - 1; x >= 0; --x) {
            size_t idx = size_t(x) + size_t(y)*var_w;
            if (y > 0) records[idx].adaptive_weight = std::max(records[idx].adaptive_weight, records[idx - var_w].adaptive_weight);
            if (x > 0) records[idx].adaptive_weight = std::max(records[idx].adaptive_weight, records[idx - 1].adaptive_weight);
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

namespace {
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
}  // namespace

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
// out = 10 uint32 per query: cut mask, deepest stack of the walk from the cut, then per walk (root, cut): occluded, node visits,
// LEAF trips, triangle tests.  *stack_need = the bound tgb200_create checks; TGB_ERR_UNSUPPORTED when it exceeds stack_size (0: the
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
        uint32_t *o10 = out + 10*size_t(r);
        std::memset(o10, 0, 10*sizeof(uint32_t));
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
            if (from_cut) o10[1] = uint32_t(deepest);
        }
    }
    return TGB_OK;
}

}  // extern "C"

// ---- test hooks: host arrays in, one probe kernel on the context's stream, host arrays out ----
namespace {
struct ProbeBufs {                  // device copies of a probe's arrays, freed on every exit
    tgb_ctx *c; std::vector<void *> p;
    explicit ProbeBufs(tgb_ctx *ctx) : c(ctx) {}
    ~ProbeBufs() { for (void *q : p) cudaFree(q); }
    template <typename T> cudaError_t alloc(T **out, size_t n) {
        void *q = nullptr;
        cudaError_t e = cudaMalloc(&q, std::max<size_t>(n, 1)*sizeof(T));
        if (e == cudaSuccess) p.push_back(q);
        *out = static_cast<T *>(q);
        return e;
    }
    template <typename T> cudaError_t upload(T **out, const T *src, size_t n) {
        cudaError_t e = alloc(out, n);
        return e != cudaSuccess ? e : cudaMemcpyAsync(*out, src, n*sizeof(T), cudaMemcpyHostToDevice, c->stream);
    }
    template <typename T> cudaError_t download(T *dst, const T *src, size_t n) {
        return cudaMemcpyAsync(dst, src, n*sizeof(T), cudaMemcpyDeviceToHost, c->stream);
    }
    int finish(cudaError_t e, const char *what) {
        if (e == cudaSuccess) e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        return e == cudaSuccess ? TGB_OK : fail(c, TGB_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
    }
};
// lobe_set 1 (the Lambert-only instantiation) exists only without curves, as in k_shade
int probe_check(tgb_ctx *c, int lobe_set) {
    if (lobe_set != 0 && lobe_set != 1) return fail(c, TGB_ERR_INVALID, "lobe_set must be 0 or 1");
    if (lobe_set == 1 && c->has_curves) return fail(c, TGB_ERR_INVALID, "lobe_set 1 has no instantiation with curves");
    return TGB_OK;
}
}  // namespace

extern "C" {

int tgb200_bsdf_probe(tgb_ctx *c, int bsdf, float u, float v, uint32_t requested, int lobe_set, uint32_t n, const float *wi_wo,
                      float *out) {
    if (!c || (n && (!wi_wo || !out))) return TGB_ERR_INVALID;
    if (int rc = probe_check(c, lobe_set)) return rc;
    if (bsdf < 0 || bsdf >= c->n_bsdfs) return fail(c, TGB_ERR_INVALID, "bsdf %d out of range", bsdf);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    float *dw = nullptr, *dout = nullptr;
    cudaError_t e = b.upload(&dw, wi_wo, 6*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, 4*size_t(n));
    if (e == cudaSuccess) {
        const uint32_t g = blocks(n, 128);
        if (c->has_curves) k_probe_bsdf<true, 0><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw, dout, n);
        else if (lobe_set == 1) k_probe_bsdf<false, 1><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw, dout, n);
        else k_probe_bsdf<false, 0><<<g, 128, 0, c->stream>>>(c->sc, bsdf, u, v, requested, dw, dout, n);
        e = b.download(out, dout, 4*size_t(n));
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
    int *db = nullptr; uint32_t *dpix = nullptr, *dl = nullptr; float *dwi = nullptr, *dout = nullptr;
    cudaError_t e = b.upload(&db, bsdf, n);
    if (e == cudaSuccess) e = b.upload(&dpix, pixel_id, n);
    if (e == cudaSuccess) e = b.upload(&dwi, wi, 3*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, 8*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dl, n);
    if (e == cudaSuccess) {
        const uint32_t g = blocks(n, 128);
        if (c->has_curves) k_probe_bsdf_sample<true, 0><<<g, 128, 0, c->stream>>>(c->sc, seed, db, dpix, sample, u, v, requested, dwi, dout, dl, n);
        else if (lobe_set == 1) k_probe_bsdf_sample<false, 1><<<g, 128, 0, c->stream>>>(c->sc, seed, db, dpix, sample, u, v, requested, dwi, dout, dl, n);
        else k_probe_bsdf_sample<false, 0><<<g, 128, 0, c->stream>>>(c->sc, seed, db, dpix, sample, u, v, requested, dwi, dout, dl, n);
        e = b.download(out, dout, 8*size_t(n));
        if (e == cudaSuccess) e = b.download(lobes, dl, n);
    }
    return b.finish(e, "bsdf_sample_probe");
}

int tgb200_light_probe(tgb_ctx *c, int prim, uint32_t seed, uint32_t n, uint32_t sample, const float *p, float *out) {
    if (!c || (n && (!p || !out))) return TGB_ERR_INVALID;
    if (prim < 0 || uint32_t(prim) >= c->sc.n_prims) return fail(c, TGB_ERR_INVALID, "primitive %d out of range", prim);
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    float *dp = nullptr, *dout = nullptr; tgb_ray *dr = nullptr; Hit *dx = nullptr;
    cudaError_t e = b.upload(&dp, p, 3*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, 12*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dr, n);
    if (e == cudaSuccess) e = b.alloc(&dx, n);
    if (e == cudaSuccess) {
        k_probe_light<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, prim, seed, sample, dp, dout, dr, n);
        if (c->prim_types[size_t(prim)] == TGB_PRIM_MESH &&(e = hook_closest(c, dr, dx, n)) == cudaSuccess)
            k_probe_light_mesh<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, prim, dr, dx, dout, n);
        if (e == cudaSuccess) e = b.download(out, dout, 12*size_t(n));
    }
    return b.finish(e, "light_probe");
}

int tgb200_choose_light_probe(tgb_ctx *c, uint32_t seed, uint32_t n, const uint32_t *pixel_id, uint32_t sample, const float *p,
                              float *out) {
    if (!c || (n && (!pixel_id || !p || !out))) return TGB_ERR_INVALID;
    if (n == 0) return TGB_OK;
    CU(cudaSetDevice(c->device));
    ProbeBufs b(c);
    uint32_t *dpix = nullptr; float *dp = nullptr, *dout = nullptr;
    cudaError_t e = b.upload(&dpix, pixel_id, n);
    if (e == cudaSuccess) e = b.upload(&dp, p, 3*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, 2*size_t(n));
    if (e == cudaSuccess) {
        k_probe_choose_light<<<blocks(n, 128), 128, 0, c->stream>>>(c->sc, seed, dpix, sample, dp, dout, n);
        e = b.download(out, dout, 2*size_t(n));
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
    float *dq = nullptr, *dout = nullptr; int *dl = nullptr; Ctl *ctl_saved = nullptr; Counters *ctr_saved = nullptr;
    cudaError_t e = b.upload(&dq, query, 8*size_t(n));
    if (e == cudaSuccess) e = b.upload(&dl, light_mis, 2*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, 8*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&ctl_saved, 1);
    if (e == cudaSuccess) e = b.alloc(&ctr_saved, 1);
    // the probe's queries must not show in the context's control block or in the next render's statistics
    const Wavefront &w = c->wf[0];
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctl_saved, w.ctl, sizeof(Ctl), cudaMemcpyDeviceToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctr_saved, c->ctr, sizeof(Counters), cudaMemcpyDeviceToDevice, c->stream);
    const bool saved = e == cudaSuccess;
    const DScene &sc = c->sc; const bool curves = c->has_curves; cudaStream_t st = c->stream;
    // one scratch slot per query: chunks of wavefront 0's capacity
    for (uint32_t off = 0; off < n && e == cudaSuccess; off += w.capacity) {
        const uint32_t m = std::min(w.capacity, n - off);
        // shadow_count, shadow_count2, cursor_trace, cursor_shadow, shadow_count_closest, cursor_closest
        e = cudaMemsetAsync(&w.ctl->shadow_count, 0, 6*sizeof(uint32_t), st);
        if (e != cudaSuccess) break;
        k_probe_shadow_setup<<<blocks(m, 128), 128, 0, st>>>(sc, w.sr, dq + 8*size_t(off), dl + 2*size_t(off), dout + 8*size_t(off),
                                                            w.squeue, w.ctl, m);
        if (curves) k_shadow_prep<true><<<blocks(m, 256), 256, 0, st>>>(sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
        else k_shadow_prep<false><<<blocks(m, 256), 256, 0, st>>>(sc, w.sr, w.squeue, w.ctl, w.squeue2, w.squeue_cl, c->ctr);
        k_probe_shadow_traversed<<<blocks(m, 256), 256, 0, st>>>(w.squeue2, w.squeue_cl, w.ctl, dout + 8*size_t(off));
        if (sc.n_nodes) launch_shadow_bvh(c, w, st, std::min(blocks(m, kTraceBlock), c->persist_blocks));
        k_probe_shadow_read<<<blocks(m, 128), 128, 0, st>>>(w.sr, dl + 2*size_t(off), dout + 8*size_t(off), m);
        e = cudaGetLastError();
    }
    // restored also when a launch failed (the copies are queued after whatever was queued)
    if (saved) {
        const cudaError_t r1 = cudaMemcpyAsync(w.ctl, ctl_saved, sizeof(Ctl), cudaMemcpyDeviceToDevice, st);
        const cudaError_t r2 = cudaMemcpyAsync(c->ctr, ctr_saved, sizeof(Counters), cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = r1 != cudaSuccess ? r1 : r2;
    }
    if (e == cudaSuccess) e = b.download(out, dout, 8*size_t(n));
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
    uint32_t *din = nullptr, *dout = nullptr, *pix = nullptr; Ctl *ctl_saved = nullptr; Counters *ctr_saved = nullptr;
    cudaError_t e = b.upload(&din, state_in, TGB_BOUNCE_WORDS*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&dout, TGB_BOUNCE_WORDS*size_t(n));
    if (e == cudaSuccess) e = b.alloc(&pix, 4*size_t(w.capacity) + 1);
    if (e == cudaSuccess) e = b.alloc(&ctl_saved, 1);
    if (e == cudaSuccess) e = b.alloc(&ctr_saved, 1);
    // the probe's paths must not show in the context's control block or in the next render's statistics
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctl_saved, w.ctl, sizeof(Ctl), cudaMemcpyDeviceToDevice, c->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ctr_saved, c->ctr, sizeof(Counters), cudaMemcpyDeviceToDevice, c->stream);
    const bool saved = e == cudaSuccess;
    const DScene &sc = c->sc; cudaStream_t st = c->stream;
    PathBuf &pb = w.pb[0], &dst = w.pb[1];
    // per chunk: one pixel per path (pix_id, pix_seed, pix_first (m + 1 offsets), pix_base), so path id = result slot = its index
    uint32_t *pix_id = pix, *pix_seed = pix + w.capacity, *pix_base = pix + 2*size_t(w.capacity), *pix_first = pix + 3*size_t(w.capacity);
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
        bi.pix_bits = 0; while ((1u << bi.pix_bits) < m) ++bi.pix_bits;
        uint32_t *o = dout + TGB_BOUNCE_WORDS*size_t(off);
        k_probe_bounce_setup<<<blocks(m, 256), 256, 0, st>>>(sc, pb, din + TGB_BOUNCE_WORDS*size_t(off), pix_id, pix_seed, pix_first,
                                                            pix_base, w.bin_keys, w.bin_hist, o, m);
        k_iter_end<<<1, 1024, 0, st>>>(w.bin_hist, w.ctl, sc.n_nodes ? 1 : 0);
        if (sc.n_nodes) {
            k_bin_scatter<<<blocks(m, 256), 256, 0, st>>>(w.bin_keys, w.bin_hist, w.ctl, w.order);
            launch_trace(c, w, pb, st, m);
        }
        launch_shade(c, w, pb, st, bi, m);
        launch_shadow_prep(c, w, st, m);
        if (sc.n_nodes) launch_shadow_bvh(c, w, st, std::min(blocks(2*m, kTraceBlock), c->persist_blocks));
        k_accum<<<blocks(m, 256), 256, 0, st>>>(sc, pb, dst, w.sr, bi, w.ctl, w.bin_keys, w.bin_hist);
        k_probe_bounce_alive<<<blocks(m, 256), 256, 0, st>>>(dst, w.ctl, o);
        k_probe_bounce_finished<<<blocks(m, 256), 256, 0, st>>>(pb, c->R, o, m);
        e = cudaGetLastError();
        // (the next chunk's control block is copied from this host variable: wait until this one is consumed)
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    // restored also when a launch failed (the copies are queued after whatever was queued)
    if (saved) {
        const cudaError_t r1 = cudaMemcpyAsync(w.ctl, ctl_saved, sizeof(Ctl), cudaMemcpyDeviceToDevice, st);
        const cudaError_t r2 = cudaMemcpyAsync(c->ctr, ctr_saved, sizeof(Counters), cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = r1 != cudaSuccess ? r1 : r2;
    }
    if (e == cudaSuccess) e = b.download(state_out, dout, TGB_BOUNCE_WORDS*size_t(n));
    return b.finish(e, "bounce_probe");
}

int tgb200_shade_variant(const tgb_ctx *c, uint32_t *variant) {
    if (!c || !variant) return TGB_ERR_INVALID;
    variant[0] = c->has_curves ? 1u : 0u; variant[1] = c->sort_materials ? 1u : 0u; variant[2] = c->diffuse_only ? 1u : 0u;
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
