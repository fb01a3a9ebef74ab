// Host-side scene preparation: a tgb_scene_desc checked and turned into the device records and the host arrays they point to
// (the reference's TraceableScene constructor and prepareForRender), with no CUDA call.  upload_scene in tgb200_api.cu puts the
// result on a device; a multi-GPU context prepares once and uploads the same HostScene to every member.
// fp32 in the reference's operation order: compiled into tgb200_api.cu with -fmad=false and -ffp-contract=off.
#pragma once
#include <algorithm>
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

extern "C" const unsigned char tgb_sobol_blob[];      // sobol_blob.cpp (.incbin of data/sobol_1024x32.u32)

namespace tgb {
namespace {

thread_local std::string g_create_error;            // why the last tgb200_create on this thread failed (tgb200_last_error(NULL))

// A refused desc: its code (TGB_ERR_INVALID / TGB_ERR_UNSUPPORTED) and reason
int refuse(int code, const char *fmt, ...) {
    char buf[1024];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_create_error = buf;
    return code;
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
    case TGB_BSDF_SMOOTH_COAT: return LOBE_SPEC_R;          // | substrate lobes, added by prepare_bsdfs
    case TGB_BSDF_ROUGH_COAT: return LOBE_GLOSSY_R;         // | substrate lobes (RoughCoatBsdf.cpp:301-306)
    case TGB_BSDF_HAIR: return LOBE_GLOSSY_R | LOBE_GLOSSY_T | LOBE_ANISO;                  // bsdfs/HairBcsdf.cpp:20
    default: return 0xFFFFFFFFu;
    }
}

struct HostTex { DTex d; V3 maxv; std::vector<float> texels, marg_pdf, marg_cdf, pdf, cdf; bool has_dist = false; };

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

// ---- prepare_scene: the desc's checks and the host-side prepare step, with no CUDA call ----
// The device records keep their pointer fields empty; next to them are the host arrays upload_scene points those fields at.
struct MeshLight { uint32_t prim; std::vector<float> pdf, cdf, verts; };    // an emissive mesh's area distribution, p0 p1 p2 per tri

// What the kernel choice depends on (select_kernels)
struct SceneKind {
    bool has_curves = false;        // curve pieces in the BVH: the instantiations with the curve-segment test and per-hit epsilon
    bool mesh_lights = false;       // a mesh is a light: closest-hit shadow queries exist, k_shadow_bvh<., true> runs
    uint32_t bsdf_types = 0;        // bit t: a surface uses a BSDF of type t (null BSDFs excluded)
    bool quad_lights = false;       // every light a quad, no infinite emitter, every emission and Lambert albedo texture constant
};

struct HostScene {
    DScene sc{};                    // the scalars: settings, camera, counts, cut, binning grid
    std::vector<HostTex> tex;       // the desc's textures, then the constant white of the default light
    std::vector<DBsdf> bsdfs;
    std::vector<HairTables> hair;   // per BSDF: its tables when it is the hair BCSDF
    std::vector<DPrim> prims;       // the desc's primitives, then the default light when nothing emits
    std::vector<MeshLight> mesh_lights;
    std::vector<int> lights, inf_lights, analytic;    // analytic: the list the ray-creating kernels loop over (BVH leaf order)
    std::vector<uint32_t> slots, tri_prim, sobol;
    std::vector<float4> tri_shade;  // shading records, in BVH leaf order
    SceneBvh bvh;
    SceneKind kind;
};

// The geometry the BVH is built over, as the primitives add it
struct BuildGeometry {
    std::vector<BuildTri> tris; std::vector<float4> tri_shade;
    std::vector<BuildBox> curve_boxes; std::vector<IsectRecord> curve_recs; std::vector<uint32_t> curve_prim;   // kCurvePieces per segment
};

// cameras/PinholeCamera.cpp:28-35, Camera.cpp:37-42
void prepare_camera(const tgb_camera &cam, DCamera &o) {
    o.pos = f3(cam.pos); std::memcpy(o.m, cam.xform, sizeof(o.m));
    float fovRad = cam.fov_deg*(PI_F/180.0f);
    o.plane_dist = 1.0f/std::tan(fovRad*0.5f);
    o.ratio = cam.res_y/float(cam.res_x);
    o.pixel_size_x = 1.0f/cam.res_x;
    o.res_x = cam.res_x; o.res_y = cam.res_y; o.filter = cam.filter;
    filter_precompute(o);
}

// The desc's textures, then at index n_textures the constant white the default light emits
int prepare_textures(const tgb_texture *textures, uint32_t n_textures, std::vector<HostTex> &tex) {
    tex.assign(n_textures + 1, HostTex{});
    for (uint32_t i = 0; i < n_textures; ++i) {
        const tgb_texture &t = textures[i]; DTex &o = tex[i].d;
        std::memset(&o, 0, sizeof(o));
        o.type = t.type; o.value = f3(t.value); o.value2 = f3(t.value2); o.res_u = int(t.res_u); o.res_v = int(t.res_v); o.flags = t.flags;
        if (t.type == TGB_TEX_BITMAP) {
            if (!t.texels || !t.res_u || !t.res_v) return refuse(TGB_ERR_INVALID, "bitmap texture %u has no texels", i);
            size_t n = size_t(t.res_u)*t.res_v;
            V3 acc = v3s(0.0f), mx = v3s(0.0f);
            for (size_t k = 0; k < n; ++k) { V3 cc = f3(t.texels + 3*k); acc = acc + cc/float(n); mx = v3(std::max(mx.x, cc.x), std::max(mx.y, cc.y), std::max(mx.z, cc.z)); }
            o.avg = acc; tex[i].maxv = mx;
            tex[i].texels.assign(t.texels, t.texels + 3*n);
        } else if (t.type == TGB_TEX_CHECKER) {
            o.avg = (o.value + o.value2)*0.5f;
            tex[i].maxv = v3(std::max(o.value.x, o.value2.x), std::max(o.value.y, o.value2.y), std::max(o.value.z, o.value2.z));
        } else if (t.type == TGB_TEX_CONSTANT) { o.avg = o.value; tex[i].maxv = o.value; }
        else return refuse(TGB_ERR_UNSUPPORTED, "texture type %u is outside the hot path", t.type);
    }
    DTex &o = tex[n_textures].d; std::memset(&o, 0, sizeof(o)); o.type = TGB_TEX_CONSTANT; o.value = v3s(1.0f); o.avg = o.value; tex[n_textures].maxv = o.value;
    return TGB_OK;
}

int prepare_bsdfs(const tgb_scene_desc *d, const std::vector<HostTex> &tex, std::vector<DBsdf> &bsdfs, std::vector<HairTables> &hair) {
    bsdfs.resize(d->n_bsdfs); hair.resize(d->n_bsdfs);
    for (uint32_t i = 0; i < d->n_bsdfs; ++i) {
        const tgb_bsdf &b = d->bsdfs[i]; DBsdf &o = bsdfs[i];
        std::memset(&o, 0, sizeof(o));
        o.type = b.type; o.lobes = bsdf_lobes(b);
        if (o.lobes == 0xFFFFFFFFu) return refuse(TGB_ERR_UNSUPPORTED, "bsdf type %u is outside the hot path", b.type);
        if (b.albedo_tex < 0 || uint32_t(b.albedo_tex) >= d->n_textures) return refuse(TGB_ERR_INVALID, "bsdf %u: bad albedo texture", i);
        bool rough = b.type == TGB_BSDF_ROUGH_CONDUCTOR || b.type == TGB_BSDF_ROUGH_DIELECTRIC || b.type == TGB_BSDF_ROUGH_PLASTIC || b.type == TGB_BSDF_ROUGH_COAT;
        if (rough && (b.roughness_tex < 0 || uint32_t(b.roughness_tex) >= d->n_textures)) return refuse(TGB_ERR_INVALID, "bsdf %u: bad roughness texture", i);
        o.dist = b.distribution; o.albedo_tex = b.albedo_tex; o.rough_tex = b.roughness_tex;
        o.ior = b.ior; o.inv_ior = 1.0f/b.ior; o.eta = f3(b.eta); o.k = f3(b.k); o.enable_t = b.enable_refraction; o.substrate = b.substrate;
        if (b.type == TGB_BSDF_SMOOTH_COAT || b.type == TGB_BSDF_ROUGH_COAT) {             // SmoothCoatBsdf.cpp:218-223, RoughCoatBsdf.cpp:301-306
            if (b.substrate < 0 || uint32_t(b.substrate) >= d->n_bsdfs || d->bsdfs[b.substrate].type == TGB_BSDF_SMOOTH_COAT ||
                d->bsdfs[b.substrate].type == TGB_BSDF_ROUGH_COAT || d->bsdfs[b.substrate].type == TGB_BSDF_HAIR)
                return refuse(TGB_ERR_UNSUPPORTED, "bsdf %u: a coat needs a substrate that is neither a coat nor the hair BCSDF", i);
            o.scaled_sigma_a = f3(b.sigma_a)*b.thickness;
            o.avg_transmittance = std::exp(-2.0f*avg(o.scaled_sigma_a));
            o.lobes = (b.type == TGB_BSDF_SMOOTH_COAT ? LOBE_SPEC_R : LOBE_GLOSSY_R) | bsdf_lobes(d->bsdfs[b.substrate]);
        }
        if (b.type == TGB_BSDF_HAIR) {                                                    // bsdfs/HairBcsdf.cpp:422-446
            hair_precompute(b.hair_roughness, b.hair_scale_angle_deg, b.sigma_a, hair[i]);
            for (int p = 0; p < 3; ++p) o.hair_v[p] = hair[i].v[p];
            o.hair_scale_rad = hair[i].scale_angle_rad;
        }
        if (b.type == TGB_BSDF_PLASTIC || b.type == TGB_BSDF_ROUGH_PLASTIC) {             // bsdfs/PlasticBsdf.cpp:179-185
            o.scaled_sigma_a = f3(b.sigma_a)*b.thickness;
            o.avg_transmittance = std::exp(-2.0f*avg(o.scaled_sigma_a));
            o.diffuse_fresnel = diffuse_fresnel(b.ior, 1000000);
            o.substrate_weight = avg(tex[b.albedo_tex].d.avg);                             // RoughPlasticBsdf.cpp:215-222
        }
    }
    return TGB_OK;
}

// ---- one function per primitive type: primitive i of the desc into its DPrim o (emissive: its emission texture glows)
int prepare_mesh(const tgb_primitive &p, uint32_t i, bool &emissive, DPrim &o, BuildGeometry &g, std::vector<uint32_t> &tri_prim,
                 std::vector<MeshLight> &mesh_lights) {
    if (p.n_tris && (!p.verts || !p.tris)) return refuse(TGB_ERR_INVALID, "mesh %u has null buffers", i);
    o.tri_first = uint32_t(g.tris.size()); o.n_tris = p.n_tris;
    if (p.smooth) o.flags |= PF_SMOOTH;
    std::vector<float> areas(p.n_tris), lverts;
    float total = 0.0f;
    for (uint32_t k = 0; k < p.n_tris; ++k) {
        const tgb_triangle &t = p.tris[k];
        if (t.v0 >= p.n_verts || t.v1 >= p.n_verts || t.v2 >= p.n_verts) return refuse(TGB_ERR_INVALID, "mesh %u: vertex index out of range", i);
        const tgb_vertex &a = p.verts[t.v0], &b = p.verts[t.v1], &cc = p.verts[t.v2];
        BuildTri bt; std::memcpy(bt.v0, a.pos, 12); std::memcpy(bt.v1, b.pos, 12); std::memcpy(bt.v2, cc.pos, 12);
        g.tris.push_back(bt); tri_prim.push_back(i);
        int mat = std::min(std::max(t.material, 0), int(p.bsdf_count) - 1);      // TriangleMesh.cpp:539
        float4 s0 = make_float4(a.normal[0], a.normal[1], a.normal[2], b.normal[0]);
        float4 s1 = make_float4(b.normal[1], b.normal[2], cc.normal[0], cc.normal[1]);
        float4 s2 = make_float4(cc.normal[2], a.uv[0], a.uv[1], b.uv[0]);
        float4 s3 = make_float4(b.uv[1], cc.uv[0], cc.uv[1], 0.0f);
        if (mat > 1023 || i >= (1u << 22)) return refuse(TGB_ERR_UNSUPPORTED, "mesh %u: more than 1024 materials in one mesh or more than 4 Mi primitives", i);
        uint32_t packed = uint32_t(mat) | (i << 10);            // material | primitive << 10 (make_surface)
        std::memcpy(&s3.w, &packed, 4);
        g.tri_shade.push_back(s0); g.tri_shade.push_back(s1); g.tri_shade.push_back(s2); g.tri_shade.push_back(s3);
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
        mesh_lights.push_back({i, std::move(pdf), std::move(cdf), std::move(lverts)});
    }
    return TGB_OK;
}

void prepare_quad(const tgb_primitive &p, DPrim &o) {                                  // primitives/Quad.cpp:298-316
    o.base = f3(p.base); o.edge0 = f3(p.edge0); o.edge1 = f3(p.edge1);
    V3 n = cross(o.edge1, o.edge0);
    o.area = length(n);
    o.normal = n/o.area;
    o.inv_uv_sq0 = 1.0f/length_sq(o.edge0); o.inv_uv_sq1 = 1.0f/length_sq(o.edge1);
}

int prepare_cube(const tgb_primitive &p, bool emissive, DPrim &o) {                    // primitives/Cube.cpp:351-367
    o.pos = f3(p.pos); o.scale = f3(p.scale);
    std::memcpy(o.rot, p.rot, sizeof(o.rot)); transpose3(o.rot, o.inv_rot);
    if (emissive) return refuse(TGB_ERR_UNSUPPORTED, "emissive cubes are outside the hot path");
    return TGB_OK;
}

int prepare_sphere_cap(const tgb_primitive &p, uint32_t i, DPrim &o) {                 // primitives/InfiniteSphereCap.cpp:231-247
    o.normal = f3(p.cap_dir); o.area = p.cap_cos;
    if (!(p.cap_cos < 1.0f)) return refuse(TGB_ERR_INVALID, "infinite_sphere_cap %u: cap angle must be positive", i);
    return TGB_OK;
}

// An infinite sphere (primitives/InfiniteSphere.cpp prepareForRender), or a skydome: an environment sphere with its own prepared
// image, looked up without rotation (Skydome::directionToUV, Skydome.cpp:29-38)
int prepare_infinite_sphere(const tgb_primitive &p, uint32_t i, bool emissive, const std::vector<HostTex> &tex, DPrim &o) {
    if (p.type == TGB_PRIM_SKYDOME) {
        if (p.emission_tex < 0 || tex[p.emission_tex].d.type != TGB_TEX_BITMAP) return refuse(TGB_ERR_INVALID, "skydome %u: pass the prepared sky image (Skydome::prepareForRender) as a bitmap emission texture", i);
        o.type = TGB_PRIM_INFINITE_SPHERE; o.flags |= PF_SKYDOME;
    }
    std::memcpy(o.rot, p.rot, sizeof(o.rot)); transpose3(o.rot, o.inv_rot);
    if (p.type == TGB_PRIM_SKYDOME) { const float id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}; std::memcpy(o.rot, id, sizeof(id)); std::memcpy(o.inv_rot, id, sizeof(id)); }
    if (emissive && tex[p.emission_tex].d.type == TGB_TEX_CHECKER) return refuse(TGB_ERR_UNSUPPORTED, "checker environment maps are outside the hot path");
    return TGB_OK;
}

// primitives/Curves.cpp:572-613 (nodes arrive prepared).  tri_first counts curve pieces here; prepare_bvh rebases it.
int prepare_curves(const tgb_primitive &p, uint32_t i, bool emissive, uint32_t albedo_type, DPrim &o, BuildGeometry &g) {
    if (p.curve_mode > TGB_CURVE_BCSDF_CYLINDER) return refuse(TGB_ERR_UNSUPPORTED, "curves %u: mode outside the hot path", i);
    if (emissive) return refuse(TGB_ERR_UNSUPPORTED, "emissive curves are outside the hot path");
    if (p.n_curve_segments && (!p.curve_nodes || !p.curve_segments)) return refuse(TGB_ERR_INVALID, "curves %u has null buffers", i);
    if (albedo_type != TGB_TEX_CONSTANT) return refuse(TGB_ERR_UNSUPPORTED, "curves %u: textured materials on curves are outside the hot path", i);
    o.curve_mode = p.curve_mode; o.tri_first = uint32_t(g.curve_boxes.size()); o.n_tris = p.n_curve_segments*kCurvePieces;
    for (uint32_t k = 0; k < p.n_curve_segments; ++k) {
        uint32_t t = p.curve_segments[k];
        if (t < 2 || t >= p.n_curve_nodes) return refuse(TGB_ERR_INVALID, "curves %u: segment index out of range", i);
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
            g.curve_boxes.push_back(bb); g.curve_prim.push_back(i);
            IsectRecord rec; std::memcpy(rec.f, n0, sizeof(rec.f));        // n0, n1, n2
            g.curve_recs.push_back(rec);
        }
    }
    return TGB_OK;
}

// The checks every primitive shares, then its type's function.  analytic: the quads and cubes, in desc order.
int prepare_primitives(const tgb_scene_desc *d, const std::vector<HostTex> &tex, std::vector<DPrim> &prims, std::vector<int> &analytic,
                       BuildGeometry &g, std::vector<uint32_t> &tri_prim, std::vector<MeshLight> &mesh_lights) {
    prims.resize(d->n_primitives);
    for (uint32_t i = 0; i < d->n_primitives; ++i) {
        const tgb_primitive &p = d->primitives[i]; DPrim &o = prims[i];
        std::memset(&o, 0, sizeof(o));
        o.type = p.type; o.emission_tex = p.emission_tex; o.bsdf_first = p.bsdf_first; o.bsdf_count = p.bsdf_count;
        if (p.emission_tex >= int(d->n_textures)) return refuse(TGB_ERR_INVALID, "primitive %u: bad emission texture", i);
        bool emissive = p.emission_tex >= 0 && max_comp(tex[p.emission_tex].maxv) > 0.0f;  // primitives/Primitive.hpp:111-115
        const bool infinite = p.type == TGB_PRIM_INFINITE_SPHERE || p.type == TGB_PRIM_INFINITE_SPHERE_CAP || p.type == TGB_PRIM_SKYDOME;
        if (!infinite) {
            if (p.bsdf_count == 0 || p.bsdf_first + p.bsdf_count > d->n_bsdf_slots) return refuse(TGB_ERR_INVALID, "primitive %u: bad bsdf range", i);
            for (uint32_t k = 0; k < p.bsdf_count; ++k) if (d->bsdf_slots[p.bsdf_first + k] >= d->n_bsdfs) return refuse(TGB_ERR_INVALID, "primitive %u: bad bsdf index", i);
            // the hair BCSDF is evaluated in the curve's tangent space (Curves::tangentSpace): on any other primitive the kernels
            // compiled for curve-free scenes would not know the lobe at all
            if (p.type != TGB_PRIM_CURVES)
                for (uint32_t k = 0; k < p.bsdf_count; ++k) {
                    const tgb_bsdf *b = &d->bsdfs[d->bsdf_slots[p.bsdf_first + k]];
                    for (int hop = 0; hop < 4 && b; ++hop) {
                        if (b->type == TGB_BSDF_HAIR) return refuse(TGB_ERR_UNSUPPORTED, "primitive %u: the hair BCSDF on a primitive that is not `curves` is outside the hot path", i);
                        b = ((b->type == TGB_BSDF_SMOOTH_COAT || b->type == TGB_BSDF_ROUGH_COAT) && b->substrate >= 0 && uint32_t(b->substrate) < d->n_bsdfs) ? &d->bsdfs[b->substrate] : nullptr;
                    }
                }
        }
        int rc = TGB_OK;
        switch (p.type) {
        case TGB_PRIM_MESH: rc = prepare_mesh(p, i, emissive, o, g, tri_prim, mesh_lights); break;
        case TGB_PRIM_QUAD: prepare_quad(p, o); analytic.push_back(int(i)); break;
        case TGB_PRIM_CUBE: rc = prepare_cube(p, emissive, o); analytic.push_back(int(i)); break;
        case TGB_PRIM_INFINITE_SPHERE_CAP: rc = prepare_sphere_cap(p, i, o); break;
        case TGB_PRIM_SKYDOME: case TGB_PRIM_INFINITE_SPHERE: rc = prepare_infinite_sphere(p, i, emissive, tex, o); break;
        case TGB_PRIM_CURVES: rc = prepare_curves(p, i, emissive, tex[d->bsdfs[d->bsdf_slots[p.bsdf_first]].albedo_tex].d.type, o, g); break;
        default: rc = refuse(TGB_ERR_UNSUPPORTED, "primitive type %u is outside the hot path", p.type);
        }
        if (rc) return rc;
        const bool samplable = !infinite || p.do_sample != 0;
        if (emissive) o.flags |= PF_EMISSIVE;
        if (samplable) o.flags |= PF_SAMPLABLE;
        if (infinite) o.flags |= PF_INFINITE;
    }
    return TGB_OK;
}

// renderer/TraceableScene.hpp:89-102: the emitters, or the default light when there are none, and the importance maps of the
// environment lights
int prepare_lights(const tgb_texture *textures, uint32_t n_textures, std::vector<DPrim> &prims, std::vector<HostTex> &tex,
                   std::vector<int> &lights, std::vector<int> &inf_lights) {
    for (size_t i = 0; i < prims.size(); ++i) {
        if (!(prims[i].flags & PF_EMISSIVE)) continue;
        if (prims[i].flags & PF_SAMPLABLE) lights.push_back(int(i));
        if (prims[i].flags & PF_INFINITE) inf_lights.push_back(int(i));
    }
    if (std::none_of(prims.begin(), prims.end(), [](const DPrim &p) { return (p.flags & PF_EMISSIVE) != 0; })) {
        DPrim o; std::memset(&o, 0, sizeof(o));
        o.type = TGB_PRIM_INFINITE_SPHERE; o.emission_tex = int(n_textures);
        o.flags = PF_EMISSIVE | PF_SAMPLABLE | PF_INFINITE;
        const float id[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
        std::memcpy(o.rot, id, sizeof(id)); std::memcpy(o.inv_rot, id, sizeof(id));
        lights.push_back(int(prims.size())); inf_lights.push_back(int(prims.size()));
        prims.push_back(o);
    }
    for (int li : lights) {
        DPrim &l = prims[li];
        if (l.type == TGB_PRIM_INFINITE_SPHERE_CAP && tex[l.emission_tex].d.type == TGB_TEX_BITMAP)
            return refuse(TGB_ERR_UNSUPPORTED, "bitmap emission on an infinite_sphere_cap is outside the hot path");
        if (l.type == TGB_PRIM_INFINITE_SPHERE && tex[l.emission_tex].d.type == TGB_TEX_BITMAP && !tex[l.emission_tex].has_dist)
            build_spherical_distribution(textures[l.emission_tex], tex[l.emission_tex]);
    }
    return TGB_OK;
}

// ---- BVH over every mesh triangle, curve piece and -- only when they are many -- analytic primitive, its cut and the ray-binning
// grid.  Analytic quads/cubes are few in most scenes and are then tested coherently by the kernel that creates a ray; from
// TGB_ANALYTIC_BVH_MIN (24) primitives on they get a third SAH tree instead (the reference keeps them in Embree's top-level
// user-geometry BVH, renderer/TraceableScene.hpp:112-134), so a ray's cost no longer grows with their number.
int prepare_bvh(BuildGeometry &g, HostScene &hs) {
    DScene &sc = hs.sc;
    size_t analytic_bvh_min = 24;
    if (const char *e = getenv("TGB_ANALYTIC_BVH_MIN")) analytic_bvh_min = size_t(std::max(1, atoi(e)));
    const bool analytic_in_bvh = hs.analytic.size() >= analytic_bvh_min;
    std::vector<Aabb> abounds(hs.analytic.size());
    for (size_t k = 0; k < hs.analytic.size(); ++k) abounds[k] = analytic_bounds(hs.prims[size_t(hs.analytic[k])]);
    SceneBvhInput in;
    in.tris = g.tris.data(); in.n_tris = uint32_t(g.tris.size());
    in.curve_boxes = g.curve_boxes.data(); in.curve_recs = g.curve_recs.data(); in.n_curve = uint32_t(g.curve_boxes.size());
    if (analytic_in_bvh) { in.analytic = abounds.data(); in.n_analytic = uint32_t(abounds.size()); }
    in.extent = std::max(std::max(std::fabs(sc.cam.pos.x), std::fabs(sc.cam.pos.y)), std::fabs(sc.cam.pos.z));
    SceneBvh &sb = hs.bvh;
    build_scene_bvh(in, bvh_options(), sb);
    const Bvh4 &bvh = sb.tree;
    if (!g.curve_boxes.empty()) {
        for (uint32_t pi : g.curve_prim) hs.tri_prim.push_back(pi);
        for (DPrim &p : hs.prims) if (p.type == TGB_PRIM_CURVES) p.tri_first += uint32_t(g.tris.size());
    }
    if (analytic_in_bvh) {                                // the ray-creating kernels loop over nothing: the list goes into leaf order
        const std::vector<int> desc_order = hs.analytic;
        for (size_t k = 0; k < sb.analytic_order.size(); ++k) hs.analytic[k] = desc_order[sb.analytic_order[k]];
    }
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
    if (sb.stack_need > uint32_t(kStackSize)) return refuse(TGB_ERR_UNSUPPORTED, "BVH depth %u (%u stack entries) exceeds the traversal stack", bvh.max_depth, sb.stack_need);
    // shading records follow the intersection records into BVH leaf order (one hop from a hit id)
    hs.tri_shade.resize(g.tri_shade.size());
    for (size_t k = 0; k < g.tris.size(); ++k) std::memcpy(&hs.tri_shade[4*k], &g.tri_shade[4*size_t(bvh.order[k])], 4*sizeof(float4));
    sc.n_analytic = analytic_in_bvh ? 0 : int(hs.analytic.size()); sc.analytic_base = analytic_in_bvh ? int(sb.isect.size()) : 0x7fffffff;
    sc.n_nodes = uint32_t(bvh.nodes.size()); sc.n_tris = uint32_t(g.tris.size());
    sc.n_curve_segs = uint32_t(g.curve_boxes.size());
    sc.qy = 0x3F80u;
    return TGB_OK;
}

// the direction matrices, then per dimension the XOR of the columns of every low byte (sampler_next1d): 1 MiB
std::vector<uint32_t> sobol_table() {
    std::vector<uint32_t> sobol(size_t(kSobolLowTable) + size_t(kSobolDims)*256);
    std::memcpy(sobol.data(), tgb_sobol_blob, size_t(kSobolLowTable)*4);
    for (uint32_t dim = 0; dim < kSobolDims; ++dim) {
        const uint32_t *m = sobol.data() + dim*32u;
        uint32_t *lo = sobol.data() + kSobolLowTable + dim*256u;
        lo[0] = 0u;
        for (uint32_t b = 1; b < 256; ++b) lo[b] = lo[b & (b - 1)] ^ m[__builtin_ctz(b)];
    }
    return sobol;
}

SceneKind scene_kind(const tgb_scene_desc *d, const HostScene &hs) {
    SceneKind s;
    s.has_curves = hs.sc.n_curve_segs != 0;
    for (int li : hs.lights) s.mesh_lights = s.mesh_lights || hs.prims[size_t(li)].type == TGB_PRIM_MESH;
    for (uint32_t i = 0; i < d->n_primitives; ++i) {
        const tgb_primitive &p = d->primitives[i];
        if (p.type == TGB_PRIM_INFINITE_SPHERE || p.type == TGB_PRIM_INFINITE_SPHERE_CAP || p.type == TGB_PRIM_SKYDOME) continue;
        for (uint32_t k = 0; k < p.bsdf_count; ++k) {
            uint32_t t = d->bsdfs[d->bsdf_slots[p.bsdf_first + k]].type;
            if (t != TGB_BSDF_NULL) s.bsdf_types |= 1u << std::min(t, 31u);
        }
    }
    const auto constant = [&](int t) { return hs.tex[size_t(t)].d.type == TGB_TEX_CONSTANT; };
    s.quad_lights = hs.inf_lights.empty();
    for (int li : hs.lights) s.quad_lights = s.quad_lights && hs.prims[size_t(li)].type == TGB_PRIM_QUAD;
    for (const DPrim &p : hs.prims) s.quad_lights = s.quad_lights && (p.emission_tex < 0 || constant(p.emission_tex));
    for (const DBsdf &b : hs.bsdfs) s.quad_lights = s.quad_lights && (b.type != TGB_BSDF_LAMBERT || constant(b.albedo_tex));
    return s;
}

// The reference's prepare step for a desc, or its refusal: TGB_ERR_INVALID / TGB_ERR_UNSUPPORTED with the reason in
// tgb200_last_error(NULL).  The settings are checked before (check_settings).
int prepare_scene(const tgb_scene_desc *d, HostScene &hs) {
    hs.sc.set = d->settings;
    prepare_camera(d->camera, hs.sc.cam);
    int rc;
    if ((rc = prepare_textures(d->textures, d->n_textures, hs.tex))) return rc;
    if ((rc = prepare_bsdfs(d, hs.tex, hs.bsdfs, hs.hair))) return rc;
    BuildGeometry g;
    if ((rc = prepare_primitives(d, hs.tex, hs.prims, hs.analytic, g, hs.tri_prim, hs.mesh_lights))) return rc;
    if ((rc = prepare_lights(d->textures, d->n_textures, hs.prims, hs.tex, hs.lights, hs.inf_lights))) return rc;
    if ((rc = prepare_bvh(g, hs))) return rc;
    hs.slots.assign(d->bsdf_slots, d->bsdf_slots + d->n_bsdf_slots);
    hs.sobol = sobol_table();
    hs.sc.n_prims = uint32_t(hs.prims.size()); hs.sc.n_lights = int(hs.lights.size()); hs.sc.n_inf_lights = int(hs.inf_lights.size());
    hs.kind = scene_kind(d, hs);
    return TGB_OK;
}

}  // namespace
}  // namespace tgb
