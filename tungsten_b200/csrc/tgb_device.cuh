// Device-side building blocks of the wavefront path tracer: fp32 vector math with the reference's
// operation order, Sobol/PCG sampling, textures, BSDF lobes, light sampling.
// Compiled with -fmad=false: the reference is built without FMA contraction (CMakeLists.txt:17-19),
// and radiance parity is judged against it.  Every function cites the reference code it replaces
// (paths relative to /root/reference/src/core).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/tgb200.h"

namespace tgb {

// ---------------------------------------------------------------- math (math/Vec.hpp:140-193)
struct V3 { float x, y, z; };
#define TGB_HD __host__ __device__ __forceinline__
#define TGB_D  __device__ __forceinline__

constexpr float PI_F = 3.1415926536f;             // math/Angle.hpp:8-16 (fp32 constexpr products)
constexpr float TWO_PI_F = PI_F*2.0f;
constexpr float INV_PI_F = 1.0f/PI_F;
constexpr float INV_TWO_PI_F = 0.5f*INV_PI_F;
constexpr float INV_FOUR_PI_F = 0.25f*INV_PI_F;

TGB_HD V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
TGB_HD V3 v3s(float a) { return v3(a, a, a); }
TGB_HD V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
TGB_HD V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
TGB_HD V3 operator*(V3 a, V3 b) { return v3(a.x*b.x, a.y*b.y, a.z*b.z); }
TGB_HD V3 operator/(V3 a, V3 b) { return v3(a.x/b.x, a.y/b.y, a.z/b.z); }
TGB_HD V3 operator*(V3 a, float s) { return v3(a.x*s, a.y*s, a.z*s); }
TGB_HD V3 operator/(V3 a, float s) { return v3(a.x/s, a.y/s, a.z/s); }
TGB_HD V3 operator-(V3 a) { return v3(-a.x, -a.y, -a.z); }
TGB_HD float dot(V3 a, V3 b) { float s = a.x*b.x; s += a.y*b.y; s += a.z*b.z; return s; }
TGB_HD V3 cross(V3 a, V3 b) { return v3(a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x); }
TGB_HD float length_sq(V3 a) { return dot(a, a); }
TGB_HD float length(V3 a) { return sqrtf(dot(a, a)); }
TGB_HD V3 normalize(V3 a) { float inv = 1.0f/length(a); return v3(a.x*inv, a.y*inv, a.z*inv); }
TGB_HD float max_comp(V3 a) { float m = a.x; if (a.y > m) m = a.y; if (a.z > m) m = a.z; return m; }
TGB_HD float sum(V3 a) { float s = a.x; s += a.y; s += a.z; return s; }
TGB_HD float avg(V3 a) { return sum(a)*(1.0f/3.0f); }
TGB_HD bool is_zero(V3 a) { return a.x == 0.0f && a.y == 0.0f && a.z == 0.0f; }       // Vec.hpp:429-435
TGB_HD V3 vabs(V3 a) { return v3(fabsf(a.x), fabsf(a.y), fabsf(a.z)); }
TGB_HD float maxf(float a, float b) { return a > b ? a : b; }                         // math/MathUtil.hpp max/min
TGB_HD float minf(float a, float b) { return a < b ? a : b; }
TGB_HD float sqr(float a) { return a*a; }
TGB_HD float sgnE(float x) { return x < 0.0f ? -1.0f : 1.0f; }
TGB_HD V3 m3mul(const float *m, V3 b) {                                               // Mat4f::transformVector
    return v3(m[0]*b.x + m[1]*b.y + m[2]*b.z, m[3]*b.x + m[4]*b.y + m[5]*b.z, m[6]*b.x + m[7]*b.y + m[8]*b.z);
}
TGB_HD float comp(V3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

struct Frame { V3 n, t, b; };
TGB_HD Frame frame_from_normal(V3 n) {                                                // math/TangentFrame.hpp:22-31
    Frame f; f.n = n;
    float sign = copysignf(1.0f, n.z);
    const float a = -1.0f/(sign + n.z);
    const float b = n.x*n.y*a;
    f.t = v3(1.0f + sign*n.x*n.x*a, sign*b, -sign*n.x);
    f.b = v3(b, sign + n.y*n.y*a, -n.y);
    return f;
}
TGB_HD V3 to_local(const Frame &f, V3 p) { return v3(dot(f.t, p), dot(f.b, p), dot(f.n, p)); }
TGB_HD V3 to_global(const Frame &f, V3 p) { return f.t*p.x + f.b*p.y + f.n*p.z; }

// ---------------------------------------------------------------- integer hashing / RNG
TGB_HD uint32_t hash32(uint32_t x) {                                                  // math/MathUtil.hpp:120-128
    x = ~x + (x << 15); x = x ^ (x >> 12); x = x + (x << 2); x = x ^ (x >> 4); x = x*2057u; x = x ^ (x >> 16);
    return x;
}
TGB_HD uint32_t pcg_next(uint64_t &state) {                                           // sampling/UniformSampler.hpp:40-47
    uint64_t old = state;
    state = old*6364136223846793005ULL + 1ULL;
    uint32_t xs = uint32_t(((old >> 18u) ^ old) >> 27u);
    uint32_t rot = uint32_t(old >> 59u);
    return (xs >> rot) | (xs << (uint32_t(-int32_t(rot)) & 31));
}
TGB_HD float normalized_uint(uint32_t i) {                                            // math/BitManip.hpp:47-50
#ifdef __CUDA_ARCH__
    return __uint_as_float((i >> 9u) | 0x3F800000u) - 1.0f;
#else
    union { uint32_t u; float f; } c; c.u = (i >> 9u) | 0x3F800000u; return c.f - 1.0f;
#endif
}

// ---------------------------------------------------------------- device scene
enum : uint32_t { LOBE_GLOSSY_R = 1, LOBE_GLOSSY_T = 2, LOBE_DIFFUSE_R = 4, LOBE_DIFFUSE_T = 8, LOBE_SPEC_R = 16,
                  LOBE_SPEC_T = 32, LOBE_ANISO = 64, LOBE_FORWARD = 128, LOBE_SPECULAR = 48,
                  LOBE_TRANSMISSIVE = 2 | 8 | 32, LOBE_ALL = 2 | 8 | 32 | 1 | 4 | 16 | 64 };   // bsdfs/BsdfLobes.hpp:13-34
constexpr uint32_t LOBE_ALL_BUT_SPECULAR = ~uint32_t(LOBE_SPECULAR | LOBE_FORWARD);

struct DTex {
    uint32_t type; V3 value, value2; int res_u, res_v; uint32_t flags;
    const float *texels;                                         // bitmap RGB fp32
    const float *marg_pdf, *marg_cdf, *pdf, *cdf;                // spherical importance map (env lights)
    V3 avg;
};
struct DBsdf {
    uint32_t type, lobes, dist; int albedo_tex, rough_tex;
    float ior, inv_ior; V3 eta, k; V3 scaled_sigma_a; float avg_transmittance, diffuse_fresnel, substrate_weight;
    uint32_t enable_t; int substrate;
    // hair (HairBcsdf.cpp:422-446): lobe variances v_p = beta_p^2, cuticle tilt, and per lobe p = R, TT, TRT the 64x64 RGB table,
    // the 64 normalised row pdfs / cdfs (65 entries per row) and the row sums
    float hair_v[3], hair_scale_rad; const float *hair_table[3], *hair_pdfs[3], *hair_cdfs[3], *hair_sums[3];
};
enum : uint32_t { PF_EMISSIVE = 1, PF_SAMPLABLE = 2, PF_INFINITE = 4, PF_SMOOTH = 8, PF_SKYDOME = 16 };
struct DPrim {
    uint32_t type, flags; int emission_tex;
    uint32_t tri_first, n_tris, bsdf_first, bsdf_count;
    V3 base, edge0, edge1, normal; float inv_uv_sq0, inv_uv_sq1, area;      // quad; infinite sphere cap: normal = cap direction, area = cos(cap angle)
    V3 pos, scale; float rot[9], inv_rot[9];                                // cube / infinite sphere rotation
    float total_area; const float *tri_pdf, *tri_cdf; const float *light_verts;   // emissive meshes: p0 p1 p2 per tri
    uint32_t curve_mode;                                                    // curves: TGB_CURVE_*; tri_first/n_tris = its segments' global ids
};
struct DCamera { V3 pos; float m[9]; float plane_dist, ratio, pixel_size_x; uint32_t res_x, res_y, filter; float filter_cdf[32]; float filter_bin; };

struct DScene {
    DCamera cam; tgb_settings set;
    const DPrim *prims; uint32_t n_prims;
    const DBsdf *bsdfs; const uint32_t *slots; const DTex *tex;
    const int *lights; int n_lights; const int *inf_lights; int n_inf_lights;
    const int *analytic; int n_analytic;    // quads/cubes: the list the ray-creating kernels loop over (n_analytic = 0 when they are BVH leaves)
    int analytic_base;                      // first leaf position of the analytic primitives when they are in the BVH, else INT_MAX
    // triangles: intersection records in BVH leaf order (3 x float4 each), leaf order -> global id,
    // global id -> primitive, shading records ALSO in leaf order (4 x float4 each: 3 normals, 3 uvs, material | primitive << 10)
    const float4 *tri_isect; const uint32_t *tri_global; const uint32_t *tri_prim; const float4 *tri_shade;
    uint32_t n_nodes; uint32_t n_tris;
    // quantised nodes (QNode4, 64 B = 4 x uint4, bvh_build.h), depth-first from the root
    const uint4 *qnodes;
    uint32_t qy;                // = 0x3F80: the constant bytes of 1 + q*2^-15 (see qplane in tgb_wavefront.cuh)
    // curve segments share the arrays above: records n_tris.. of tri_isect hold a segment's three nodes (x, y, z, width),
    // tri_global / tri_prim continue with global ids n_tris + segment
    uint32_t n_curve_segs;          // BVH primitives for curves = kCurvePieces sub-ranges per segment
    // "cut": <= 16 boxes of the BVH's top levels that together cover every triangle (same padded boxes the nodes hold).
    // A ray that misses all of them is answered by the kernel that creates it and never reaches a traversal kernel.
    // (8-byte aligned: mesh_cut_hit reads two boxes' planes per 64-bit load from the kernel parameters)
    int n_cut; alignas(8) float cut[6][16];        // lo.x, hi.x, lo.y, hi.y, lo.z, hi.z
    // where an any-hit shadow query enters the tree: the QNode4 index (or leaf code) below each cut box; cut_entry = 0 starts
    // every query at the root instead (TGB_SHADOW_CUT_ENTRY=0, for A/B comparisons)
    int32_t cut_link[16]; int cut_entry;
    V3 bin_lo, bin_inv;         // ray-binning grid over the scene bounds: cell = (o - bin_lo)*bin_inv, 16 cells per axis
    const uint32_t *sobol;      // 1024 x 32 direction matrices, then the 1024 x 256 low-byte table (sampler_next1d)
    const float4 *lambert;      // k_shade's emitter set 1 only: per BSDF its constant albedo and type | lobes << 16 (lambert_rec)
};

// ---------------------------------------------------------------- sampler
// SobolPathSampler (sampling/SobolPathSampler.hpp:12-84) with the per-path reseed of the supplemental
// PCG stream (parity contract, DESIGN.md section 3).
struct Sampler { const uint32_t *sobol; uint64_t pcg; uint32_t scramble, index, dimension; };

TGB_D void sampler_start(Sampler &s, const uint32_t *sobol, uint32_t tile_seed, uint32_t pixel_id, uint32_t sample) {
    s.sobol = sobol;
    s.scramble = tile_seed ^ hash32(pixel_id);
    s.index = sample; s.dimension = 0;
    s.pcg = (uint64_t(s.scramble) << 32) | uint64_t(hash32(sample));
}
TGB_D float sampler_pcg1d(Sampler &s) { return normalized_uint(pcg_next(s.pcg)); }
TGB_D bool sampler_boolean(Sampler &s, float p_true) { return sampler_pcg1d(s) < p_true; }
// The value is scramble ^ the XOR of the matrix columns of the set bits of index' = (index & ~0xFF) | ((index + scramble) & 0xFF)
// (thirdparty/sobol/sobol.h:39-53).  The two parts of index' share no bits and XOR is associative and commutative, so the low
// byte's columns come from one load of a table of all 256 of their XORs (kSobolLowTable words after the matrices), and only
// the high bits -- zero to two set bits at the usual sample counts, nearly uniform across a warp -- walk the matrix.
constexpr uint32_t kSobolDims = 1024, kSobolLowTable = kSobolDims*32u;
TGB_D float sampler_next1d(Sampler &s) {
    if (s.dimension >= kSobolDims) return sampler_pcg1d(s);
    uint32_t result = s.scramble ^ __ldg(s.sobol + kSobolLowTable + s.dimension*256u + ((s.index + s.scramble) & 0xFFu));
    uint32_t index = s.index & ~0xFFu;
    const uint32_t *m = s.sobol + s.dimension*32u;
    s.dimension++;
    while (index) {
        int b = __ffs(int(index)) - 1;
        result ^= __ldg(m + b);
        index &= index - 1;
    }
    return normalized_uint(result);
}

// ---------------------------------------------------------------- textures
TGB_D V3 bitmap_texel(const DTex &t, int x, int y) {
    const float *p = t.texels + 3*(size_t(y)*t.res_u + x);
    return v3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}
// CONST: every texture the caller can reach is constant (emitter set 1, k_shade): the lookups are compiled out
template <bool CONST = false>
TGB_D V3 tex_eval(const DTex &t, float u, float v) {
    if (CONST || t.type == TGB_TEX_CONSTANT) return t.value;                          // textures/ConstantTexture.cpp:50-58
    if (t.type == TGB_TEX_CHECKER) {                                                  // textures/CheckerTexture.cpp:64-69
        int ui = int(u*float(t.res_u)), vi = int(v*float(t.res_v));
        return ((ui ^ vi) & 1) ? t.value : t.value2;
    }
    // BitmapTexture::operator[] (textures/BitmapTexture.cpp:298-352)
    float fu = u*t.res_u, fv = (1.0f - v)*t.res_v;
    bool linear = t.flags & 1, clampm = (t.flags >> 1) & 1;
    if (linear) { fu -= 0.5f; fv -= 0.5f; }
    int iu0 = fu < 0.0f ? -int(-fu) - 1 : int(fu);
    int iv0 = fv < 0.0f ? -int(-fv) - 1 : int(fv);
    int iu1 = iu0 + 1, iv1 = iv0 + 1;
    fu -= iu0; fv -= iv0;
    int w = t.res_u, h = t.res_v;
    if (clampm) {
        iu0 = min(max(iu0, 0), w - 1); iu1 = min(max(iu1, 0), w - 1);
        iv0 = min(max(iv0, 0), h - 1); iv1 = min(max(iv1, 0), h - 1);
    } else {
        iu0 = ((iu0 % w) + w) % w; iu1 = ((iu1 % w) + w) % w;
        iv0 = ((iv0 % h) + h) % h; iv1 = ((iv1 % h) + h) % h;
    }
    if (!linear) return bitmap_texel(t, iu0, iv0);
    V3 x00 = bitmap_texel(t, iu0, iv0), x01 = bitmap_texel(t, iu1, iv0);
    V3 x10 = bitmap_texel(t, iu0, iv1), x11 = bitmap_texel(t, iu1, iv1);
    V3 a = x00*(1.0f - fu) + x01*fu;
    V3 b = x10*(1.0f - fu) + x11*fu;
    return a*(1.0f - fv) + b*fv;
}

// ---------------------------------------------------------------- camera filter (cameras/ReconstructionFilter.hpp:86-103)
TGB_D float filter_sample1(const DCamera &c, float xi) {
    const int R = 31;
    bool negative = xi < 0.5f;
    xi = negative ? xi*2.0f : (xi - 0.5f)*2.0f;
    int idx = R - 1;
    for (int i = 0; i < R - 1; ++i) if (xi < c.filter_cdf[i]) { idx = i; break; }
    float pdf = c.filter_cdf[idx] - c.filter_cdf[idx - 1];
    float u = c.filter_bin*(idx + (xi - c.filter_cdf[idx - 1])/pdf);
    return negative ? -u : u;
}

// ---------------------------------------------------------------- Fresnel / microfacet
TGB_D float dielectric_reflectance(float eta, float cosThetaI, float &cosThetaT) {    // bsdfs/Fresnel.hpp:75-92
    if (cosThetaI < 0.0f) { eta = 1.0f/eta; cosThetaI = -cosThetaI; }
    float sinThetaTSq = eta*eta*(1.0f - cosThetaI*cosThetaI);
    if (sinThetaTSq > 1.0f) { cosThetaT = 0.0f; return 1.0f; }
    cosThetaT = sqrtf(maxf(1.0f - sinThetaTSq, 0.0f));
    float Rs = (eta*cosThetaI - cosThetaT)/(eta*cosThetaI + cosThetaT);
    float Rp = (eta*cosThetaT - cosThetaI)/(eta*cosThetaT + cosThetaI);
    return (Rs*Rs + Rp*Rp)*0.5f;
}
TGB_D float dielectric_reflectance(float eta, float c) { float t; return dielectric_reflectance(eta, c, t); }
TGB_D float conductor_reflectance(float eta, float k, float cosThetaI) {              // bsdfs/Fresnel.hpp:102-118
    float cosThetaISq = cosThetaI*cosThetaI;
    float sinThetaISq = maxf(1.0f - cosThetaISq, 0.0f);
    float sinThetaIQu = sinThetaISq*sinThetaISq;
    float innerTerm = eta*eta - k*k - sinThetaISq;
    float aSqPlusBSq = sqrtf(maxf(innerTerm*innerTerm + 4.0f*eta*eta*k*k, 0.0f));
    float a = sqrtf(maxf((aSqPlusBSq + innerTerm)*0.5f, 0.0f));
    float Rs = ((aSqPlusBSq + cosThetaISq) - (2.0f*a*cosThetaI))/((aSqPlusBSq + cosThetaISq) + (2.0f*a*cosThetaI));
    float Rp = ((cosThetaISq*aSqPlusBSq + sinThetaIQu) - (2.0f*a*cosThetaI*sinThetaISq))/
               ((cosThetaISq*aSqPlusBSq + sinThetaIQu) + (2.0f*a*cosThetaI*sinThetaISq));
    return 0.5f*(Rs + Rs*Rp);
}
TGB_D V3 conductor_reflectance(V3 eta, V3 k, float c) {
    return v3(conductor_reflectance(eta.x, k.x, c), conductor_reflectance(eta.y, k.y, c), conductor_reflectance(eta.z, k.z, c));
}
// bsdfs/Microfacet.hpp:27-130
TGB_D float mf_roughness_to_alpha(uint32_t dist, float roughness) {
    roughness = maxf(roughness, 1e-3f);
    if (dist == TGB_DIST_PHONG) return 2.0f/(roughness*roughness) - 2.0f;
    return roughness;
}
TGB_D float mf_D(uint32_t dist, float alpha, V3 m) {
    if (m.z <= 0.0f) return 0.0f;
    if (dist == TGB_DIST_PHONG) return (alpha + 2.0f)*INV_TWO_PI_F*float(pow(double(m.z), double(alpha)));
    float alphaSq = alpha*alpha, cosThetaSq = m.z*m.z;
    float tanThetaSq = maxf(1.0f - cosThetaSq, 0.0f)/cosThetaSq;
    float cosThetaQu = cosThetaSq*cosThetaSq;
    if (dist == TGB_DIST_BECKMANN) return INV_PI_F*expf(-tanThetaSq/alphaSq)/(alphaSq*cosThetaQu);
    return alphaSq*INV_PI_F/(cosThetaQu*sqr(alphaSq + tanThetaSq));
}
TGB_D float mf_G1(uint32_t dist, float alpha, V3 v, V3 m) {
    if (dot(v, m)*v.z <= 0.0f) return 0.0f;
    float cosThetaSq = v.z*v.z;
    if (dist == TGB_DIST_GGX) {
        float alphaSq = alpha*alpha;
        float tanThetaSq = maxf(1.0f - cosThetaSq, 0.0f)/cosThetaSq;
        return 2.0f/(1.0f + sqrtf(1.0f + alphaSq*tanThetaSq));
    }
    float tanTheta = fabsf(sqrtf(maxf(1.0f - cosThetaSq, 0.0f))/v.z);
    float a = dist == TGB_DIST_BECKMANN ? 1.0f/(alpha*tanTheta) : sqrtf(0.5f*alpha + 1.0f)/tanTheta;
    if (a < 1.6f) return (3.535f*a + 2.181f*a*a)/(1.0f + 2.276f*a + 2.577f*a*a);
    return 1.0f;
}
TGB_D float mf_G(uint32_t dist, float alpha, V3 i, V3 o, V3 m) { return mf_G1(dist, alpha, i, m)*mf_G1(dist, alpha, o, m); }
TGB_D float mf_pdf(uint32_t dist, float alpha, V3 m) { return mf_D(dist, alpha, m)*m.z; }
TGB_D V3 mf_sample(uint32_t dist, float alpha, float xix, float xiy) {
    float phi = xiy*TWO_PI_F;
    float cosTheta;
    if (dist == TGB_DIST_BECKMANN) { float tanThetaSq = -alpha*alpha*logf(1.0f - xix); cosTheta = 1.0f/sqrtf(1.0f + tanThetaSq); }
    else if (dist == TGB_DIST_PHONG) cosTheta = float(pow(double(xix), 1.0/(double(alpha) + 2.0)));
    else { float tanThetaSq = alpha*alpha*xix/(1.0f - xix); cosTheta = 1.0f/sqrtf(1.0f + tanThetaSq); }
    float r = sqrtf(maxf(1.0f - cosTheta*cosTheta, 0.0f));
    return v3(cosf(phi)*r, sinf(phi)*r, cosTheta);
}
TGB_D V3 cosine_hemisphere(float xix, float xiy) {                                     // sampling/SampleWarp.hpp:42-52
    float phi = xix*TWO_PI_F;
    float r = sqrtf(xiy);
    return v3(cosf(phi)*r, sinf(phi)*r, sqrtf(maxf(1.0f - xiy, 0.0f)));
}
TGB_D float cosine_hemisphere_pdf(V3 p) { return fabsf(p.z)*INV_PI_F; }
TGB_D float power_heuristic(float a, float b) { return (a*a)/(a*a + b*b); }            // SampleWarp.hpp:189-192

// ---------------------------------------------------------------- surface records
struct Surface {            // IntersectionInfo (primitives/IntersectionInfo.hpp:11-22) + what evalDirect needs
    V3 Ng, Ns, p, w; float u, v; int prim, bsdf; bool backside;
    float eps;              // IntersectionInfo::epsilon: 5e-4 (TraceableScene.hpp:39), raised by curves (Curves.cpp:512-515)
    bool curve; V3 tangent; // curve hits: unnormalised BSpline::quadraticDeriv at the hit (for Curves::tangentSpace)
};
struct Event {              // SurfaceScatterEvent (samplerecords/SurfaceScatterEvent.hpp:14-66)
    Frame frame; V3 wi, wo, weight; float pdf; uint32_t requested, sampled; bool flipped;
};

TGB_D V3 bsdf_albedo(const DScene &sc, const DBsdf &b, const Surface &s) { return tex_eval(sc.tex[b.albedo_tex], s.u, s.v); }
TGB_D float bsdf_roughness(const DScene &sc, const DBsdf &b, const Surface &s) { return tex_eval(sc.tex[b.rough_tex], s.u, s.v).x; }
TGB_D bool check_reflection_constraint(V3 wi, V3 wo) {                                 // bsdfs/Bsdf.hpp:43-46
    return fabsf(wi.z*wo.z - wi.x*wo.x - wi.y*wo.y - 1.0f) < 1e-3f;
}
TGB_D bool check_refraction_constraint(V3 wi, V3 wo, float eta, float cosThetaT) {      // bsdfs/Bsdf.hpp:49-53
    float dotP = -wi.x*wo.x*eta - wi.y*wo.y*eta - copysignf(cosThetaT, wi.z)*wo.z;
    return fabsf(dotP - 1.0f) < 1e-3f;
}
TGB_D V3 vexp(V3 a) { return v3(expf(a.x), expf(a.y), expf(a.z)); }

// RoughDielectricBsdf::sampleBase / evalBase / pdfBase (bsdfs/RoughDielectricBsdf.cpp:55-131,133-164,198-234)
TGB_D bool rd_sample_base(Sampler &smp, Event &e, bool sampleR, bool sampleT, float roughness, float ior, uint32_t dist) {
    float wiDotN = e.wi.z;
    float eta = wiDotN < 0.0f ? ior : 1.0f/ior;
    float sampleRoughness = (1.2f - 0.2f*sqrtf(fabsf(wiDotN)))*roughness;
    float alpha = mf_roughness_to_alpha(dist, roughness);
    float sampleAlpha = mf_roughness_to_alpha(dist, sampleRoughness);
    float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
    V3 m = mf_sample(dist, sampleAlpha, xa, xb);
    float pm = mf_pdf(dist, sampleAlpha, m);
    if (pm < 1e-10f) return false;
    float wiDotM = dot(e.wi, m);
    float cosThetaT = 0.0f;
    float F = dielectric_reflectance(1.0f/ior, wiDotM, cosThetaT);
    float etaM = wiDotM < 0.0f ? ior : 1.0f/ior;
    bool reflect;
    if (sampleR && sampleT) reflect = sampler_boolean(smp, F);
    else if (sampleT) { if (F == 1.0f) return false; reflect = false; }
    else if (sampleR) reflect = true;
    else return false;
    if (reflect) e.wo = m*(2.0f*wiDotM) - e.wi;
    else e.wo = m*(etaM*wiDotM - sgnE(wiDotM)*cosThetaT) - e.wi*etaM;
    float woDotN = e.wo.z;
    bool reflected = wiDotN*woDotN > 0.0f;
    if (reflected != reflect) return false;
    float woDotM = dot(e.wo, m);
    float G = mf_G(dist, alpha, e.wi, e.wo, m);
    float D = mf_D(dist, alpha, m);
    e.weight = v3s(fabsf(wiDotM)*G*D/(fabsf(wiDotN)*pm));
    if (reflect) { e.pdf = pm*0.25f/fabsf(wiDotM); e.sampled = LOBE_GLOSSY_R; }
    else { e.pdf = pm*fabsf(woDotM)/sqr(eta*wiDotM + woDotM); e.sampled = LOBE_GLOSSY_T; }
    if (sampleR && sampleT) { if (reflect) e.pdf *= F; else e.pdf *= 1.0f - F; }
    else { if (reflect) e.weight = e.weight*F; else e.weight = e.weight*(1.0f - F); }
    return true;
}
TGB_D void rd_microfacet_normal(const Event &e, bool reflect, float eta, float wiDotN, V3 &m) {
    if (reflect) m = normalize(e.wi + e.wo)*sgnE(wiDotN);
    else m = -normalize(e.wi*eta + e.wo);
}
TGB_D V3 rd_eval_base(const Event &e, bool sampleR, bool sampleT, float roughness, float ior, uint32_t dist) {
    float wiDotN = e.wi.z, woDotN = e.wo.z;
    bool reflect = wiDotN*woDotN >= 0.0f;
    if ((reflect && !sampleR) || (!reflect && !sampleT)) return v3s(0.0f);
    float alpha = mf_roughness_to_alpha(dist, roughness);
    float eta = wiDotN < 0.0f ? ior : 1.0f/ior;
    V3 m; rd_microfacet_normal(e, reflect, eta, wiDotN, m);
    float wiDotM = dot(e.wi, m), woDotM = dot(e.wo, m);
    float F = dielectric_reflectance(1.0f/ior, wiDotM);
    float G = mf_G(dist, alpha, e.wi, e.wo, m);
    float D = mf_D(dist, alpha, m);
    if (reflect) return v3s((F*G*D*0.25f)/fabsf(wiDotN));
    return v3s(fabsf(wiDotM*woDotM)*(1.0f - F)*G*D/(sqr(eta*wiDotM + woDotM)*fabsf(wiDotN)));
}
TGB_D float rd_pdf_base(const Event &e, bool sampleR, bool sampleT, float roughness, float ior, uint32_t dist) {
    float wiDotN = e.wi.z, woDotN = e.wo.z;
    bool reflect = wiDotN*woDotN >= 0.0f;
    if ((reflect && !sampleR) || (!reflect && !sampleT)) return 0.0f;
    float sampleRoughness = (1.2f - 0.2f*sqrtf(fabsf(wiDotN)))*roughness;
    float sampleAlpha = mf_roughness_to_alpha(dist, sampleRoughness);
    float eta = wiDotN < 0.0f ? ior : 1.0f/ior;
    V3 m; rd_microfacet_normal(e, reflect, eta, wiDotN, m);
    float wiDotM = dot(e.wi, m), woDotM = dot(e.wo, m);
    float F = dielectric_reflectance(1.0f/ior, wiDotM);
    float pm = mf_pdf(dist, sampleAlpha, m);
    float pdf;
    if (reflect) pdf = pm*0.25f/fabsf(wiDotM);
    else pdf = pm*fabsf(woDotM)/sqr(eta*wiDotM + woDotM);
    if (sampleR && sampleT) { if (reflect) pdf *= F; else pdf *= 1.0f - F; }
    return pdf;
}
TGB_D V3 plastic_substrate(const DBsdf &b, V3 albedo, float Fi, float Fo, float eta) {
    V3 denom = v3s(1.0f) - albedo*b.diffuse_fresnel;
    return (albedo/denom)*((1.0f - Fi)*(1.0f - Fo)*eta*eta);
}
TGB_D float bsdf_eta(const DBsdf &b, const Event &e) {                                 // bsdfs/Bsdf.hpp:99-103; RoughDielectricBsdf.cpp:274-280
    if (b.type == TGB_BSDF_ROUGH_DIELECTRIC || b.type == TGB_BSDF_DIELECTRIC) {         // DielectricBsdf.cpp:166-172
        if (e.wi.z*e.wo.z >= 0.0f) return 1.0f;
        return e.wi.z < 0.0f ? b.ior : b.inv_ior;
    }
    return 1.0f;
}

// Bsdf::sample(event, adjoint=false) (bsdfs/Bsdf.hpp:71-83) over the per-lobe sample() bodies
TGB_D bool bsdf_sample_base(const DScene &sc, const DBsdf &b, const Surface &s, Sampler &smp, Event &e) {
    bool ok = false;
    switch (b.type) {
    case TGB_BSDF_LAMBERT: {                                                           // bsdfs/LambertBsdf.cpp:27-38
        if (!(e.requested & LOBE_DIFFUSE_R)) break;
        if (e.wi.z <= 0.0f) break;
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        e.wo = cosine_hemisphere(xa, xb);
        e.pdf = cosine_hemisphere_pdf(e.wo);
        e.weight = bsdf_albedo(sc, b, s);
        e.sampled = LOBE_DIFFUSE_R;
        ok = true; break; }
    case TGB_BSDF_ROUGH_CONDUCTOR: {                                                   // bsdfs/RoughConductorBsdf.cpp:60-90
        if (!(e.requested & LOBE_GLOSSY_R)) break;
        if (e.wi.z <= 0.0f) break;
        float roughness = bsdf_roughness(sc, b, s);
        float alpha = mf_roughness_to_alpha(b.dist, roughness);
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        V3 m = mf_sample(b.dist, alpha, xa, xb);
        float wiDotM = dot(e.wi, m);
        e.wo = m*(2.0f*wiDotM) - e.wi;
        if (wiDotM <= 0.0f || e.wo.z <= 0.0f) break;
        float G = mf_G(b.dist, alpha, e.wi, e.wo, m);
        float D = mf_D(b.dist, alpha, m);
        float mPdf = mf_pdf(b.dist, alpha, m);
        float pdf = mPdf*0.25f/wiDotM;
        float weight = wiDotM*G*D/(e.wi.z*mPdf);
        V3 F = conductor_reflectance(b.eta, b.k, wiDotM);
        e.pdf = pdf;
        e.weight = bsdf_albedo(sc, b, s)*(F*weight);
        e.sampled = LOBE_GLOSSY_R;
        ok = true; break; }
    case TGB_BSDF_ROUGH_DIELECTRIC: {                                                  // RoughDielectricBsdf.cpp:236-244
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0;
        bool sampleT = (e.requested & LOBE_GLOSSY_T) != 0 && b.enable_t;
        float roughness = bsdf_roughness(sc, b, s);
        ok = rd_sample_base(smp, e, sampleR, sampleT, roughness, b.ior, b.dist);
        e.weight = e.weight*bsdf_albedo(sc, b, s);
        break; }
    case TGB_BSDF_MIRROR: {                                                            // bsdfs/MirrorBsdf.cpp:28-37
        if (!(e.requested & LOBE_SPEC_R)) break;
        e.wo = v3(-e.wi.x, -e.wi.y, e.wi.z);
        e.pdf = 1.0f;
        e.sampled = LOBE_SPEC_R;
        e.weight = bsdf_albedo(sc, b, s);
        ok = true; break; }
    case TGB_BSDF_CONDUCTOR: {                                                         // bsdfs/ConductorBsdf.cpp:58-68
        if (!(e.requested & LOBE_SPEC_R)) break;
        e.wo = v3(-e.wi.x, -e.wi.y, e.wi.z);
        e.pdf = 1.0f;
        e.weight = bsdf_albedo(sc, b, s)*conductor_reflectance(b.eta, b.k, e.wi.z);
        e.sampled = LOBE_SPEC_R;
        ok = true; break; }
    case TGB_BSDF_DIELECTRIC: {                                                        // bsdfs/DielectricBsdf.cpp:49-87
        bool sampleR = (e.requested & LOBE_SPEC_R) != 0;
        bool sampleT = (e.requested & LOBE_SPEC_T) != 0 && b.enable_t;
        float eta = e.wi.z < 0.0f ? b.ior : b.inv_ior;
        float cosThetaT = 0.0f;
        float F = dielectric_reflectance(eta, fabsf(e.wi.z), cosThetaT);
        float reflectionProbability;
        if (sampleR && sampleT) reflectionProbability = F;
        else if (sampleR) reflectionProbability = 1.0f;
        else if (sampleT) reflectionProbability = 0.0f;
        else break;
        if (sampler_boolean(smp, reflectionProbability)) {
            e.wo = v3(-e.wi.x, -e.wi.y, e.wi.z);
            e.pdf = reflectionProbability;
            e.sampled = LOBE_SPEC_R;
            e.weight = sampleT ? v3s(1.0f) : v3s(F);
        } else {
            if (F == 1.0f) break;
            e.wo = v3(-e.wi.x*eta, -e.wi.y*eta, -copysignf(cosThetaT, e.wi.z));
            e.pdf = 1.0f - reflectionProbability;
            e.sampled = LOBE_SPEC_T;
            e.weight = sampleR ? v3s(1.0f) : v3s(1.0f - F);
        }
        e.weight = e.weight*bsdf_albedo(sc, b, s);
        ok = true; break; }
    case TGB_BSDF_PLASTIC: {                                                           // bsdfs/PlasticBsdf.cpp:45-88
        if (e.wi.z <= 0.0f) break;
        bool sampleR = (e.requested & LOBE_SPEC_R) != 0, sampleT = (e.requested & LOBE_DIFFUSE_R) != 0;
        V3 wi = e.wi;
        float eta = 1.0f/b.ior;
        float Fi = dielectric_reflectance(eta, wi.z);
        float substrateWeight = b.avg_transmittance*(1.0f - Fi);
        float specularWeight = Fi;
        float specularProbability;
        if (sampleR && sampleT) specularProbability = specularWeight/(specularWeight + substrateWeight);
        else if (sampleR) specularProbability = 1.0f;
        else if (sampleT) specularProbability = 0.0f;
        else break;
        if (sampleR && sampler_boolean(smp, specularProbability)) {
            e.wo = v3(-wi.x, -wi.y, wi.z);
            e.pdf = specularProbability;
            e.weight = v3s(Fi/specularProbability);
            e.sampled = LOBE_SPEC_R;
        } else {
            float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
            V3 wo = cosine_hemisphere(xa, xb);
            float Fo = dielectric_reflectance(eta, wo.z);
            V3 diffuseAlbedo = bsdf_albedo(sc, b, s);
            e.wo = wo;
            e.weight = plastic_substrate(b, diffuseAlbedo, Fi, Fo, eta);
            if (max_comp(b.scaled_sigma_a) > 0.0f)
                e.weight = e.weight*vexp(b.scaled_sigma_a*(-1.0f/e.wo.z - 1.0f/e.wi.z));
            e.pdf = cosine_hemisphere_pdf(e.wo)*(1.0f - specularProbability);
            e.weight = e.weight/(1.0f - specularProbability);
            e.sampled = LOBE_DIFFUSE_R;
        }
        ok = true; break; }
    case TGB_BSDF_ROUGH_PLASTIC: {                                                     // bsdfs/RoughPlasticBsdf.cpp:54-113
        if (e.wi.z <= 0.0f) break;
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & LOBE_DIFFUSE_R) != 0;
        if (!sampleR && !sampleT) break;
        V3 wi = e.wi;
        float eta = 1.0f/b.ior;
        float Fi = dielectric_reflectance(eta, wi.z);
        float substrateWeight = b.substrate_weight*b.avg_transmittance*(1.0f - Fi);
        float specularWeight = Fi;
        float specularProbability = specularWeight/(specularWeight + substrateWeight);
        if (sampleR && (sampler_boolean(smp, specularProbability) || !sampleT)) {
            float roughness = bsdf_roughness(sc, b, s);
            if (!rd_sample_base(smp, e, true, false, roughness, b.ior, b.dist)) break;
            if (sampleT) {
                V3 diffuseAlbedo = bsdf_albedo(sc, b, s);
                float Fo = dielectric_reflectance(eta, e.wo.z);
                V3 brdfSubstrate = (plastic_substrate(b, diffuseAlbedo, Fi, Fo, eta)*INV_PI_F)*e.wo.z;
                V3 brdfSpecular = e.weight*e.pdf;
                float pdfSubstrate = cosine_hemisphere_pdf(e.wo)*(1.0f - specularProbability);
                float pdfSpecular = e.pdf*specularProbability;
                e.weight = (brdfSpecular + brdfSubstrate)/(pdfSpecular + pdfSubstrate);
                e.pdf = pdfSpecular + pdfSubstrate;
            }
        } else {
            float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
            V3 wo = cosine_hemisphere(xa, xb);
            float Fo = dielectric_reflectance(eta, wo.z);
            V3 diffuseAlbedo = bsdf_albedo(sc, b, s);
            e.wo = wo;
            e.weight = plastic_substrate(b, diffuseAlbedo, Fi, Fo, eta);
            if (max_comp(b.scaled_sigma_a) > 0.0f)
                e.weight = e.weight*vexp(b.scaled_sigma_a*(-1.0f/e.wo.z - 1.0f/e.wi.z));
            e.pdf = cosine_hemisphere_pdf(e.wo);
            if (sampleR) {
                float roughness = bsdf_roughness(sc, b, s);
                V3 brdfSubstrate = e.weight*e.pdf;
                float pdfSubstrate = e.pdf*(1.0f - specularProbability);
                V3 brdfSpecular = rd_eval_base(e, true, false, roughness, b.ior, b.dist);
                float pdfSpecular = rd_pdf_base(e, true, false, roughness, b.ior, b.dist);
                pdfSpecular *= specularProbability;
                e.weight = (brdfSpecular + brdfSubstrate)/(pdfSpecular + pdfSubstrate);
                e.pdf = pdfSpecular + pdfSubstrate;
            }
            e.sampled = LOBE_DIFFUSE_R;
        }
        ok = true; break; }
    default: break;                                                                    // bsdfs/NullBsdf.cpp: sample() == false
    }
    return ok;
}

// Bsdf::eval(event, adjoint=false) (bsdfs/Bsdf.hpp:85-97)
TGB_D V3 bsdf_eval_base(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    V3 f = v3s(0.0f);
    switch (b.type) {
    case TGB_BSDF_LAMBERT:                                                             // LambertBsdf.cpp:40-47
        if (!(e.requested & LOBE_DIFFUSE_R)) break;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) break;
        f = (bsdf_albedo(sc, b, s)*INV_PI_F)*e.wo.z;
        break;
    case TGB_BSDF_ROUGH_CONDUCTOR: {                                                   // RoughConductorBsdf.cpp:92-110
        if (!(e.requested & LOBE_GLOSSY_R)) break;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) break;
        float alpha = mf_roughness_to_alpha(b.dist, bsdf_roughness(sc, b, s));
        V3 hr = normalize(e.wi + e.wo);
        float cosThetaM = dot(e.wi, hr);
        V3 F = conductor_reflectance(b.eta, b.k, cosThetaM);
        float G = mf_G(b.dist, alpha, e.wi, e.wo, hr);
        float D = mf_D(b.dist, alpha, hr);
        float fr = (G*D*0.25f)/e.wi.z;
        f = bsdf_albedo(sc, b, s)*(F*fr);
        break; }
    case TGB_BSDF_ROUGH_DIELECTRIC: {                                                  // RoughDielectricBsdf.cpp:246-252
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0;
        bool sampleT = (e.requested & LOBE_GLOSSY_T) != 0 && b.enable_t;
        f = rd_eval_base(e, sampleR, sampleT, bsdf_roughness(sc, b, s), b.ior, b.dist)*bsdf_albedo(sc, b, s);
        break; }
    case TGB_BSDF_MIRROR:                                                              // MirrorBsdf.cpp:39-46
        if ((e.requested & LOBE_SPEC_R) && check_reflection_constraint(e.wi, e.wo)) f = bsdf_albedo(sc, b, s);
        break;
    case TGB_BSDF_CONDUCTOR:                                                           // ConductorBsdf.cpp:70-77
        if ((e.requested & LOBE_SPEC_R) && check_reflection_constraint(e.wi, e.wo))
            f = bsdf_albedo(sc, b, s)*conductor_reflectance(b.eta, b.k, e.wi.z);
        break;
    case TGB_BSDF_DIELECTRIC: {                                                        // DielectricBsdf.cpp:89-109
        bool evalR = (e.requested & LOBE_SPEC_R) != 0;
        bool evalT = (e.requested & LOBE_SPEC_T) != 0 && b.enable_t;
        float eta = e.wi.z < 0.0f ? b.ior : b.inv_ior;
        float cosThetaT = 0.0f;
        float F = dielectric_reflectance(eta, fabsf(e.wi.z), cosThetaT);
        if (e.wi.z*e.wo.z >= 0.0f) { if (evalR && check_reflection_constraint(e.wi, e.wo)) f = bsdf_albedo(sc, b, s)*F; }
        else if (evalT && check_refraction_constraint(e.wi, e.wo, eta, cosThetaT)) f = bsdf_albedo(sc, b, s)*(1.0f - F);
        break; }
    case TGB_BSDF_PLASTIC: {                                                           // PlasticBsdf.cpp:125-151
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) break;
        bool evalR = (e.requested & LOBE_SPEC_R) != 0, evalT = (e.requested & LOBE_DIFFUSE_R) != 0;
        float eta = 1.0f/b.ior;
        float Fi = dielectric_reflectance(eta, e.wi.z);
        float Fo = dielectric_reflectance(eta, e.wo.z);
        if (evalR && check_reflection_constraint(e.wi, e.wo)) f = v3s(Fi);
        else if (evalT) {
            V3 diffuseAlbedo = bsdf_albedo(sc, b, s);
            V3 denom = v3s(1.0f) - diffuseAlbedo*b.diffuse_fresnel;
            V3 brdf = (diffuseAlbedo/denom)*((1.0f - Fi)*(1.0f - Fo)*eta*eta*e.wo.z*INV_PI_F);
            if (max_comp(b.scaled_sigma_a) > 0.0f)
                brdf = brdf*vexp(b.scaled_sigma_a*(-1.0f/e.wo.z - 1.0f/e.wi.z));
            f = brdf;
        }
        break; }
    case TGB_BSDF_ROUGH_PLASTIC: {                                                     // RoughPlasticBsdf.cpp:115-140
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & LOBE_DIFFUSE_R) != 0;
        if (!sampleR && !sampleT) break;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) break;
        V3 glossyR = v3s(0.0f);
        if (sampleR) glossyR = rd_eval_base(e, true, false, bsdf_roughness(sc, b, s), b.ior, b.dist);
        V3 diffuseR = v3s(0.0f);
        if (sampleT) {
            float eta = 1.0f/b.ior;
            float Fi = dielectric_reflectance(eta, e.wi.z);
            float Fo = dielectric_reflectance(eta, e.wo.z);
            V3 diffuseAlbedo = bsdf_albedo(sc, b, s);
            V3 denom = v3s(1.0f) - diffuseAlbedo*b.diffuse_fresnel;
            diffuseR = (diffuseAlbedo/denom)*((1.0f - Fi)*(1.0f - Fo)*eta*eta*e.wo.z*INV_PI_F);
            if (max_comp(b.scaled_sigma_a) > 0.0f)
                diffuseR = diffuseR*vexp(b.scaled_sigma_a*(-1.0f/e.wo.z - 1.0f/e.wi.z));
        }
        f = glossyR + diffuseR;
        break; }
    default: break;
    }
    return f;
}

TGB_D float bsdf_pdf_base(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    switch (b.type) {
    case TGB_BSDF_LAMBERT:                                                             // LambertBsdf.cpp:61-68
        if (!(e.requested & LOBE_DIFFUSE_R)) return 0.0f;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
        return cosine_hemisphere_pdf(e.wo);
    case TGB_BSDF_ROUGH_CONDUCTOR: {                                                   // RoughConductorBsdf.cpp:128-143
        if (!(e.requested & LOBE_GLOSSY_R)) return 0.0f;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
        float sampleAlpha = mf_roughness_to_alpha(b.dist, bsdf_roughness(sc, b, s));
        V3 hr = normalize(e.wi + e.wo);
        return mf_pdf(b.dist, sampleAlpha, hr)*0.25f/dot(e.wi, hr); }
    case TGB_BSDF_ROUGH_DIELECTRIC: {                                                  // RoughDielectricBsdf.cpp:266-272
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0;
        bool sampleT = (e.requested & LOBE_GLOSSY_T) != 0 && b.enable_t;
        return rd_pdf_base(e, sampleR, sampleT, bsdf_roughness(sc, b, s), b.ior, b.dist); }
    case TGB_BSDF_MIRROR:                                                              // MirrorBsdf.cpp:57-64
    case TGB_BSDF_CONDUCTOR:                                                           // ConductorBsdf.cpp:84-91
        return ((e.requested & LOBE_SPEC_R) && check_reflection_constraint(e.wi, e.wo)) ? 1.0f : 0.0f;
    case TGB_BSDF_DIELECTRIC: {                                                        // DielectricBsdf.cpp:144-164
        bool sampleR = (e.requested & LOBE_SPEC_R) != 0;
        bool sampleT = (e.requested & LOBE_SPEC_T) != 0 && b.enable_t;
        float eta = e.wi.z < 0.0f ? b.ior : b.inv_ior;
        float cosThetaT = 0.0f;
        float F = dielectric_reflectance(eta, fabsf(e.wi.z), cosThetaT);
        if (e.wi.z*e.wo.z >= 0.0f) return (sampleR && check_reflection_constraint(e.wi, e.wo)) ? (sampleT ? F : 1.0f) : 0.0f;
        return (sampleT && check_refraction_constraint(e.wi, e.wo, eta, cosThetaT)) ? (sampleR ? 1.0f - F : 1.0f) : 0.0f; }
    case TGB_BSDF_PLASTIC: {                                                           // PlasticBsdf.cpp:153-177
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
        bool sampleR = (e.requested & LOBE_SPEC_R) != 0, sampleT = (e.requested & LOBE_DIFFUSE_R) != 0;
        if (sampleR && sampleT) {
            float Fi = dielectric_reflectance(1.0f/b.ior, e.wi.z);
            float substrateWeight = b.avg_transmittance*(1.0f - Fi);
            float specularWeight = Fi;
            float specularProbability = specularWeight/(specularWeight + substrateWeight);
            if (check_reflection_constraint(e.wi, e.wo)) return specularProbability;
            return cosine_hemisphere_pdf(e.wo)*(1.0f - specularProbability);
        } else if (sampleT) return cosine_hemisphere_pdf(e.wo);
        else if (sampleR) return check_reflection_constraint(e.wi, e.wo) ? 1.0f : 0.0f;
        return 0.0f; }
    case TGB_BSDF_ROUGH_PLASTIC: {                                                     // RoughPlasticBsdf.cpp:186-213
        bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & LOBE_DIFFUSE_R) != 0;
        if (!sampleR && !sampleT) return 0.0f;
        if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
        float glossyPdf = 0.0f;
        if (sampleR) glossyPdf = rd_pdf_base(e, true, false, bsdf_roughness(sc, b, s), b.ior, b.dist);
        float diffusePdf = 0.0f;
        if (sampleT) diffusePdf = cosine_hemisphere_pdf(e.wo);
        if (sampleT && sampleR) {
            float Fi = dielectric_reflectance(1.0f/b.ior, e.wi.z);
            float substrateWeight = b.substrate_weight*b.avg_transmittance*(1.0f - Fi);
            float specularWeight = Fi;
            float specularProbability = specularWeight/(specularWeight + substrateWeight);
            diffusePdf *= (1.0f - specularProbability);
            glossyPdf *= specularProbability;
        }
        return glossyPdf + diffusePdf; }
    default: return 0.0f;
    }
}

// SmoothCoatBsdf (bsdfs/SmoothCoatBsdf.cpp:41-100,146-179,181-216): a Dirac dielectric coat over a substrate lobe
// (one level of nesting: the substrate is never a coat) + the public Bsdf::sample/eval wrappers (bsdfs/Bsdf.hpp:71-97).
TGB_D void coat_warp(const DBsdf &b, const Event &e, Event &q, float &Fi, float &Fo, float &cosThetaTi, float &cosThetaTo) {
    float eta = 1.0f/b.ior;
    Fi = dielectric_reflectance(eta, e.wi.z, cosThetaTi);
    Fo = dielectric_reflectance(eta, e.wo.z, cosThetaTo);
    q = e;
    q.wi = v3(e.wi.x*eta, e.wi.y*eta, copysignf(cosThetaTi, e.wi.z));
    q.wo = v3(e.wo.x*eta, e.wo.y*eta, copysignf(cosThetaTo, e.wo.z));
}
// HairBcsdf (bsdfs/HairBcsdf.cpp:24-160,183-315): longitudinal lobes M_p in closed form, azimuthal lobes N_p from the three
// 64x64 tables the host precomputes (PrecomputedAzimuthalLobe + InterpolatedDistribution1D); the tables stay in L2.
// Local frame: y along the fibre, z the shading normal.
constexpr int kHairRes = 64;
TGB_D float trig_inverse(float x) { return minf(sqrtf(maxf(1.0f - x*x, 0.0f)), 1.0f); }                  // MathUtil.hpp:100-103
TGB_D float clampf(float v, float lo, float hi) { return minf(maxf(v, lo), hi); }
TGB_D int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
TGB_D float hair_I0(float x) {
    float result = 1.0f, xSq = x*x, xi = xSq, denom = 4.0f;
    for (int i = 1; i <= 10; ++i) { result += xi/denom; xi *= xSq; denom *= 4.0f*float((i + 1)*(i + 1)); }
    return result;
}
TGB_D float hair_logI0(float x) {
    if (x > 12.0f) return x + 0.5f*(logf(1.0f/(TWO_PI_F*x)) + 1.0f/(8.0f*x));
    return logf(hair_I0(x));
}
TGB_D float hair_M(float v, float sinThetaI, float sinThetaO, float cosThetaI, float cosThetaO) {
    float a = cosThetaI*cosThetaO/v;
    float b = sinThetaI*sinThetaO/v;
    if (v < 0.1f) return expf(-b + hair_logI0(a) - 1.0f/v + 0.6931f + logf(1.0f/(2.0f*v)));
    return expf(-b)*hair_I0(a)/(2.0f*v*sinhf(1.0f/v));
}
TGB_D float hair_sampleM(float v, float sinThetaI, float cosThetaI, float xi1, float xi2) {
    float cosTheta = 1.0f + v*logf(xi1 + (1.0f - xi1)*expf(-2.0f/v));
    float sinTheta = trig_inverse(cosTheta);
    float cosPhi = cosf(TWO_PI_F*xi2);
    return -cosTheta*sinThetaI + sinTheta*cosPhi*cosThetaI;
}
struct HairLobe { const float *table, *pdfs, *cdfs, *sums; };
TGB_D HairLobe hair_lobe(const DBsdf &b, int p) { HairLobe l; l.table = b.hair_table[p]; l.pdfs = b.hair_pdfs[p]; l.cdfs = b.hair_cdfs[p]; l.sums = b.hair_sums[p]; return l; }
TGB_D void lobe_dist(float distribution, int &d0, int &d1, float &v) {          // InterpolatedDistribution1D.hpp:74-78
    d0 = clampi(int(distribution), 0, kHairRes - 1);
    d1 = d0 + 1 < kHairRes - 1 ? d0 + 1 : kHairRes - 1;
    v = clampf(distribution - float(d0), 0.0f, 1.0f);
}
TGB_D float lobe_dist_pdf(const HairLobe &l, float distribution, int x) {
    int d0, d1; float v; lobe_dist(distribution, d0, d1, v);
    return __ldg(l.pdfs + x + d0*kHairRes)*(1.0f - v) + __ldg(l.pdfs + x + d1*kHairRes)*v;
}
TGB_D float lobe_weight(const HairLobe &l, float cosThetaD) {                   // PrecomputedAzimuthalLobe.hpp:64-68
    float dist = float(kHairRes - 1)*cosThetaD;
    int d0, d1; float v; lobe_dist(dist, d0, d1, v);
    return (__ldg(l.sums + d0)*(1.0f - v) + __ldg(l.sums + d1)*v)*(TWO_PI_F/float(kHairRes));
}
TGB_D void lobe_sample(const HairLobe &l, float cosThetaD, float xi, float &phi, float &pdf) {   // :29-38 + warp (:74-99)
    float dist = float(kHairRes - 1)*cosThetaD;
    int d0, d1; float v; lobe_dist(dist, d0, d1, v);
    int lower = 0, upper = kHairRes; float lowerU = 0.0f, upperU = 1.0f;
    while (upper - lower != 1) {
        int midpoint = (upper + lower)/2;
        float midpointU = __ldg(l.cdfs + midpoint + d0*(kHairRes + 1))*(1.0f - v) + __ldg(l.cdfs + midpoint + d1*(kHairRes + 1))*v;
        if (midpointU < xi) { lower = midpoint; lowerU = midpointU; } else { upper = midpoint; upperU = midpointU; }
    }
    xi = clampf((xi - lowerU)/(upperU - lowerU), 0.0f, 1.0f);
    phi = TWO_PI_F*(float(lower) + xi)*(1.0f/float(kHairRes));
    pdf = lobe_dist_pdf(l, dist, lower)*(float(kHairRes)*INV_TWO_PI_F);
}
TGB_D V3 lobe_eval(const HairLobe &l, float phi, float cosThetaD) {              // :40-54
    float u = float(kHairRes - 1)*phi*INV_TWO_PI_F;
    float v = float(kHairRes - 1)*cosThetaD;
    int x0 = clampi(int(u), 0, kHairRes - 2), y0 = clampi(int(v), 0, kHairRes - 2);
    int x1 = x0 + 1, y1 = y0 + 1;
    u = clampf(u - float(x0), 0.0f, 1.0f); v = clampf(v - float(y0), 0.0f, 1.0f);
    auto T = [&](int x, int y) { const float *t = l.table + 3*(x + y*kHairRes); return v3(__ldg(t), __ldg(t + 1), __ldg(t + 2)); };
    return (T(x0, y0)*(1.0f - u) + T(x1, y0)*u)*(1.0f - v) + (T(x0, y1)*(1.0f - u) + T(x1, y1)*u)*v;
}
TGB_D float lobe_pdf(const HairLobe &l, float phi, float cosThetaD) {            // :56-61
    float u = float(kHairRes - 1)*phi*INV_TWO_PI_F;
    float v = float(kHairRes - 1)*cosThetaD;
    return lobe_dist_pdf(l, v, int(u))*(float(kHairRes)*INV_TWO_PI_F);
}
struct HairAngles { float sinThetaO, cosThetaO, cosThetaI, cosThetaD, phi, thetaIR, thetaITT, thetaITRT; };
TGB_D HairAngles hair_angles(const DBsdf &b, const Event &e) {
    HairAngles a;
    float sinThetaI = e.wi.y; a.sinThetaO = e.wo.y;
    a.cosThetaI = trig_inverse(sinThetaI); a.cosThetaO = trig_inverse(a.sinThetaO);
    float thetaI = asinf(clampf(sinThetaI, -1.0f, 1.0f)), thetaO = asinf(clampf(a.sinThetaO, -1.0f, 1.0f));
    float thetaD = (thetaO - thetaI)*0.5f;
    a.cosThetaD = cosf(thetaD);
    a.phi = atan2f(e.wo.x, e.wo.z);
    if (a.phi < 0.0f) a.phi += TWO_PI_F;
    a.thetaIR = thetaI - 2.0f*b.hair_scale_rad; a.thetaITT = thetaI + b.hair_scale_rad; a.thetaITRT = thetaI + 4.0f*b.hair_scale_rad;
    return a;
}
TGB_D V3 hair_eval(const DBsdf &b, const Event &e) {                             // HairBcsdf.cpp:183-216
    if (!(e.requested & (LOBE_GLOSSY_R | LOBE_GLOSSY_T))) return v3s(0.0f);
    HairAngles a = hair_angles(b, e);
    float MR   = hair_M(b.hair_v[0], sinf(a.thetaIR),   a.sinThetaO, cosf(a.thetaIR),   a.cosThetaO);
    float MTT  = hair_M(b.hair_v[1], sinf(a.thetaITT),  a.sinThetaO, cosf(a.thetaITT),  a.cosThetaO);
    float MTRT = hair_M(b.hair_v[2], sinf(a.thetaITRT), a.sinThetaO, cosf(a.thetaITRT), a.cosThetaO);
    return lobe_eval(hair_lobe(b, 0), a.phi, a.cosThetaD)*MR + lobe_eval(hair_lobe(b, 1), a.phi, a.cosThetaD)*MTT
         + lobe_eval(hair_lobe(b, 2), a.phi, a.cosThetaD)*MTRT;
}
TGB_D float hair_pdf(const DBsdf &b, const Event &e) {                           // :280-315
    if (!(e.requested & (LOBE_GLOSSY_R | LOBE_GLOSSY_T))) return 0.0f;
    HairAngles a = hair_angles(b, e);
    float weightR = lobe_weight(hair_lobe(b, 0), a.cosThetaI), weightTT = lobe_weight(hair_lobe(b, 1), a.cosThetaI),
          weightTRT = lobe_weight(hair_lobe(b, 2), a.cosThetaI);
    float weightSum = weightR + weightTT + weightTRT;
    float pdfR   = weightR  *hair_M(b.hair_v[0], sinf(a.thetaIR),   a.sinThetaO, cosf(a.thetaIR),   a.cosThetaO);
    float pdfTT  = weightTT *hair_M(b.hair_v[1], sinf(a.thetaITT),  a.sinThetaO, cosf(a.thetaITT),  a.cosThetaO);
    float pdfTRT = weightTRT*hair_M(b.hair_v[2], sinf(a.thetaITRT), a.sinThetaO, cosf(a.thetaITRT), a.cosThetaO);
    return (1.0f/weightSum)*(pdfR*lobe_pdf(hair_lobe(b, 0), a.phi, a.cosThetaD) + pdfTT*lobe_pdf(hair_lobe(b, 1), a.phi, a.cosThetaD)
                             + pdfTRT*lobe_pdf(hair_lobe(b, 2), a.phi, a.cosThetaD));
}
TGB_D bool hair_sample(const DBsdf &b, Sampler &smp, Event &e) {                 // :218-278 (4 Sobol dimensions)
    if (!(e.requested & (LOBE_GLOSSY_R | LOBE_GLOSSY_T))) return false;
    float xiNx = sampler_next1d(smp), xiNy = sampler_next1d(smp);
    float xiMx = sampler_next1d(smp), xiMy = sampler_next1d(smp);
    float sinThetaI = e.wi.y;
    float cosThetaI = trig_inverse(sinThetaI);
    float thetaI = asinf(clampf(sinThetaI, -1.0f, 1.0f));
    float thetaIR = thetaI - 2.0f*b.hair_scale_rad, thetaITT = thetaI + b.hair_scale_rad, thetaITRT = thetaI + 4.0f*b.hair_scale_rad;
    float weightR = lobe_weight(hair_lobe(b, 0), cosThetaI), weightTT = lobe_weight(hair_lobe(b, 1), cosThetaI),
          weightTRT = lobe_weight(hair_lobe(b, 2), cosThetaI);
    int p; float theta;
    float target = xiNx*(weightR + weightTT + weightTRT);
    if (target < weightR) { p = 0; theta = thetaIR; }
    else if (target < weightR + weightTT) { p = 1; theta = thetaITT; }
    else { p = 2; theta = thetaITRT; }
    float sinThetaO = hair_sampleM(b.hair_v[p], sinf(theta), cosf(theta), xiMx, xiMy);
    float cosThetaO = trig_inverse(sinThetaO);
    float thetaO = asinf(clampf(sinThetaO, -1.0f, 1.0f));
    float thetaD = (thetaO - thetaI)*0.5f;
    float cosThetaD = cosf(thetaD);
    float phi, phiPdf;
    lobe_sample(hair_lobe(b, p), cosThetaD, xiNy, phi, phiPdf);
    float sinPhi = sinf(phi), cosPhi = cosf(phi);
    e.wo = v3(sinPhi*cosThetaO, sinThetaO, cosPhi*cosThetaO);
    e.pdf = hair_pdf(b, e);
    e.weight = hair_eval(b, e)/e.pdf;
    e.sampled = LOBE_GLOSSY_R | LOBE_GLOSSY_T;
    return true;
}

// RoughCoatBsdf (bsdfs/RoughCoatBsdf.cpp): a rough dielectric interface (RoughDielectricBsdf::*Base, reflection only) over any
// non-coat substrate.  substrateEvalAndPdf :50-80, sample :82-151, eval :153-195, pdf :257-299.
TGB_D void rcoat_substrate_eval_pdf(const DScene &sc, const DBsdf &b, const DBsdf &sub, const Surface &s, const Event &e, float eta,
                                    float Fi, float cosThetaTi, float &pdf, V3 &brdf) {
    float cosThetaTo;
    float Fo = dielectric_reflectance(eta, e.wo.z, cosThetaTo);
    if (Fi == 1.0f || Fo == 1.0f) { pdf = 0.0f; brdf = v3s(0.0f); return; }
    Event q = e;
    q.wi = v3(e.wi.x*eta, e.wi.y*eta, copysignf(cosThetaTi, e.wi.z));
    q.wo = v3(e.wo.x*eta, e.wo.y*eta, copysignf(cosThetaTo, e.wo.z));
    pdf = bsdf_pdf_base(sc, sub, s, q);
    pdf *= eta*eta*fabsf(e.wo.z/cosThetaTo);
    float compressionProjection = eta*eta*e.wo.z/cosThetaTo;
    V3 substrateF = bsdf_eval_base(sc, sub, s, q);
    if (max_comp(b.scaled_sigma_a) > 0.0f)
        substrateF = substrateF*vexp(b.scaled_sigma_a*(-1.0f/cosThetaTo - 1.0f/cosThetaTi));
    brdf = substrateF*(compressionProjection*(1.0f - Fi)*(1.0f - Fo));
}
TGB_D bool rcoat_sample(const DScene &sc, const DBsdf &b, const Surface &s, Sampler &smp, Event &e) {
    const DBsdf &sub = sc.bsdfs[b.substrate];
    if (e.wi.z <= 0.0f) return false;
    bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & sub.lobes) != 0;
    if (!sampleR && !sampleT) return false;
    V3 wi = e.wi;
    float eta = 1.0f/b.ior;
    float cosThetaTi;
    float Fi = dielectric_reflectance(eta, wi.z, cosThetaTi);
    float substrateWeight = b.avg_transmittance*(1.0f - Fi);
    float specularWeight = Fi;
    float specularProbability = specularWeight/(specularWeight + substrateWeight);
    if (sampleR && (sampler_boolean(smp, specularProbability) || !sampleT)) {
        float roughness = bsdf_roughness(sc, b, s);
        if (!rd_sample_base(smp, e, true, false, roughness, b.ior, b.dist)) return false;
        if (sampleT) {
            V3 brdfSubstrate, brdfSpecular = e.weight*e.pdf;
            float pdfSubstrate, pdfSpecular = e.pdf*specularProbability;
            rcoat_substrate_eval_pdf(sc, b, sub, s, e, eta, Fi, cosThetaTi, pdfSubstrate, brdfSubstrate);
            pdfSubstrate *= 1.0f - specularProbability;
            e.weight = (brdfSpecular + brdfSubstrate)/(pdfSpecular + pdfSubstrate);
            e.pdf = pdfSpecular + pdfSubstrate;
        }
        return true;
    }
    V3 wiSubstrate = v3(wi.x*eta, wi.y*eta, cosThetaTi);
    e.wi = wiSubstrate;
    bool success = bsdf_sample_base(sc, sub, s, smp, e);
    e.wi = wi;
    if (!success) return false;
    float cosThetaTo;
    float Fo = dielectric_reflectance(b.ior, e.wo.z, cosThetaTo);
    if (Fo == 1.0f) return false;
    float cosThetaSubstrate = e.wo.z;
    e.wo = v3(e.wo.x*b.ior, e.wo.y*b.ior, cosThetaTo);
    e.weight = e.weight*((1.0f - Fi)*(1.0f - Fo));
    if (max_comp(b.scaled_sigma_a) > 0.0f)
        e.weight = e.weight*vexp(b.scaled_sigma_a*(-1.0f/cosThetaSubstrate - 1.0f/cosThetaTi));
    e.weight = e.weight*(wi.z/wiSubstrate.z);
    e.pdf *= eta*eta*cosThetaTo/cosThetaSubstrate;
    if (sampleR) {
        float roughness = bsdf_roughness(sc, b, s);
        V3 brdfSubstrate = e.weight*e.pdf;
        float pdfSubstrate = e.pdf*(1.0f - specularProbability);
        V3 brdfSpecular = rd_eval_base(e, true, false, roughness, b.ior, b.dist);
        float pdfSpecular = rd_pdf_base(e, true, false, roughness, b.ior, b.dist);
        pdfSpecular *= specularProbability;
        e.weight = (brdfSpecular + brdfSubstrate)/(pdfSpecular + pdfSubstrate);
        e.pdf = pdfSpecular + pdfSubstrate;
    }
    return true;
}
TGB_D V3 rcoat_eval(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    const DBsdf &sub = sc.bsdfs[b.substrate];
    bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & sub.lobes) != 0;
    if (!sampleT && !sampleR) return v3s(0.0f);
    if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return v3s(0.0f);
    V3 glossyR = v3s(0.0f);
    if (sampleR) glossyR = rd_eval_base(e, true, false, bsdf_roughness(sc, b, s), b.ior, b.dist);
    V3 substrateR = v3s(0.0f);
    if (sampleT) {
        float eta = 1.0f/b.ior, cosThetaTi, cosThetaTo;
        float Fi = dielectric_reflectance(eta, e.wi.z, cosThetaTi);
        float Fo = dielectric_reflectance(eta, e.wo.z, cosThetaTo);
        if (Fi == 1.0f || Fo == 1.0f) return glossyR;
        Event q = e;
        q.wi = v3(e.wi.x*eta, e.wi.y*eta, copysignf(cosThetaTi, e.wi.z));
        q.wo = v3(e.wo.x*eta, e.wo.y*eta, copysignf(cosThetaTo, e.wo.z));
        float compressionProjection = eta*eta*e.wo.z/cosThetaTo;
        V3 substrateF = bsdf_eval_base(sc, sub, s, q);
        if (max_comp(b.scaled_sigma_a) > 0.0f)
            substrateF = substrateF*vexp(b.scaled_sigma_a*(-1.0f/cosThetaTo - 1.0f/cosThetaTi));
        substrateR = substrateF*(compressionProjection*(1.0f - Fi)*(1.0f - Fo));
    }
    return glossyR + substrateR;
}
TGB_D float rcoat_pdf(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    const DBsdf &sub = sc.bsdfs[b.substrate];
    bool sampleR = (e.requested & LOBE_GLOSSY_R) != 0, sampleT = (e.requested & sub.lobes) != 0;
    if (!sampleT && !sampleR) return 0.0f;
    if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
    float eta = 1.0f/b.ior, cosThetaTi, cosThetaTo;
    float Fi = dielectric_reflectance(eta, e.wi.z, cosThetaTi);
    float Fo = dielectric_reflectance(eta, e.wo.z, cosThetaTo);
    float specularProbability;
    if (sampleR && sampleT) {
        float substrateWeight = b.avg_transmittance*(1.0f - Fi);
        float specularWeight = Fi;
        specularProbability = specularWeight/(specularWeight + substrateWeight);
    } else specularProbability = sampleR ? 1.0f : 0.0f;
    float glossyPdf = 0.0f;
    if (sampleR) glossyPdf = rd_pdf_base(e, true, false, bsdf_roughness(sc, b, s), b.ior, b.dist);
    float substratePdf = 0.0f;
    if (sampleT && Fi < 1.0f && Fo < 1.0f) {
        Event q = e;
        q.wi = v3(e.wi.x*eta, e.wi.y*eta, copysignf(cosThetaTi, e.wi.z));
        q.wo = v3(e.wo.x*eta, e.wo.y*eta, copysignf(cosThetaTo, e.wo.z));
        substratePdf = bsdf_pdf_base(sc, sub, s, q);
        substratePdf *= eta*eta*fabsf(e.wo.z/cosThetaTo);
    }
    return glossyPdf*specularProbability + substratePdf*(1.0f - specularProbability);
}

// LS = lobe set the kernel is compiled for: 0 = every lobe model on the path; 1 = scenes whose surfaces are all Lambert (or the
// null BSDF of lights): the same Lambert arithmetic without the other models' code (k_shade<.., .., 1>)
template <bool HAIR = false, int LS = 0>
TGB_D bool bsdf_sample(const DScene &sc, const DBsdf &b, const Surface &s, Sampler &smp, Event &e) {
    if (LS == 1) {
        if (b.type != TGB_BSDF_LAMBERT) return false;                          // NullBsdf::sample() == false
        if (!(e.requested & LOBE_DIFFUSE_R)) return false;
        if (e.wi.z <= 0.0f) return false;
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        e.wo = cosine_hemisphere(xa, xb);
        e.pdf = cosine_hemisphere_pdf(e.wo);
        e.weight = bsdf_albedo(sc, b, s);
        e.sampled = LOBE_DIFFUSE_R;
        e.weight = e.weight*sqr(1.0f);                                          // (Bsdf::sample scales by eta^2 = 1)
        return true;
    }
    if (HAIR && b.type == TGB_BSDF_HAIR) return hair_sample(b, smp, e);      // Bsdf::eta() is 1 for the BCSDF
    if (b.type == TGB_BSDF_ROUGH_COAT) return rcoat_sample(sc, b, s, smp, e);
    if (b.type != TGB_BSDF_SMOOTH_COAT) {
        if (!bsdf_sample_base(sc, b, s, smp, e)) return false;
        e.weight = e.weight*sqr(bsdf_eta(b, e));
        return true;
    }
    const DBsdf &sub = sc.bsdfs[b.substrate];
    if (e.wi.z <= 0.0f) return false;
    bool sampleR = (e.requested & LOBE_SPEC_R) != 0, sampleT = (e.requested & sub.lobes) != 0;
    if (!sampleR && !sampleT) return false;
    V3 wi = e.wi;
    float eta = 1.0f/b.ior;
    float cosThetaTi;
    float Fi = dielectric_reflectance(eta, wi.z, cosThetaTi);
    float substrateWeight = b.avg_transmittance*(1.0f - Fi);
    float specularWeight = Fi;
    float specularProbability;
    if (sampleR && sampleT) specularProbability = specularWeight/(specularWeight + substrateWeight);
    else if (sampleR) specularProbability = 1.0f;
    else specularProbability = 0.0f;
    if (sampleR && sampler_boolean(smp, specularProbability)) {
        e.wo = v3(-wi.x, -wi.y, wi.z);
        e.pdf = specularProbability;
        e.weight = v3s(Fi/specularProbability);
        e.sampled = LOBE_SPEC_R;
    } else {
        e.wi = v3(wi.x*eta, wi.y*eta, cosThetaTi);
        bool success = bsdf_sample_base(sc, sub, s, smp, e);
        e.wi = wi;
        if (!success) return false;
        float cosThetaTo;
        float Fo = dielectric_reflectance(b.ior, e.wo.z, cosThetaTo);
        if (Fo == 1.0f) return false;
        float cosThetaSubstrate = e.wo.z;
        e.wo = v3(e.wo.x*b.ior, e.wo.y*b.ior, cosThetaTo);
        e.weight = e.weight*((1.0f - Fi)*(1.0f - Fo));
        if (max_comp(b.scaled_sigma_a) > 0.0f)
            e.weight = e.weight*vexp(b.scaled_sigma_a*(-1.0f/cosThetaSubstrate - 1.0f/cosThetaTi));
        e.weight = e.weight/(1.0f - specularProbability);
        e.pdf *= 1.0f - specularProbability;
        e.pdf *= eta*eta*cosThetaTo/cosThetaSubstrate;
    }
    return true;
}
template <bool HAIR = false, int LS = 0>
TGB_D V3 bsdf_eval(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    if (LS == 1) {
        if (b.type != TGB_BSDF_LAMBERT || !(e.requested & LOBE_DIFFUSE_R) || e.wi.z <= 0.0f || e.wo.z <= 0.0f) return v3s(0.0f)*sqr(1.0f);
        return ((bsdf_albedo(sc, b, s)*INV_PI_F)*e.wo.z)*sqr(1.0f);
    }
    if (HAIR && b.type == TGB_BSDF_HAIR) return hair_eval(b, e);
    if (b.type == TGB_BSDF_ROUGH_COAT) return rcoat_eval(sc, b, s, e);
    if (b.type != TGB_BSDF_SMOOTH_COAT) return bsdf_eval_base(sc, b, s, e)*sqr(bsdf_eta(b, e));
    const DBsdf &sub = sc.bsdfs[b.substrate];
    if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return v3s(0.0f);
    bool evalR = (e.requested & LOBE_SPEC_R) != 0, evalT = (e.requested & sub.lobes) != 0;
    float eta = 1.0f/b.ior, Fi, Fo, cosThetaTi, cosThetaTo; Event q;
    coat_warp(b, e, q, Fi, Fo, cosThetaTi, cosThetaTo);
    if (evalR && check_reflection_constraint(e.wi, e.wo)) return v3s(Fi);
    if (evalT) {
        float laplacian = eta*eta*e.wo.z/cosThetaTo;
        V3 substrateF = bsdf_eval_base(sc, sub, s, q);
        if (max_comp(b.scaled_sigma_a) > 0.0f)
            substrateF = substrateF*vexp(b.scaled_sigma_a*(-1.0f/cosThetaTo - 1.0f/cosThetaTi));
        return substrateF*(laplacian*(1.0f - Fi)*(1.0f - Fo));
    }
    return v3s(0.0f);
}
template <bool HAIR = false, int LS = 0>
TGB_D float bsdf_pdf(const DScene &sc, const DBsdf &b, const Surface &s, const Event &e) {
    if (LS == 1) {
        if (b.type != TGB_BSDF_LAMBERT || !(e.requested & LOBE_DIFFUSE_R) || e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
        return cosine_hemisphere_pdf(e.wo);
    }
    if (HAIR && b.type == TGB_BSDF_HAIR) return hair_pdf(b, e);
    if (b.type == TGB_BSDF_ROUGH_COAT) return rcoat_pdf(sc, b, s, e);
    if (b.type != TGB_BSDF_SMOOTH_COAT) return bsdf_pdf_base(sc, b, s, e);
    const DBsdf &sub = sc.bsdfs[b.substrate];
    if (e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
    bool sampleR = (e.requested & LOBE_SPEC_R) != 0, sampleT = (e.requested & sub.lobes) != 0;
    float eta = 1.0f/b.ior, Fi, Fo, cosThetaTi, cosThetaTo; Event q;
    coat_warp(b, e, q, Fi, Fo, cosThetaTi, cosThetaTo);
    if (sampleR && sampleT) {
        float substrateWeight = b.avg_transmittance*(1.0f - Fi);
        float specularWeight = Fi;
        float specularProbability = specularWeight/(specularWeight + substrateWeight);
        if (check_reflection_constraint(e.wi, e.wo)) return specularProbability;
        return bsdf_pdf_base(sc, sub, s, q)*(1.0f - specularProbability)*eta*eta*fabsf(e.wo.z/cosThetaTo);
    } else if (sampleT) return bsdf_pdf_base(sc, sub, s, q)*eta*eta*fabsf(e.wo.z/cosThetaTo);
    else if (sampleR) return check_reflection_constraint(e.wi, e.wo) ? 1.0f : 0.0f;
    return 0.0f;
}

// LS = 1 in the emitter-set-1 k_shade (every texture constant): a BSDF is one 16-byte record (DScene::lambert) instead of the
// DBsdf -> texture chain of loads.  Same arithmetic as the LS = 1 branches of bsdf_sample / bsdf_eval / bsdf_pdf.
struct LambertRec { uint32_t type, lobes; V3 albedo; };
TGB_D LambertRec lambert_rec(const DScene &sc, int bsdf) {
    const float4 r = __ldg(sc.lambert + bsdf);
    const uint32_t w = __float_as_uint(r.w);
    LambertRec l; l.type = w & 0xFFFFu; l.lobes = w >> 16; l.albedo = v3(r.x, r.y, r.z);
    return l;
}
TGB_D bool lambert_sample(const LambertRec &b, Sampler &smp, Event &e) {
    if (b.type != TGB_BSDF_LAMBERT) return false;                              // NullBsdf::sample() == false
    if (!(e.requested & LOBE_DIFFUSE_R)) return false;
    if (e.wi.z <= 0.0f) return false;
    float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
    e.wo = cosine_hemisphere(xa, xb);
    e.pdf = cosine_hemisphere_pdf(e.wo);
    e.weight = b.albedo;
    e.sampled = LOBE_DIFFUSE_R;
    e.weight = e.weight*sqr(1.0f);
    return true;
}
TGB_D V3 lambert_eval(const LambertRec &b, const Event &e) {
    if (b.type != TGB_BSDF_LAMBERT || !(e.requested & LOBE_DIFFUSE_R) || e.wi.z <= 0.0f || e.wo.z <= 0.0f) return v3s(0.0f)*sqr(1.0f);
    return ((b.albedo*INV_PI_F)*e.wo.z)*sqr(1.0f);
}
TGB_D float lambert_pdf(const LambertRec &b, const Event &e) {
    if (b.type != TGB_BSDF_LAMBERT || !(e.requested & LOBE_DIFFUSE_R) || e.wi.z <= 0.0f || e.wo.z <= 0.0f) return 0.0f;
    return cosine_hemisphere_pdf(e.wo);
}

// ---------------------------------------------------------------- lights
struct LightSample { V3 d; float dist, pdf; };

TGB_D int dist1d_warp(const float *cdf, const float *pdf, int n, float &u) {           // sampling/Distribution1D.hpp:37-41
    // std::upper_bound = the first index whose cdf exceeds u.  The cdf is non-decreasing, so any bracketing order finds the same
    // index; three independent probes per step (4-ary search) halve the chain of dependent loads of the binary search (a
    // 1024 x 512 environment map: 10 + 9 dependent loads per sample -> 5 + 5).
    int lo = 0, hi = n + 1;
    while (hi - lo >= 4) {
        const int q = (hi - lo) >> 2, m1 = lo + q, m2 = m1 + q, m3 = m2 + q;
        const bool p1 = u < __ldg(cdf + m1), p2 = u < __ldg(cdf + m2), p3 = u < __ldg(cdf + m3);
        if (p1) hi = m1; else if (p2) { lo = m1 + 1; hi = m2; } else if (p3) { lo = m2 + 1; hi = m3; } else lo = m3 + 1;
    }
    while (lo < hi) { int mid = (lo + hi) >> 1; if (u < __ldg(cdf + mid)) hi = mid; else lo = mid + 1; }
    int idx = lo - 1;
    float r = (u - __ldg(cdf + idx))/__ldg(pdf + idx);
    u = r < 0.0f ? 0.0f : (r > 1.0f ? 1.0f : r);
    return idx;
}
TGB_D float bitmap_pdf_uv(const DTex &t, float u, float v) {                           // textures/BitmapTexture.cpp pdf(MAP_SPHERICAL)
    int w = t.res_u, h = t.res_v;
    int col = min(max(int(u*w), 0), w - 1);
    int row = min(max(int((1.0f - v)*h), 0), h - 1);
    return __ldg(t.pdf + size_t(row)*w + col)*__ldg(t.marg_pdf + row)*w*h;
}
TGB_D void direction_to_uv(const DPrim &p, V3 wi, float &u, float &v, float *sinTheta) {    // primitives/InfiniteSphere.cpp:27-39
    V3 wl = m3mul(p.inv_rot, wi);
    if (sinTheta) *sinTheta = sqrtf(maxf(1.0f - wl.y*wl.y, 0.0f));
    u = atan2f(wl.z, wl.x)*INV_TWO_PI_F + 0.5f;
    v = acosf(-wl.y)*INV_PI_F;
}

// ES (emitter set the caller is compiled for): 0 = every light type; 1 = every light is a quad (k_shade<.., .., 1, 1>)
template <int ES = 0>
TGB_D bool light_sample_direct(const DScene &sc, const DPrim &l, V3 p, Sampler &smp, LightSample &out) {
    if (ES == 1 || l.type == TGB_PRIM_QUAD) {                                          // primitives/Quad.cpp:172-188
        if (dot(l.normal, p - l.base) <= 0.0f) return false;
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        V3 q = l.base + l.edge0*xa + l.edge1*xb;
        out.d = q - p;
        float rSq = length_sq(out.d);
        out.dist = sqrtf(rSq);
        out.d = out.d/out.dist;
        float cosTheta = -dot(l.normal, out.d);
        out.pdf = rSq/(cosTheta*l.area);
        return true;
    }
    if (l.type == TGB_PRIM_MESH) {                                                     // primitives/TriangleMesh.cpp:413-436,448-465
        float u = sampler_next1d(smp);
        int idx = dist1d_warp(l.tri_cdf, l.tri_pdf, int(l.n_tris), u);
        const float *lv = l.light_verts + 9*size_t(idx);
        V3 p0 = v3(__ldg(lv), __ldg(lv + 1), __ldg(lv + 2)), p1 = v3(__ldg(lv + 3), __ldg(lv + 4), __ldg(lv + 5));
        V3 p2 = v3(__ldg(lv + 6), __ldg(lv + 7), __ldg(lv + 8));
        V3 normal = normalize(cross(p1 - p0, p2 - p0));
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        float uSqrt = sqrtf(xa);                                                       // SampleWarp::uniformTriangleUv
        float alpha = 1.0f - uSqrt, beta = (1.0f - xb)*uSqrt;
        V3 pp = p0*alpha + p1*beta + p2*(1.0f - alpha - beta);
        V3 L = pp - p;
        float rSq = length_sq(L);
        out.dist = sqrtf(rSq);
        out.d = L/out.dist;
        float cosTheta = -dot(normal, out.d);
        if (cosTheta <= 0.0f) return false;
        out.pdf = rSq/(cosTheta*l.total_area);
        return true;
    }
    if (l.type == TGB_PRIM_INFINITE_SPHERE) {                                          // primitives/InfiniteSphere.cpp:161-176
        const DTex &em = sc.tex[l.emission_tex];
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        if (em.type == TGB_TEX_CONSTANT) {
            float phi = xa*TWO_PI_F, z = xb*2.0f - 1.0f;                               // SampleWarp::uniformSphere
            float r = sqrtf(maxf(1.0f - z*z, 0.0f));
            out.d = v3(cosf(phi)*r, sinf(phi)*r, z);
            out.dist = INFINITY; out.pdf = INV_FOUR_PI_F;
            return true;
        }
        // BitmapTexture::sample(MAP_SPHERICAL) via Distribution2D::warp
        float u = xa, v = xb;
        int row = dist1d_warp(em.marg_cdf, em.marg_pdf, em.res_v, v);
        int col = dist1d_warp(em.cdf + size_t(row)*(em.res_u + 1), em.pdf + size_t(row)*em.res_u, em.res_u, u);
        float tu = (u + col)/em.res_u, tv = 1.0f - (v + row)/em.res_v;
        float phi = (tu - 0.5f)*TWO_PI_F, theta = tv*PI_F;                             // uvToDirection (InfiniteSphere.cpp:41-51)
        float sinTheta = sinf(theta);
        out.d = m3mul(l.rot, v3(cosf(phi)*sinTheta, -cosf(theta), sinf(phi)*sinTheta));
        out.pdf = INV_PI_F*INV_TWO_PI_F*bitmap_pdf_uv(em, tu, tv)/sinTheta;
        out.dist = INFINITY;
        return out.pdf != 0.0f;
    }
    if (l.type == TGB_PRIM_INFINITE_SPHERE_CAP) {                                      // primitives/InfiniteSphereCap.cpp:131-139
        float xa = sampler_next1d(smp), xb = sampler_next1d(smp);
        float phi = xa*TWO_PI_F;                                                       // SampleWarp::uniformSphericalCap (SampleWarp.hpp:119-129)
        float z = xb*(1.0f - l.area) + l.area;
        float r = sqrtf(maxf(1.0f - z*z, 0.0f));
        out.d = to_global(frame_from_normal(l.normal), v3(cosf(phi)*r, sinf(phi)*r, z));
        out.dist = INFINITY;
        out.pdf = INV_TWO_PI_F/(1.0f - l.area);                                        // uniformSphericalCapPdf (:131-134)
        return true;
    }
    return false;
}
// InfiniteSphereCap::intersect (InfiniteSphereCap.cpp:69-80): the cap is "hit" by directions inside its cone
TGB_D bool cap_hit(const DPrim &l, V3 d) { return !(dot(d, l.normal) < l.area); }
// TraceableScene::intersectInfinites (renderer/TraceableScene.hpp:194-209): every infinite light is asked in list order and the
// LAST one that is hit owns the ray -> walk the list backwards to the first hit.  Returns the primitive index or -1.
TGB_D int infinite_light_hit(const DScene &sc, V3 d) {
    for (int i = sc.n_inf_lights - 1; i >= 0; --i) {
        int li = sc.inf_lights[i];
        const DPrim &l = sc.prims[li];
        if (l.type != TGB_PRIM_INFINITE_SPHERE_CAP || cap_hit(l, d)) return li;
    }
    return -1;
}

template <int ES = 0>
TGB_D float light_approx_radiance(const DScene &sc, const DPrim &l, V3 p) {
    if (ES == 1 || l.type == TGB_PRIM_QUAD) {                                          // primitives/Quad.cpp:256-278
        if (!(l.flags & PF_EMISSIVE)) return 0.0f;
        V3 R0 = l.base - p;
        if (dot(R0, l.normal) >= 0.0f) return 0.0f;
        V3 R1 = R0 + l.edge0, R2 = R1 + l.edge1, R3 = R0 + l.edge1;
        V3 n0 = normalize(cross(R0, R1)), n1 = normalize(cross(R1, R2));
        V3 n2 = normalize(cross(R2, R3)), n3 = normalize(cross(R3, R0));
        float Q = acosf(dot(n0, n1)) + acosf(dot(n1, n2)) + acosf(dot(n2, n3)) + acosf(dot(n3, n0));
        return (TWO_PI_F - fabsf(Q))*max_comp(sc.tex[l.emission_tex].avg);
    }
    if (l.type == TGB_PRIM_MESH) return -1.0f;                                         // primitives/TriangleMesh.cpp:514-517
    if (l.type == TGB_PRIM_INFINITE_SPHERE) {                                          // primitives/InfiniteSphere.cpp:261-266
        if (l.flags & PF_SKYDOME) return (TWO_PI_F*2.0f)*max_comp(sc.tex[l.emission_tex].avg);   // Skydome.cpp:279-282: FOUR_PI*average().max(), no flag test
        if (!(l.flags & PF_EMISSIVE) || !(l.flags & PF_SAMPLABLE)) return 0.0f;
        return TWO_PI_F*max_comp(sc.tex[l.emission_tex].avg);
    }
    if (l.type == TGB_PRIM_INFINITE_SPHERE_CAP) {                                      // InfiniteSphereCap.cpp:207-212
        if (!(l.flags & PF_EMISSIVE) || !(l.flags & PF_SAMPLABLE)) return 0.0f;
        return TWO_PI_F*(1.0f - l.area)*max_comp(sc.tex[l.emission_tex].avg);
    }
    return 0.0f;
}

// TraceBase::chooseLight (integrators/TraceBase.cpp:416-459).  Returns the primitive index or -1.
// The reference keeps one pdf per light in a vector.  Up to 16 lights they live in registers/local memory here; beyond that
// (any number of lights) the approximate radiances are re-evaluated in three passes -- totals, the running-total replacement of
// the "unknown" (negative) entries, selection -- which performs the same float operations in the same order.
template <int ES = 0>
TGB_D int choose_light(const DScene &sc, V3 p, Sampler &smp, float &weight) {
    const int n = sc.n_lights;
    if (n == 0) return -1;
    if (n == 1) { weight = 1.0f; return sc.lights[0]; }
    if (n <= 16) {
        float pdfs[16];
        float total = 0.0f; unsigned numNonNegative = 0;
        for (int i = 0; i < n; ++i) {
            pdfs[i] = light_approx_radiance<ES>(sc, sc.prims[sc.lights[i]], p);
            if (pdfs[i] >= 0.0f) { total += pdfs[i]; numNonNegative++; }
        }
        if (numNonNegative == 0) { for (int i = 0; i < n; ++i) pdfs[i] = 1.0f; total = float(n); }
        else if (numNonNegative < unsigned(n)) {
            for (int i = 0; i < n; ++i) {
                float uniformWeight = (total == 0.0f ? 1.0f : total)/numNonNegative;
                if (pdfs[i] < 0.0f) { pdfs[i] = uniformWeight; total += uniformWeight; }
            }
        }
        if (total == 0.0f) return -1;
        float t = sampler_next1d(smp)*total;
        for (int i = 0; i < n; ++i) {
            if (t < pdfs[i] || i == n - 1) { weight = total/pdfs[i]; return sc.lights[i]; }
            t -= pdfs[i];
        }
        return -1;
    }
    float known = 0.0f; unsigned numNonNegative = 0;
    for (int i = 0; i < n; ++i) {
        const float r = light_approx_radiance<ES>(sc, sc.prims[sc.lights[i]], p);
        if (r >= 0.0f) { known += r; numNonNegative++; }
    }
    const bool none_known = numNonNegative == 0, some_unknown = numNonNegative < unsigned(n);
    float total = known;
    if (none_known) total = float(n);
    else if (some_unknown) {
        for (int i = 0; i < n; ++i)
            if (light_approx_radiance<ES>(sc, sc.prims[sc.lights[i]], p) < 0.0f) total += (total == 0.0f ? 1.0f : total)/numNonNegative;
    }
    if (total == 0.0f) return -1;
    float t = sampler_next1d(smp)*total;
    float running = known;
    for (int i = 0; i < n; ++i) {
        float pdf = 1.0f;
        if (!none_known) {
            pdf = light_approx_radiance<ES>(sc, sc.prims[sc.lights[i]], p);
            if (pdf < 0.0f) { pdf = (running == 0.0f ? 1.0f : running)/numNonNegative; running += pdf; }
        }
        if (t < pdf || i == n - 1) { weight = total/pdf; return sc.lights[i]; }
        t -= pdf;
    }
    return -1;
}

}  // namespace tgb
