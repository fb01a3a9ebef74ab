// Kernels of the test hooks (tgb200_bsdf_probe, tgb200_bsdf_sample_probe, tgb200_light_probe, tgb200_choose_light_probe,
// tgb200_shadow_probe): one thread per input, each calling the device functions k_shade calls (bsdf_eval / bsdf_pdf / bsdf_sample
// with k_shade's template arguments, light_sample_direct + light_hit_direct / mesh_direct_pdf, choose_light, light_query).
// tgb200_bounce_probe's kernels only set up and read back path state around the renderer's own wavefront kernels.
// Nothing here restates their arithmetic.
#pragma once
#include "tgb_wavefront.cuh"

namespace tgb {

// The surface record the BSDF code reads: only the texture coordinates (albedo / roughness textures) matter
TGB_D Surface probe_surface(int bsdf, float u, float v) {
    Surface s;
    s.Ng = s.Ns = v3(0.0f, 0.0f, 1.0f); s.p = v3s(0.0f); s.w = v3(0.0f, 0.0f, -1.0f); s.u = u; s.v = v;
    s.prim = 0; s.bsdf = bsdf; s.backside = false; s.eps = 5e-4f; s.curve = false; s.tangent = v3s(0.0f);
    return s;
}
TGB_D Event probe_event(V3 wi, V3 wo, uint32_t requested) {
    Event e;
    e.frame = frame_from_normal(v3(0.0f, 0.0f, 1.0f)); e.wi = wi; e.wo = wo; e.weight = v3s(1.0f); e.pdf = 1.0f;
    e.requested = requested; e.sampled = 0; e.flipped = false;
    return e;
}

template <bool HAIR, int LS>
__global__ void __launch_bounds__(128) k_probe_bsdf(DScene sc, int bsdf, float u, float v, uint32_t requested, const float *wi_wo,
                                                    float *out, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *w = wi_wo + 6*size_t(i);
    const Surface s = probe_surface(bsdf, u, v);
    const Event e = probe_event(v3(w[0], w[1], w[2]), v3(w[3], w[4], w[5]), requested);
    const DBsdf &b = sc.bsdfs[bsdf];
    const V3 f = bsdf_eval<HAIR, LS>(sc, b, s, e);
    const float pdf = bsdf_pdf<HAIR, LS>(sc, b, s, e);
    float *o = out + 4*size_t(i);
    o[0] = f.x; o[1] = f.y; o[2] = f.z; o[3] = pdf;
}

template <bool HAIR, int LS>
__global__ void __launch_bounds__(128) k_probe_bsdf_sample(DScene sc, uint32_t seed, const int *bsdf, const uint32_t *pixel_id,
                                                           uint32_t sample, float u, float v, uint32_t requested, const float *wi,
                                                           float *out, uint32_t *lobes, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Surface s = probe_surface(bsdf[i], u, v);
    Event e = probe_event(v3(wi[3*size_t(i)], wi[3*size_t(i) + 1], wi[3*size_t(i) + 2]), v3s(0.0f), requested);
    Sampler smp; sampler_start(smp, sc.sobol, seed, pixel_id[i], sample);
    const bool ok = bsdf_sample<HAIR, LS>(sc, sc.bsdfs[bsdf[i]], s, smp, e);
    float *o = out + 8*size_t(i);
    o[0] = ok ? 1.0f : 0.0f; o[1] = e.wo.x; o[2] = e.wo.y; o[3] = e.wo.z;
    o[4] = e.weight.x; o[5] = e.weight.y; o[6] = e.weight.z; o[7] = e.pdf;
    lobes[i] = ok ? e.sampled : 0u;
}

// sampleDirect + (quad / cap / environment) the light's hit, directPdf and emission.  Mesh lights leave a closest-hit query in
// rays[i] (tmax = 0: none) for k_probe_light_mesh.
constexpr float kProbeEpsilon = 5e-4f;                  // IntersectionInfo::epsilon of a surface hit (TraceableScene.hpp:39)
__global__ void __launch_bounds__(128) k_probe_light(DScene sc, int li, uint32_t seed, uint32_t sample, const float *p, float *out,
                                                     tgb_ray *rays, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    float *o = out + 12*size_t(i);
    for (int k = 0; k < 12; ++k) o[k] = 0.0f;
    const V3 pt = v3(p[3*size_t(i)], p[3*size_t(i) + 1], p[3*size_t(i) + 2]);
    tgb_ray r; r.o[0] = pt.x; r.o[1] = pt.y; r.o[2] = pt.z; r.d[0] = 0.0f; r.d[1] = 0.0f; r.d[2] = 1.0f;
    r.tmin = kProbeEpsilon; r.tmax = 0.0f;
    const DPrim &l = sc.prims[li];
    Sampler smp; sampler_start(smp, sc.sobol, seed, i, sample);
    LightSample ls;
    if (light_sample_direct(sc, l, pt, smp, ls)) {
        o[0] = 1.0f; o[1] = ls.d.x; o[2] = ls.d.y; o[3] = ls.d.z; o[4] = ls.dist; o[5] = ls.pdf;
        if (l.type == TGB_PRIM_MESH) {
            r.d[0] = ls.d.x; r.d[1] = ls.d.y; r.d[2] = ls.d.z; r.tmax = INFINITY;
        } else {
            V3 em; float tfar, direct_pdf;
            if (light_hit_direct(sc, l, pt, ls.d, kProbeEpsilon, -1.0f, em, tfar, direct_pdf)) {
                o[6] = 1.0f; o[7] = tfar; o[8] = direct_pdf; o[9] = em.x; o[10] = em.y; o[11] = em.z;
            }
        }
    }
    rays[i] = r;
}
// Mesh lights: the scene's closest hit along the sampled direction, when it lies on the light (shadow_resolve_closest's test)
__global__ void __launch_bounds__(128) k_probe_light_mesh(DScene sc, int li, const tgb_ray *rays, const Hit *hits, float *out,
                                                          uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Hit h = hits[i];
    if (rays[i].tmax == 0.0f || h.id == HID_MISS) return;
    const V3 pt = v3(rays[i].o[0], rays[i].o[1], rays[i].o[2]), d = v3(rays[i].d[0], rays[i].d[1], rays[i].d[2]);
    Surface ls; make_surface<true>(sc, h, pt, d, ls);
    if (ls.prim != li) return;
    const V3 em = eval_direct(sc, ls);
    float *o = out + 12*size_t(i);
    o[6] = 1.0f; o[7] = h.t; o[8] = mesh_direct_pdf(sc.prims[li], pt, d, ls); o[9] = em.x; o[10] = em.y; o[11] = em.z;
}

// tgb200_shadow_probe, before k_shadow_prep / k_shadow_bvh: query i gets scratch slot i and the records k_shade writes for it
// (light_query with f = 1, pdfL = 1, pdfB = 0 for NEE, weight = 1 and the given BSDF pdf for MIS), and is queued when k_shade
// would queue it.  out = 8 floats per query: light hit, t of the light, vis, finished value.rgb (filled in by k_probe_shadow_read),
// queued (1; 2 once k_probe_shadow_traversed saw it reach the BVH pass), any.  query = 8 floats: p.xyz, d.xyz, epsilon, arg (NEE: expected distance, MIS: BSDF pdf); light_mis = 2 ints.
__global__ void __launch_bounds__(128) k_probe_shadow_setup(DScene sc, Scratch sr, const float *query, const int *light_mis, float *out,
                                                            uint32_t *squeue, Ctl *ctl, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float *q = query + 8*size_t(i);
    const V3 p = v3(q[0], q[1], q[2]), d = v3(q[3], q[4], q[5]);
    const float eps = q[6], arg = q[7];
    const int li = light_mis[2*size_t(i)]; const bool mis = light_mis[2*size_t(i) + 1] != 0;
    const DPrim &l = sc.prims[li];
    float4 nx = make_float4(0.0f, 0.0f, 0.0f, 0.0f), mx = nx; float t = INFINITY; bool any = false;
    const bool queued = light_query(sc, l, p, d, eps, mis, v3s(1.0f), mis ? arg : 1.0f, 0.0f, arg, mis ? mx : nx, t, any);
    sr.P[i] = make_float4(p.x, p.y, p.z, eps);
    if (mis) sr.M0[i] = make_float4(d.x, d.y, d.z, t); else sr.N0[i] = make_float4(d.x, d.y, d.z, t);
    sr.N1[i] = nx; sr.M1[i] = mx;
    sr.D1[i] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(li));
    *reinterpret_cast<uint2 *>(sr.vis + 2*size_t(i)) = make_uint2(0u, 0u);
    if (queued) squeue[atomicAdd(&ctl->shadow_count, 1u)] = (i << 2) | (mis ? 1u : 0u) | (any ? 2u : 0u);
    float *o = out + 8*size_t(i);
    o[0] = 1.0f; o[1] = 0.0f;                            // mesh lights: the hit is the traversal's (vis)
    if (l.type != TGB_PRIM_MESH) {                       // the light's own hit, also when light_query found it emits nothing
        V3 em; float directPdf;
        o[0] = light_hit_direct(sc, l, p, d, eps, mis ? -1.0f : arg, em, o[1], directPdf) ? 1.0f : 0.0f;
    }
    o[6] = queued ? 1.0f : 0.0f; o[7] = any ? 1.0f : 0.0f;
}
// after k_shadow_prep: queued = 2 for the queries it left to k_shadow_bvh (the others it settled itself)
__global__ void __launch_bounds__(256) k_probe_shadow_traversed(const uint32_t *squeue2, const uint32_t *squeue_cl, const Ctl *ctl, float *out) {
    const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
    if (j < ctl->shadow_count2) out[8*size_t(squeue2[j] >> 2) + 6] = 2.0f;
    if (j < ctl->shadow_count_closest) out[8*size_t(squeue_cl[j] >> 2) + 6] = 2.0f;
}
// after k_shadow_bvh: vis and the finished lightF (NEE) / bsdfF (MIS) of each query
__global__ void __launch_bounds__(128) k_probe_shadow_read(Scratch sr, const int *light_mis, float *out, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool mis = light_mis[2*size_t(i) + 1] != 0;
    const float4 x = mis ? sr.M1[i] : sr.N1[i];
    float *o = out + 8*size_t(i);
    o[2] = float(sr.vis[2*size_t(i) + (mis ? 1 : 0)]); o[3] = x.x; o[4] = x.y; o[5] = x.z;
}

// tgb200_bounce_probe, before k_iter_end: state i (TGB_BOUNCE_WORDS words, include/tgb200.h) goes into slot i of pb as k_accum hands
// a survivor over -- the analytic part of its closest hit in T2, path id i in T3.w, its ray-coherence key (kBins: it misses the BVH's
// top-level cut and is not traversed) in keys[i], counted in the cleared histogram -- and becomes pixel i of an adaptive BatchInfo
// (result slot pix_first[i] = i, first sample index pix_base[i] = its sample index).  out = the input with status 0 (finished).
__global__ void __launch_bounds__(256) k_probe_bounce_setup(DScene sc, PathBuf pb, const uint32_t *in, uint32_t *pix_id, uint32_t *pix_seed,
                                                            uint32_t *pix_first, uint32_t *pix_base, uint32_t *keys, uint32_t *hist,
                                                            uint32_t *out, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i == 0) pix_first[n] = n;
    if (i >= n) return;
    const uint32_t *r = in + TGB_BOUNCE_WORDS*size_t(i);
    uint32_t *o = out + TGB_BOUNCE_WORDS*size_t(i);
    for (int k = 0; k < TGB_BOUNCE_WORDS; ++k) o[k] = r[k];
    o[TGB_BR_STATUS] = 0u;
    const V3 org = v3(__uint_as_float(r[TGB_BR_ORIGIN]), __uint_as_float(r[TGB_BR_ORIGIN + 1]), __uint_as_float(r[TGB_BR_ORIGIN + 2]));
    const V3 d = v3(__uint_as_float(r[TGB_BR_DIR]), __uint_as_float(r[TGB_BR_DIR + 1]), __uint_as_float(r[TGB_BR_DIR + 2]));
    const float tmin = __uint_as_float(r[TGB_BR_TMIN]);
    const uint32_t info = (r[TGB_BR_DIMENSION] & 0xFFFFu) | (r[TGB_BR_BOUNCE] << 16) | ((r[TGB_BR_FLAGS] & 1u) ? F_WAS_SPECULAR : 0u) | F_ALIVE;
    const Hit h = analytic_closest(sc, org, d, tmin, INFINITY);
    pb.T0[i] = make_float4(org.x, org.y, org.z, tmin);
    pb.T1[i] = make_float4(d.x, d.y, d.z, __uint_as_float(info));
    pb.T2[i] = pack_hit(h);
    pb.T3[i] = make_float4(__uint_as_float(r[TGB_BR_THROUGHPUT]), __uint_as_float(r[TGB_BR_THROUGHPUT + 1]),
                           __uint_as_float(r[TGB_BR_THROUGHPUT + 2]), __uint_as_float(i));
    pb.E[i] = make_float4(__uint_as_float(r[TGB_BR_EMISSION]), __uint_as_float(r[TGB_BR_EMISSION + 1]),
                          __uint_as_float(r[TGB_BR_EMISSION + 2]), 0.0f);
    pb.pcg[i] = uint64_t(r[TGB_BR_PCG]) | (uint64_t(r[TGB_BR_PCG + 1]) << 32);
    pix_id[i] = r[TGB_BR_PIXEL]; pix_seed[i] = r[TGB_BR_SEED]; pix_first[i] = i; pix_base[i] = r[TGB_BR_SAMPLE];
    const uint32_t key = mesh_cut_hit(sc, org, d, tmin, h.t) ? ray_bin(sc, org, d) : kBins;       // as k_accum keys a survivor
    keys[i] = key;
    if (key != kBins) atomicAdd(hist + key, 1u);
}
// after k_accum: the survivors k_accum compacted into dst, put back in input order through their path id
__global__ void __launch_bounds__(256) k_probe_bounce_alive(PathBuf dst, const Ctl *ctl, uint32_t *out) {
    const uint32_t t = blockIdx.x*blockDim.x + threadIdx.x;
    if (t >= ctl->next_count) return;
    const float4 t0 = dst.T0[t], t1 = dst.T1[t], t3 = dst.T3[t], e = dst.E[t];
    const uint32_t info = __float_as_uint(t1.w);
    uint32_t *o = out + TGB_BOUNCE_WORDS*size_t(__float_as_uint(t3.w));
    o[TGB_BR_ORIGIN] = __float_as_uint(t0.x); o[TGB_BR_ORIGIN + 1] = __float_as_uint(t0.y); o[TGB_BR_ORIGIN + 2] = __float_as_uint(t0.z);
    o[TGB_BR_TMIN] = __float_as_uint(t0.w);
    o[TGB_BR_DIR] = __float_as_uint(t1.x); o[TGB_BR_DIR + 1] = __float_as_uint(t1.y); o[TGB_BR_DIR + 2] = __float_as_uint(t1.z);
    o[TGB_BR_STATUS] = (info & F_ALIVE) ? 1u : 0u;
    o[TGB_BR_THROUGHPUT] = __float_as_uint(t3.x); o[TGB_BR_THROUGHPUT + 1] = __float_as_uint(t3.y); o[TGB_BR_THROUGHPUT + 2] = __float_as_uint(t3.z);
    o[TGB_BR_BOUNCE] = (info >> 16) & 0xFFu;
    o[TGB_BR_EMISSION] = __float_as_uint(e.x); o[TGB_BR_EMISSION + 1] = __float_as_uint(e.y); o[TGB_BR_EMISSION + 2] = __float_as_uint(e.z);
    o[TGB_BR_FLAGS] = (info & F_WAS_SPECULAR) ? 1u : 0u;
    o[TGB_BR_DIMENSION] = info & 0xFFFFu;
    const uint64_t pcg = dst.pcg[t];
    o[TGB_BR_PCG] = uint32_t(pcg); o[TGB_BR_PCG + 1] = uint32_t(pcg >> 32);
}
// ... and the finished ones: the radiance k_accum wrote to R, the sampler state k_shade left in the path's slot
__global__ void __launch_bounds__(256) k_probe_bounce_finished(PathBuf pb, const float4 *R, uint32_t *out, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t *o = out + TGB_BOUNCE_WORDS*size_t(i);
    if (o[TGB_BR_STATUS]) return;
    const float4 c = R[i];
    o[TGB_BR_EMISSION] = __float_as_uint(c.x); o[TGB_BR_EMISSION + 1] = __float_as_uint(c.y); o[TGB_BR_EMISSION + 2] = __float_as_uint(c.z);
    o[TGB_BR_DIMENSION] = __float_as_uint(pb.T1[i].w) & 0xFFFFu;
    const uint64_t pcg = pb.pcg[i];
    o[TGB_BR_PCG] = uint32_t(pcg); o[TGB_BR_PCG + 1] = uint32_t(pcg >> 32);
}

__global__ void __launch_bounds__(128) k_probe_choose_light(DScene sc, uint32_t seed, const uint32_t *pixel_id, uint32_t sample,
                                                            const float *p, float *out, uint32_t n) {
    const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= n) return;
    Sampler smp; sampler_start(smp, sc.sobol, seed, pixel_id[i], sample);
    float weight = 0.0f;
    const int li = choose_light(sc, v3(p[3*size_t(i)], p[3*size_t(i) + 1], p[3*size_t(i) + 2]), smp, weight);
    out[2*size_t(i)] = float(li); out[2*size_t(i) + 1] = li >= 0 ? weight : 0.0f;
}

}  // namespace tgb
