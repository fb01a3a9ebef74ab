/*
 * tgb200.h -- C ABI of the H100-native path_tracer hot path (libtgb200.so).
 *
 * This is the drop-in boundary that sits UNDER Tungsten's C++ `Integrator` interface
 * (reference: src/core/integrators/Integrator.hpp:16-63).  The reference has no C ABI; an in-tree
 * adapter class (`B200PathTraceIntegrator`, see INTEGRATION.md) forwards
 *     prepareForRender(TraceableScene&, seed)  -> tgb200_create()
 *     startRender()/renderTile()               -> tgb200_render_tiles()
 *     abortRender()                            -> tgb200_abort()
 *     teardownAfterRender()                    -> tgb200_destroy()
 * and converts non-zero return codes into std::runtime_error (reference: src/core/Debug.hpp:26-33).
 *
 * Conventions: plain pointers and sizes only; the caller owns every host buffer passed in (they may
 * be freed as soon as the call returns); the context owns all device memory; no call throws;
 * one host thread drives a context at a time (tgb200_abort may be called from any thread).
 * All geometry is WORLD SPACE, i.e. what the reference holds after `prepareForRender()`
 * (TriangleMesh::_tfVerts, Quad::_base/_edge0/_edge1, Cube::_pos/_rot/_scale), fp32.
 */
#ifndef TGB200_H_
#define TGB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TGB200_ABI_VERSION 3

/* ---- return codes -------------------------------------------------------------------------- */
enum {
    TGB_OK               =  0,
    TGB_ERR_INVALID      = -1,   /* bad argument / malformed scene description                   */
    TGB_ERR_UNSUPPORTED  = -2,   /* scene uses a feature outside the hot path (see DESIGN.md)    */
    TGB_ERR_NO_DEVICE    = -3,   /* no CUDA device / wrong architecture: there is NO CPU fallback */
    TGB_ERR_CUDA         = -4,   /* CUDA runtime error, text in tgb200_last_error()               */
    TGB_ERR_ABORTED      = -5,   /* tgb200_abort() was called during the render                   */
    TGB_ERR_OOM          = -6
};

/* ---- textures (reference: src/core/textures/{ConstantTexture,CheckerTexture,BitmapTexture}) - */
enum { TGB_TEX_CONSTANT = 0, TGB_TEX_CHECKER = 1, TGB_TEX_BITMAP = 2 };

typedef struct tgb_texture {
    uint32_t type;
    float    value[3];      /* CONSTANT: value;  CHECKER: "on" colour                              */
    float    value2[3];     /* CHECKER: "off" colour                                               */
    uint32_t res_u, res_v;  /* CHECKER: res_u/res_v;  BITMAP: width/height                         */
    uint32_t flags;         /* BITMAP: bit0 linear filter, bit1 clamp (else repeat)                */
    const float *texels;    /* BITMAP: res_u*res_v RGB fp32, row-major, top row first (host ptr)   */
} tgb_texture;

/* ---- BSDFs (reference: src/core/bsdfs/; the lobes north_star names + Null, the coat of config C0, the Dirac lobes the
 *      shipped scenes use: MirrorBsdf, ConductorBsdf, DielectricBsdf) ------------------------------------------------ */
enum {
    TGB_BSDF_NULL = 0, TGB_BSDF_LAMBERT = 1, TGB_BSDF_ROUGH_CONDUCTOR = 2,
    TGB_BSDF_ROUGH_DIELECTRIC = 3, TGB_BSDF_PLASTIC = 4, TGB_BSDF_ROUGH_PLASTIC = 5,
    TGB_BSDF_SMOOTH_COAT = 6, TGB_BSDF_CONDUCTOR = 7, TGB_BSDF_DIELECTRIC = 8, TGB_BSDF_MIRROR = 9,
    TGB_BSDF_HAIR = 10,         /* bsdfs/HairBcsdf.cpp; only on CURVES primitives                  */
    TGB_BSDF_ROUGH_COAT = 11    /* bsdfs/RoughCoatBsdf.cpp: rough dielectric coat over `substrate`  */
};
enum { TGB_DIST_BECKMANN = 0, TGB_DIST_PHONG = 1, TGB_DIST_GGX = 2 };

typedef struct tgb_bsdf {
    uint32_t type;
    int32_t  albedo_tex;        /* index into textures[]                                           */
    uint32_t distribution;      /* TGB_DIST_* (rough lobes)                                        */
    int32_t  roughness_tex;     /* index into textures[] (rough lobes), -1 if unused               */
    float    ior;               /* dielectric / plastic / coat                                     */
    float    eta[3], k[3];      /* conductor complex IOR (RGB)                                     */
    float    thickness;         /* plastic / coat                                                  */
    float    sigma_a[3];        /* plastic / coat absorption                                       */
    int32_t  substrate;         /* SMOOTH_COAT / ROUGH_COAT: index of the substrate bsdf, else -1   */
    uint32_t enable_refraction; /* (rough) dielectric "enable_refraction"                          */
    /* HAIR: sigma_a[] = HairBcsdf::_sigmaA as prepared (HairBcsdf.cpp:435-443), plus:              */
    float    hair_scale_angle_deg, hair_roughness;
} tgb_bsdf;

/* ---- geometry ------------------------------------------------------------------------------- */
/* 32 B / 16 B: identical to the reference's Vertex / TriangleI and to the .wo3 on-disk layout
 * (src/core/primitives/Vertex.hpp:12-13, Triangle.hpp:14-20, io/MeshIO.cpp:19-25).               */
typedef struct tgb_vertex   { float pos[3]; float normal[3]; float uv[2]; } tgb_vertex;
typedef struct tgb_triangle { uint32_t v0, v1, v2; int32_t material; } tgb_triangle;

enum { TGB_PRIM_MESH = 0, TGB_PRIM_QUAD = 1, TGB_PRIM_CUBE = 2, TGB_PRIM_INFINITE_SPHERE = 3, TGB_PRIM_CURVES = 4,
       TGB_PRIM_INFINITE_SPHERE_CAP = 5,   /* primitives/InfiniteSphereCap.cpp: a disc of directions on the sky ("sun")          */
       TGB_PRIM_SKYDOME = 6 };             /* primitives/Skydome.cpp: an InfiniteSphere whose emission bitmap is the prepared
                                              512x256 sky image (Skydome::prepareForRender; the caller passes its texels), lookup
                                              without rotation, approximateRadiance 4 pi avg (Skydome.cpp:281)                 */
/* Curves::CurveMode (primitives/Curves.cpp:20-25); "ribbon" is outside the hot path                 */
enum { TGB_CURVE_CYLINDER = 0, TGB_CURVE_HALF_CYLINDER = 1, TGB_CURVE_BCSDF_CYLINDER = 2 };

/* One entry per scene primitive, in the reference's Scene::primitives() order.                    */
typedef struct tgb_primitive {
    uint32_t type;
    int32_t  emission_tex;      /* -1 = not emissive (Primitive::_emission)                        */
    /* MESH: world-space vertices/triangles; triangle.material indexes bsdfs[bsdf_first + m]        */
    const tgb_vertex   *verts;  uint32_t n_verts;
    const tgb_triangle *tris;   uint32_t n_tris;
    uint32_t smooth;            /* TriangleMesh::_smoothed                                          */
    uint32_t bsdf_first, bsdf_count;   /* range in bsdf_slots[] (QUAD/CUBE: exactly one)            */
    /* QUAD: Quad::_base/_edge0/_edge1 as prepared (Quad.cpp:298-305)                               */
    float base[3], edge0[3], edge1[3];
    /* CUBE: Cube::_pos, _rot (row-major 3x3), _scale as prepared (Cube.cpp:351-355)                */
    float pos[3], rot[9], scale[3];
    /* INFINITE_SPHERE: rotation (row-major 3x3, InfiniteSphere::_rotTransform), sample flag        */
    uint32_t do_sample;
    /* CURVES: quadratic B-spline nodes (x, y, z, width) in WORLD space as Curves::prepareForRender leaves
     * them (Curves.cpp:572-587); segment k spans nodes curve_segments[k]-2 .. curve_segments[k], in the
     * order prepareForRender emits them (after the `subsample` draw, :589-611); one bsdf slot.       */
    const float    *curve_nodes;    uint32_t n_curve_nodes;
    const uint32_t *curve_segments; uint32_t n_curve_segments;
    uint32_t curve_mode;        /* TGB_CURVE_*                                                      */
    /* INFINITE_SPHERE_CAP: InfiniteSphereCap::_capDir and _cosCapAngle as prepared (InfiniteSphereCap.cpp:231-247); do_sample;
     * emission_tex is evaluated at uv (0, 0) (:191-199)                                                                   */
    float cap_dir[3]; float cap_cos;
} tgb_primitive;

/* ---- camera (reference: cameras/PinholeCamera.cpp:28-35,70-86; Camera.cpp:44-68) ------------ */
enum { TGB_FILTER_DIRAC = 0, TGB_FILTER_BOX = 1, TGB_FILTER_TENT = 2, TGB_FILTER_GAUSSIAN = 3,
       TGB_FILTER_MITCHELL = 4, TGB_FILTER_CATMULL_ROM = 5, TGB_FILTER_LANCZOS = 6 };

typedef struct tgb_camera {
    float    pos[3];            /* Camera::_pos                                                     */
    float    xform[9];          /* upper 3x3 of Camera::_transform AFTER setRight(-right), row-major */
    float    fov_deg;           /* PinholeCamera::_fovDeg                                           */
    uint32_t res_x, res_y;
    uint32_t filter;            /* TGB_FILTER_*                                                     */
} tgb_camera;

/* ---- integrator + renderer settings (PathTracerSettings.hpp:25-32, TraceSettings.hpp:23-29,
 *      RendererSettings.hpp:49-76) ----------------------------------------------------------- */
typedef struct tgb_settings {
    int32_t  min_bounces, max_bounces;
    uint32_t enable_light_sampling;
    uint32_t enable_two_sided_shading;
    uint32_t enable_consistency_checks;
    uint32_t use_sobol;         /* renderer.stratified_sampler; only 1 is supported                  */
    uint32_t supplemental_mode; /* 0 = per-path reseed (parity contract, DESIGN.md section 3)        */
    int32_t  device;            /* CUDA ordinal, -1 = current                                        */
    uint32_t max_paths_in_flight; /* 0 = library default                                             */
    /* Device list (SURVEY 8b): n_devices >= 2 replicates the scene on devices[0 .. n_devices) of this process.  Every render
     * call then deals its 16x16 tiles to the GPUs in Morton order of the tile grid (tgb200_shard_tiles), the GPUs render their
     * shares concurrently (one host thread each), and the shares are gathered on devices[0] with peer-to-peer copies over
     * NVLink (the single collective of the path; a multi-PROCESS caller uses tgb200_pack_tiles + its own NCCL all-gather
     * instead, as bench.py does).  Framebuffer reads, tgb200_trace_closest and the device pointers refer to devices[0].
     * n_devices 0 or 1: one GPU, `device`.                                                                           */
    uint32_t n_devices;
    int32_t  devices[8];
} tgb_settings;

typedef struct tgb_scene_desc {
    uint32_t abi_version;       /* TGB200_ABI_VERSION                                                */
    tgb_camera    camera;
    tgb_settings  settings;
    const tgb_primitive *primitives;  uint32_t n_primitives;
    const tgb_bsdf      *bsdfs;       uint32_t n_bsdfs;
    const uint32_t      *bsdf_slots;  uint32_t n_bsdf_slots;   /* per-primitive bsdf index lists    */
    const tgb_texture   *textures;    uint32_t n_textures;
} tgb_scene_desc;

/* ImageTile minus the sampler object (reference: integrators/ImageTile.hpp:12-31); sampler_seed is
 * the value the tile's SobolPathSampler was constructed with (PathTraceIntegrator.cpp:27-42).      */
typedef struct tgb_tile { uint32_t x, y, w, h; uint32_t sampler_seed; } tgb_tile;

/* Parity hook: one closest-hit query == one TraceableScene::intersect (TraceableScene.hpp:170-192) */
typedef struct tgb_ray { float o[3]; float d[3]; float tmin, tmax; } tgb_ray;
typedef struct tgb_hit {
    int32_t  primitive;         /* index into primitives[], -1 = miss                               */
    int32_t  prim_id;           /* triangle index within the mesh / segment index within the curves (0 for quad/cube) */
    float    t, u, v;           /* curves: u = position along the segment, v = interpolated width   */
    uint32_t backside;
} tgb_hit;

/* Counters with the definitions of SURVEY.md section 8(d): a "ray" is one closest-hit query
 * (primary + continuation + NEE shadow + MIS), a "hit" is a query that found a surface.            */
typedef struct tgb_stats {
    uint64_t samples;           /* camera paths started                                             */
    uint64_t rays;
    uint64_t hits;
    uint64_t kernel_launches;   /* launches of this library's own kernels                           */
    double   trace_ms;          /* CUDA-event time inside k_trace (path rays), profiling mode only  */
    uint64_t trace_launches;
    double   total_ms;          /* CUDA-event time of the whole device section                      */
    uint64_t path_rays;         /* queries issued by k_trace (primary + continuation)               */
    uint64_t shadow_rays;       /* queries issued by k_shadow (NEE + MIS)                           */
    double   shadow_ms;         /* CUDA-event time inside k_shadow_bvh, profiling mode only         */
    uint64_t shadow_launches;
    uint64_t path_rays_traversed;    /* path rays that reached k_trace (the rest miss the BVH's top-level cut) */
    uint64_t shadow_rays_traversed;  /* queries that reached k_shadow_bvh (not resolved by k_shadow_prep)         */
    /* profiling mode only: CUDA-event time inside the other kernels of the wavefront loop, and its iteration count */
    double   regen_ms, shade_ms, prep_ms, accum_ms, sort_ms;
    uint64_t iterations;
} tgb_stats;

typedef struct tgb_ctx tgb_ctx;

/* Flatten + upload the scene, build the BVH, allocate the wavefront queues.
 * Replaces: TraceableScene ctor body that prepares primitives/lights + PathTraceIntegrator::
 * prepareForRender (renderer/TraceableScene.hpp:57-137; PathTraceIntegrator.cpp:184-201).           */
int tgb200_create(const tgb_scene_desc *scene, tgb_ctx **out);

/* Render samples [spp_begin, spp_begin+spp_count) of every pixel of the given tiles and fold them
 * into rgb_mean (w*h*3 floats, row-major, top row first) with the reference's running mean
 * (OutputBuffer::addSample, cameras/OutputBuffer.hpp:104-132); count (w*h, may be NULL) receives
 * the per-pixel accepted-sample count.  n_tiles == 0 renders the whole image with the reference's
 * own tile dicing and tile seeds derived from `seed` (PathTraceIntegrator.cpp:27-42,187).
 * rgb_mean/count are HOST pointers: input state on entry (may hold earlier samples), updated on exit.
 * Replaces: PathTraceIntegrator::renderTile over all tiles (PathTraceIntegrator.cpp:136-156).       */
int tgb200_render_tiles(tgb_ctx *ctx, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed,
                        uint32_t spp_begin, uint32_t spp_count, float *rgb_mean, uint32_t *count);

/* Same, but the framebuffer stays resident on the device between calls (no host<->device copy);
 * fetch it with tgb200_read_framebuffer.  Used by the multi-GPU path and the device-resident bench. */
int tgb200_render_resident(tgb_ctx *ctx, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed,
                           uint32_t spp_begin, uint32_t spp_count);
int tgb200_clear_framebuffer(tgb_ctx *ctx);
int tgb200_read_framebuffer(tgb_ctx *ctx, float *rgb_mean, uint32_t *count);
/* Device address of the resident fp32 RGB framebuffer (w*h*3) for zero-copy hand-off to NCCL.       */
int tgb200_framebuffer_device_ptr(tgb_ctx *ctx, void **rgb_mean_dev, uint64_t *n_bytes);

int tgb200_write_framebuffer(tgb_ctx *ctx, const float *rgb_mean, const uint32_t *count);   /* resume: OutputBuffer -> device */

/* ---- adaptive sampling (integrators/path_tracer/PathTraceIntegrator.cpp:44-156, SampleRecord.hpp:11-66) ----------------
 * One record per 4x4 pixel block (PathTraceIntegrator::VarianceTileSize), row-major over ceil(w/4) x ceil(h/4): the
 * reference's SampleRecord, field for field (it is also what saveState/loadState stream, SampleRecord.hpp:24-42).        */
typedef struct tgb_sample_record {
    uint32_t sample_count, next_sample_count, sample_index;
    float    adaptive_weight, mean, running_variance;
} tgb_sample_record;
/* Host only, no GPU: PathTraceIntegrator::generateWork -- advance the blocks' sample indices and decide every block's sample
 * count for the step [current_spp, next_spp): uniform, or (adaptive_sampling and current_spp >= 16) the 95th-percentile
 * clamp + dilation + stochastic distribution of the reference, drawing from the integrator's UniformSampler whose 64-bit
 * state is *sampler_state (= the stream that produced the tile seeds).  Returns 1 = render the step, 0 = nothing to do.    */
int tgb200_generate_work(tgb_sample_record *records, uint32_t res_x, uint32_t res_y, uint32_t current_spp, uint32_t next_spp,
                         int adaptive_sampling, uint64_t *sampler_state);
/* Render one step with per-block sample counts / sample indices taken from `records` (host, in/out): the framebuffer stays
 * resident (tgb200_read_framebuffer), the records come back with sample_count / mean / running_variance updated by every
 * sample's luminance in the reference's order.  Replaces renderTile's per-block bookkeeping (PathTraceIntegrator.cpp:136-156). */
int tgb200_render_adaptive(tgb_ctx *ctx, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed, tgb_sample_record *records);

/* Multi-GPU hand-off (DESIGN.md section 7): pack the resident pixels of `tiles` tile-major (3 floats per
 * pixel, tiles in list order, rows top-down inside a tile) into a DEVICE buffer -- the send buffer of the
 * single all-gather on this path -- and the inverse (de-tile a received buffer into the resident
 * framebuffer, setting the per-pixel sample count).  Both return after the work has completed.      */
int tgb200_pack_tiles(tgb_ctx *ctx, const tgb_tile *tiles, uint32_t n_tiles, void *rgb_out_dev);
int tgb200_unpack_tiles(tgb_ctx *ctx, const tgb_tile *tiles, uint32_t n_tiles, const void *rgb_in_dev,
                        uint32_t sample_count);

/* The tile deal of the multi-GPU path: writes into `order` (n_tiles entries) the tile indices in Morton (Z) order of the tile grid;
 * share k of N = order[k], order[k + N], ...  Any N consecutive entries form a compact block of the image, so every share samples
 * the whole frame evenly (row-major `id mod N` degenerates into column stripes whenever a tile row holds a multiple of N tiles).
 * Host only.                                                                                                          */
int tgb200_shard_tiles(const tgb_tile *tiles, uint32_t n_tiles, uint32_t *order);

/* Batch of closest-hit queries through the same traversal kernel the renderer uses.  As in a render, a ray that misses the
 * BVH's top-level cut before its analytic hit skips the traversal; environment TGB_HOOK_CUT=0 traverses every ray.        */
int tgb200_trace_closest(tgb_ctx *ctx, const tgb_ray *rays, tgb_hit *hits, uint32_t n);

int  tgb200_get_stats(tgb_ctx *ctx, tgb_stats *out);
/* Time every kernel of the wavefront loop with CUDA events on the streams of both wavefronts (fills the *_ms fields of
 * tgb_stats with sums over both; their kernels overlap, so the sums do not add up to total_ms).                         */
int  tgb200_set_profiling(tgb_ctx *ctx, int enable);
/* Run the context's work on the caller's CUDA stream (a cudaStream_t; NULL = back to the context's own stream), so that a
 * caller's events and collectives on that stream order with the renders.  A render runs its second wavefront on a stream
 * of the context's own, forked from the caller's stream at its start and joined back into it before the framebuffer is
 * written: work queued on the caller's stream after the call sees the finished render.                               */
int  tgb200_set_stream(tgb_ctx *ctx, void *cuda_stream);
/* Size of what was built: triangles, BVH nodes, BVH depth, bytes of nodes+triangle records, and the
 * wavefront capacity (paths in flight).  Any pointer may be NULL.                                   */
int  tgb200_scene_info(tgb_ctx *ctx, uint32_t *n_tris, uint32_t *n_nodes, uint32_t *bvh_depth,
                       uint64_t *geom_bytes, uint32_t *capacity);
int  tgb200_reset_stats(tgb_ctx *ctx);
/* Host-only self-check of the BVH builder (no GPU): n triangles, 9 floats each (v0 v1 v2).  Returns TGB_OK when every
 * triangle sits in exactly one leaf and inside every box of its root-to-leaf chain.                    */
int  tgb200_bvh_selftest(const float *tri_verts, uint32_t n, uint32_t *n_nodes, uint32_t *depth, uint32_t *max_leaf);
/* Host-only: the hair BCSDF tables tgb200_create precomputes for one material (HairBcsdf.cpp:318-446): tables = 3 lobes
 * (R, TT, TRT) x 64 x 64 x RGB, sums = 3 x 64 row sums of the sampling weights, v = the three longitudinal variances. */
int  tgb200_hair_selftest(float roughness, float scale_angle_deg, const float *sigma_a, float *tables, float *sums, float *v);
/* Host-only check of the quantised device BVH (QNode4, 8-bit child boxes): builds the tree tgb200_create builds for a scene of
 * n triangles (the rays' origins take the camera's part in the box padding), walks it on the host with the kernels' node
 * arithmetic and triangle test on the records tgb200_create uploads for n_rays rays (8 floats each: o, d, tmin, tmax) and
 * compares the closest t with brute force over all triangles, bit for bit.  *mismatches = rays that differ (must be 0).  */
int  tgb200_qbvh_selftest(const float *tri_verts, uint32_t n, const float *rays, uint32_t n_rays,
                          uint32_t *mismatches, uint32_t *n_nodes, uint64_t *node_visits);
/* Host-only count of the any-hit shadow walk (no GPU): builds the tree, top-level cut and records tgb200_create builds for a
 * scene of n triangles seen from camera_pos, then walks n_queries occlusion queries (8 floats each: o, d, tnear, t_light)
 * both as a sorted walk from the root and as the unsorted walk from the top-level cut boxes the segment enters.
 * out = 11 uint32 per query: cut mask, deepest stack of the cut walk, then per walk
 * (root, cut): occluded, node visits, leaf trips, triangle tests, then the deepest stack of the root walk (for a query that
 * meets no triangle, that of k_trace's closest-hit walk of the same ray).  *stack_need = the traversal stack bound tgb200_create checks;
 * TGB_ERR_UNSUPPORTED when it exceeds stack_size (0: the traversal's own stack).                                           */
int  tgb200_shadow_walk_count(const float *tri_verts, uint32_t n, const float *camera_pos, const float *queries, uint32_t n_queries,
                              uint32_t stack_size, uint32_t *stack_need, uint32_t *out);
/* Test hooks: each launches one kernel on the context's stream that calls the device functions the shading kernel calls, on
 * host arrays in and out.  A NULL context returns TGB_ERR_INVALID.
 * tgb200_bsdf_probe: Bsdf::eval(event, adjoint=false) rgb + Bsdf::pdf of bsdf `bsdf` for n (wi, wo) pairs in the local frame
 *   (6 floats each), texture coordinates (u, v), lobe mask `requested`; out = 4 floats per pair.  lobe_set 1 runs the
 *   Lambert-only kernel instantiation (contexts without curves only); the hair BCSDF needs a context with curves.
 * tgb200_bsdf_sample_probe: Bsdf::sample(event, adjoint=false) for local wi (3 floats each) on the path (pixel_id[i], sample)
 *   of sampler seed `seed`; out = success, wo.xyz, weight.xyz, pdf; lobes = sampled lobe mask (0 on failure).
 * tgb200_light_probe: Primitive::sampleDirect of primitive `prim` from n points (3 floats each, path (i, sample)), then the
 *   light's hit along the sampled direction (mesh lights: the scene's closest hit, when it is on the light), directPdf and
 *   evalDirect; out = 12 floats per point: ok, d.xyz, dist, pdf, hit, t, directPdf, emission.rgb.
 * tgb200_choose_light_probe: TraceBase::chooseLight from n points on the paths (pixel_id[i], sample); out = 2 floats per point:
 *   chosen primitive (-1: none), weight. */
int  tgb200_bsdf_probe(tgb_ctx *ctx, int bsdf, float u, float v, uint32_t requested, int lobe_set, uint32_t n, const float *wi_wo,
                       float *out);
int  tgb200_bsdf_sample_probe(tgb_ctx *ctx, uint32_t seed, uint32_t n, const int *bsdf, const uint32_t *pixel_id, uint32_t sample,
                              float u, float v, uint32_t requested, int lobe_set, const float *wi, float *out, uint32_t *lobes);
int  tgb200_light_probe(tgb_ctx *ctx, int prim, uint32_t seed, uint32_t n, uint32_t sample, const float *p, float *out);
int  tgb200_choose_light_probe(tgb_ctx *ctx, uint32_t seed, uint32_t n, const uint32_t *pixel_id, uint32_t sample, const float *p,
                               float *out);
/* tgb200_shadow_probe: TraceBase::attenuatedEmission of n queries through the renderer's own shadow kernels.  Query i = 8 floats
 * (point p.xyz, direction d.xyz, epsilon, arg) + 2 ints light_mis = (light primitive, mis).  A NEE query (mis = 0, arg = the
 * expected distance) is set up as the shading kernel sets up lightSample's with f = 1, pdfL = 1, pdfB = 0; a MIS query (mis = 1,
 * arg = the BSDF pdf) as bsdfSample's with weight = 1.  Then the analytic / cut pass and the BVH pass run as in a render, in
 * chunks of half the context's capacity (the path slots of its first wavefront).  out = 8 floats per query: light hit (mesh lights: 1), t of the light (mesh lights: 0), vis,
 * the finished lightF / bsdfF rgb (emission, or emission x the power heuristic for MIS; counts only when vis = 1), queued
 * (0: no query, 1: settled by the analytic / cut pass, 2: reached the BVH pass), traced as a blocker test.  A failed probe
 * still restores them unless the device itself faulted.  The context's control block and ray counters are left as they were. */
int  tgb200_shadow_probe(tgb_ctx *ctx, uint32_t n, const float *query, const int *light_mis, float *out);
/* tgb200_bounce_probe: one iteration of the wavefront loop -- the path ray's closest hit, the shading kernel the context renders
 * with, the shadow kernels and the fold into the path -- for n path states.  A state is a record of TGB_BOUNCE_WORDS 32-bit
 * words (float unless marked):
 *   [TGB_BR_ORIGIN + 0..2]  ray origin        [TGB_BR_TMIN]        ray tmin
 *   [TGB_BR_DIR + 0..2]     ray direction     [TGB_BR_STATUS]      uint: out 1 = alive, 0 = finished (ignored on input)
 *   [TGB_BR_THROUGHPUT+0..2] throughput       [TGB_BR_BOUNCE]      uint: bounce of the ray
 *   [TGB_BR_EMISSION + 0..2] radiance so far  [TGB_BR_FLAGS]       uint: bit 0 = wasSpecular
 *   [TGB_BR_PIXEL]  uint: pixel id (x + y*width)   [TGB_BR_SEED] uint: sampler seed of the pixel's tile
 *   [TGB_BR_SAMPLE] uint: sample index             [TGB_BR_DIMENSION] uint: the sampler's next Sobol dimension
 *   [TGB_BR_PCG + 0..1] uint: the supplemental PCG state (low word first); the remaining words are zero.
 * An alive input is a path about to trace its ray at `bounce` (< maxBounces; other inputs are refused with TGB_ERR_INVALID).  The
 * states enter the loop as survivors just handed over: they are binned by ray-coherence key and traced in key order, and those
 * that miss the BVH's top-level cut keep their analytic hit, as in a render.  An alive output is the next state, as the survivor
 * hand-off stores it.  A finished output holds the sample's radiance in EMISSION, the sampler's dimension and PCG state after
 * the bounce, and the input's other fields.  Runs in chunks of half the context's capacity on its first wavefront; the
 * context's control block and ray counters are left as they were. */
enum { TGB_BR_ORIGIN = 0, TGB_BR_TMIN = 3, TGB_BR_DIR = 4, TGB_BR_STATUS = 7, TGB_BR_THROUGHPUT = 8, TGB_BR_BOUNCE = 11,
       TGB_BR_EMISSION = 12, TGB_BR_FLAGS = 15, TGB_BR_PIXEL = 16, TGB_BR_SEED = 17, TGB_BR_SAMPLE = 18, TGB_BR_DIMENSION = 19,
       TGB_BR_PCG = 20, TGB_BOUNCE_WORDS = 24 };
int  tgb200_bounce_probe(tgb_ctx *ctx, uint32_t n, const uint32_t *state_in, uint32_t *state_out);
/* tgb200_bin_probe: the survivor sort of the wavefront loop (the ray-coherence counting sort that orders the next traversal) on n
 * given keys.  keys[t] is survivor t's key as the survivor hand-off leaves it, in [0, 32767], or 32768 for a survivor that misses
 * the BVH's top-level cut and is not traversed.  The histogram is counted by the hand-off's own code, then the scan and the
 * scatter run as in a render, with a render's grid for n survivors.  Out: *n_sorted = the survivors the traversal visits,
 * order[0 .. *n_sorted) = their indices t in visiting order (bins ascending, any order within a bin; order holds n entries), and
 * cursors[0 .. 32768) = each bin's end in order.  n must fit the first wavefront (half the context's capacity) and no key may
 * exceed 32768 (TGB_ERR_INVALID).  keys and order may be NULL when n = 0.  The context's control block and ray counters are left
 * as they were. */
int  tgb200_bin_probe(tgb_ctx *ctx, uint32_t n, const uint32_t *keys, uint32_t *order, uint32_t *cursors, uint32_t *n_sorted);
/* tgb200_shade_variant: the shading kernel the context renders (and tgb200_bounce_probe runs) with, as its template arguments,
 * into variant[0..3]: variant[0] = curves, variant[1] = material sort, variant[2] = lobe set (1: the Lambert-only
 * instantiation), variant[3] = emitter set (1: the Lambert-only instantiation for scenes whose lights are all quads, with no
 * infinite emitter and only constant albedo and emission textures). */
int  tgb200_shade_variant(const tgb_ctx *ctx, uint32_t *variant);
/* tgb200_abort cancels the render in progress (it returns TGB_ERR_ABORTED) or, if none is running, the next one -- so an
 * abort that lands between an asynchronous start and the worker reaching the render call is not lost.  A caller that
 * starts renders asynchronously calls tgb200_clear_abort before spawning the worker (the adapter's startRender does).   */
int  tgb200_abort(tgb_ctx *ctx);
int  tgb200_clear_abort(tgb_ctx *ctx);
void tgb200_destroy(tgb_ctx *ctx);
/* Last error text of the context; with ctx == NULL the text of the last failed tgb200_create.       */
const char *tgb200_last_error(const tgb_ctx *ctx);
uint32_t tgb200_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* TGB200_H_ */
