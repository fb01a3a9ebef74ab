/*
 * pt_oracle.h -- CPU restatement of the reference's path_tracer hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Nothing under tungsten_b200/ may include, link or call this.  It is used by tests/, by
 * __graft_entry__.smoke() and by bench.py's cpu_baseline leg as the checker for the CUDA path.
 * It consumes the same POD scene description as the product (include/tgb200.h) so both sides see
 * bit-identical inputs, and it is itself pinned against the reference binary (oracle/_ref, built
 * by oracle/ref/Makefile) through the golden framebuffers in tests/golden/.
 */
#ifndef PT_ORACLE_H_
#define PT_ORACLE_H_

#include "../include/tgb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct oracle_scene oracle_scene;

/* sobol = 1024 x 32 uint32 direction matrices (Joe-Kuo D6; tungsten_b200/data/sobol_1024x32.u32). */
oracle_scene *oracle_create(const tgb_scene_desc *desc, const uint32_t *sobol, char *err, int err_len);
void oracle_destroy(oracle_scene *s);

/* Same contract as tgb200_render_tiles.  threads <= 0: all cores. */
int oracle_render_tiles(oracle_scene *s, const tgb_tile *tiles, uint32_t n_tiles, uint32_t seed,
                        uint32_t spp_begin, uint32_t spp_count, float *rgb_mean, uint32_t *count,
                        int threads, tgb_stats *stats);

int oracle_trace_closest(oracle_scene *s, const tgb_ray *rays, tgb_hit *hits, uint32_t n);

/* Tile dicing + per-tile sampler seeds (PathTraceIntegrator.cpp:27-42,187).  tiles may be NULL to
 * query the count. */
uint32_t oracle_dice_tiles(uint32_t w, uint32_t h, uint32_t seed, tgb_tile *tiles);

/* Small known-answer hooks for the unit tests. */
uint32_t oracle_hash32(uint32_t x);
uint32_t oracle_pcg_next(uint64_t *state);
float    oracle_normalized_uint(uint32_t i);
uint32_t oracle_sobol_sample(const uint32_t *sobol, uint32_t index, uint32_t dim, uint32_t scramble);
void     oracle_filter_cdf(uint32_t filter, float *cdf32, float *bin_size);
float    oracle_diffuse_fresnel(float ior, int sample_count);
int      oracle_kat_eval(int which, const float *in, float *out);
int      oracle_bsdf_eval(oracle_scene *s, int index, float u, float v, const float *wi_wo, int n, float *out);
int      oracle_bsdf_sample(oracle_scene *s, uint32_t seed, int n, const int *bsdf_index, const uint32_t *pixel_id, uint32_t sample,
                            float u, float v, const float *wi, float *out, uint32_t *lobes);
int      oracle_light_probe(oracle_scene *s, int prim, uint32_t seed, int n, uint32_t sample, const float *p, float *out);
/* The same with a lobe mask `requested` and / or the supplemental PCG mode (0: reseeded per path like the renderer, 1: the stock
 * reference's serial stream, which the three above use). */
int      oracle_bsdf_eval_lobes(oracle_scene *s, int index, float u, float v, uint32_t requested, const float *wi_wo, int n, float *out);
int      oracle_bsdf_sample_lobes(oracle_scene *s, uint32_t seed, uint32_t supplemental_mode, uint32_t requested, int n,
                                  const int *bsdf_index, const uint32_t *pixel_id, uint32_t sample, float u, float v, const float *wi,
                                  float *out, uint32_t *lobes);
int      oracle_light_probe_mode(oracle_scene *s, int prim, uint32_t seed, uint32_t supplemental_mode, int n, uint32_t sample,
                                 const float *p, float *out);
int      oracle_choose_light(oracle_scene *s, uint32_t seed, int n, const uint32_t *pixel_id, uint32_t sample, const float *p, float *out);
int      oracle_shadow_probe(oracle_scene *s, int n, const float *query, const int *light_mis, float *out);
/* tgb200_bounce_probe's twin on records of TGB_BOUNCE_WORDS words.  camera = 0: one iteration of traceSample's loop from each
 * state (the sampler resumes at the record's dimension and PCG state); camera = 1: the camera state of (pixel, sample) for the
 * record's seed, the input of bounce 0 (only PIXEL, SEED and SAMPLE are read).  Returns -1 (nothing written) when a state to
 * step has bounce >= maxBounces. */
int      oracle_bounce_probe(oracle_scene *s, int camera, int n, const uint32_t *in, uint32_t *out);
/* Each segment of curve primitive prim on its own, for each ray: 7 words (see pt_oracle.c).  -1 when prim is not a curve. */
int      oracle_curve_segments_probe(oracle_scene *s, int prim, const tgb_ray *rays, const int *only, int n, uint32_t *out);
int      oracle_hair_eval(float roughness, float scale_angle_deg, const float *sigma_a, const float *wi_wo, int n, float *out);
int      oracle_hair_tables(float roughness, float scale_angle_deg, const float *sigma_a, float *tables, float *sums, float *v);

#ifdef __cplusplus
}
#endif
#endif
