/*
 * Capture shim for tests/test_dropin_scene.py: a stand-in for libtgb200.so's tgb200_create that writes the scene description
 * the drop-in adapter hands the library (every struct and every array it points to) to the file named by $TGB_CAPTURE, then
 * ends the process with _exit(0).  Preloaded (LD_PRELOAD) into oracle/_ref/dropin/tungsten_b200, it takes the place of the
 * library's symbol, so the adapter's desc is read without a GPU and without touching CUDA.
 *
 * File format: a sequence of blocks, each a little-endian uint64 byte count followed by that many bytes:
 *   desc, primitives[n_primitives], bsdfs[n_bsdfs], bsdf_slots[n_bsdf_slots], textures[n_textures],
 *   then per primitive: verts, tris, curve_nodes (4 floats each), curve_segments,
 *   then per texture: texels (res_u*res_v*3 floats for bitmaps, empty otherwise),
 *   then the 8-byte end marker "TGBCAPOK".
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <unistd.h>

#include "tgb200.h"

static void block(FILE *f, const void *p, uint64_t n)
{
    fwrite(&n, sizeof(n), 1, f);
    if (n && p)
        fwrite(p, 1, (size_t)n, f);
    else if (n) {
        /* a NULL pointer with a non-zero count: write zeros so the reader still sees the declared size */
        static const char zero[4096];
        for (uint64_t done = 0; done < n; done += sizeof(zero))
            fwrite(zero, 1, (size_t)(n - done < sizeof(zero) ? n - done : sizeof(zero)), f);
    }
}

int tgb200_create(const tgb_scene_desc *s, tgb_ctx **out)
{
    const char *path = getenv("TGB_CAPTURE");
    FILE *f = path ? fopen(path, "wb") : NULL;
    uint32_t i;
    (void)out;
    if (!f)
        _exit(3);
    block(f, s, sizeof(*s));
    block(f, s->primitives, sizeof(tgb_primitive)*(uint64_t)s->n_primitives);
    block(f, s->bsdfs, sizeof(tgb_bsdf)*(uint64_t)s->n_bsdfs);
    block(f, s->bsdf_slots, sizeof(uint32_t)*(uint64_t)s->n_bsdf_slots);
    block(f, s->textures, sizeof(tgb_texture)*(uint64_t)s->n_textures);
    for (i = 0; i < s->n_primitives; ++i) {
        const tgb_primitive *p = s->primitives + i;
        block(f, p->verts, sizeof(tgb_vertex)*(uint64_t)p->n_verts);
        block(f, p->tris, sizeof(tgb_triangle)*(uint64_t)p->n_tris);
        block(f, p->curve_nodes, 4*sizeof(float)*(uint64_t)p->n_curve_nodes);
        block(f, p->curve_segments, sizeof(uint32_t)*(uint64_t)p->n_curve_segments);
    }
    for (i = 0; i < s->n_textures; ++i) {
        const tgb_texture *t = s->textures + i;
        block(f, t->texels, t->type == TGB_TEX_BITMAP ? 3*sizeof(float)*(uint64_t)t->res_u*t->res_v : 0);
    }
    fwrite("TGBCAPOK", 1, 8, f);
    if (fclose(f) != 0)
        _exit(4);
    _exit(0);
}
