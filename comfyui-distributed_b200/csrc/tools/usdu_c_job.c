/*
 * usdu_c_job.c -- a whole single-GPU Ultimate-SD-Upscale tile job driven through the C ABI of libusdu_b200.so
 * alone: no Python, no torch.  It is the host flow of INTEGRATION.md option B, with the deterministic T0 sampler
 * stand-in (usdu_t0_denoise) in place of a real sampler:
 *
 *   plan -> canvas (usdu_canvas_bytes, usdu_quantize_canvas) -> tables + feather masks on the device ->
 *   per dependency wave: usdu_tile_crop_resize, sampler, usdu_tile_blend -> the u8 canvas rows.
 *
 * usage: usdu_c_job W H B tile_width tile_height padding mask_blur uniform denoise image.f32 noise.bin out.u8
 *   image.f32  B*H*W*3 float32, values in [0, 1] (the IMAGE tensor, [B][H][W][3])
 *   noise.bin  the sampler's noise, already multiplied by `denoise`: records {int32 ph, int32 pw, then B*ph*pw*3 float32},
 *              one per processing size the plan uses (every tile of that size gets the same noise)
 *   out.u8     written: the B*H*W*3 bytes of the final canvas (the result is byte / 255.0f)
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cuda_runtime_api.h>

#include "../../../include/usdu_b200.h"

static void die(const char* what) {
    fprintf(stderr, "usdu_c_job: %s\n", what);
    exit(1);
}

static void check(int status, const char* what) {
    if (status < 0) {
        fprintf(stderr, "usdu_c_job: %s failed (%d): %s\n", what, status, usdu_last_error());
        exit(1);
    }
}

/* the size queries return int64_t: a size, or a negative usdu_status */
static int64_t check_size(int64_t n, const char* what) {
    if (n < 0) check((int)n, what);
    return n;
}

static void check_cuda(cudaError_t e, const char* what) {
    if (e != cudaSuccess) {
        fprintf(stderr, "usdu_c_job: %s: %s\n", what, cudaGetErrorString(e));
        exit(1);
    }
}

static void* xmalloc(size_t n) {
    void* p = malloc(n ? n : 1);
    if (!p) die("out of host memory");
    return p;
}

static void* dev_alloc(size_t n) {
    void* p = NULL;
    check_cuda(cudaMalloc(&p, n ? n : 16), "cudaMalloc");
    return p;
}

static void* upload(const void* src, size_t n) {
    void* p = dev_alloc(n);
    if (n) check_cuda(cudaMemcpy(p, src, n, cudaMemcpyHostToDevice), "cudaMemcpy (upload)");
    return p;
}

static void read_file(const char* path, void* dst, size_t n) {
    FILE* f = fopen(path, "rb");
    if (!f) die(path);
    if (fread(dst, 1, n, f) != n) die("short read");
    fclose(f);
}

typedef struct {
    int ph, pw;
    float* dev;
} noise_rec;

static const int32_t* g_geo;   /* usdu_plan_tiles, for by_shape */

/* same-shape tiles adjacent inside a wave: one sampler call per shape (ascending ph, pw, then tile id) */
static int by_shape(const void* a, const void* b) {
    const int i = *(const int32_t*)a, j = *(const int32_t*)b;
    const int32_t* ti = g_geo + (int64_t)i * USDU_PLAN_TILE_WORDS;
    const int32_t* tj = g_geo + (int64_t)j * USDU_PLAN_TILE_WORDS;
    if (ti[7] != tj[7]) return ti[7] < tj[7] ? -1 : 1;
    if (ti[6] != tj[6]) return ti[6] < tj[6] ? -1 : 1;
    return i < j ? -1 : (i > j);
}

int main(int argc, char** argv) {
    if (argc != 13) {
        fprintf(stderr, "usage: %s W H B tile_width tile_height padding mask_blur uniform denoise image.f32 noise.bin out.u8\n", argv[0]);
        return 2;
    }
    const int W = atoi(argv[1]), H = atoi(argv[2]), B = atoi(argv[3]);
    const int tile_w = atoi(argv[4]), tile_h = atoi(argv[5]), padding = atoi(argv[6]), mask_blur = atoi(argv[7]);
    const int uniform = atoi(argv[8]);
    const float denoise = strtof(argv[9], NULL);
    const float one_minus_d = 1.0f - denoise;          /* rounded in fp32, like the Python T0 sampler */
    if (B <= 0) die("B must be positive");

    /* ---- plan (host only) ---- */
    usdu_plan* plan = NULL;
    check(usdu_plan_create(W, H, tile_w, tile_h, padding, mask_blur, uniform, &plan), "usdu_plan_create");
    int64_t info[USDU_PLAN_INFO_WORDS];
    check(usdu_plan_info(plan, info), "usdu_plan_info");
    const int T = (int)info[USDU_PI_TILES], n_cls = (int)info[USDU_PI_MASK_CLASSES];
    int32_t* geo = xmalloc((size_t)T * USDU_PLAN_TILE_WORDS * sizeof(int32_t));
    int32_t* desc = xmalloc((size_t)T * USDU_TILE_WORDS * sizeof(int32_t));
    int32_t* tabs = xmalloc((size_t)info[USDU_PI_TAB_WORDS] * sizeof(int32_t));
    int32_t* specs = xmalloc((size_t)n_cls * USDU_MASK_WORDS * sizeof(int32_t));
    check(usdu_plan_tiles(plan, geo), "usdu_plan_tiles");
    check(usdu_plan_tile_desc(plan, desc), "usdu_plan_tile_desc");
    check(usdu_plan_tables(plan, tabs), "usdu_plan_tables");
    check(usdu_plan_mask_specs(plan, specs), "usdu_plan_mask_specs");

    /* ---- sampler noise, one record per processing size ---- */
    noise_rec* noise = NULL;
    int n_noise = 0;
    {
        FILE* f = fopen(argv[11], "rb");
        if (!f) die(argv[11]);
        int32_t hdr[2];
        while (fread(hdr, sizeof(int32_t), 2, f) == 2) {
            if (hdr[0] <= 0 || hdr[1] <= 0) die("bad noise record header");
            const size_t n = (size_t)B * hdr[0] * hdr[1] * 3;
            float* h = xmalloc(n * sizeof(float));
            if (fread(h, sizeof(float), n, f) != n) die("short noise record");
            noise = realloc(noise, (size_t)(n_noise + 1) * sizeof(noise_rec));
            if (!noise) die("out of host memory");
            noise[n_noise].ph = hdr[0];
            noise[n_noise].pw = hdr[1];
            noise[n_noise].dev = upload(h, n * sizeof(float));
            ++n_noise;
            free(h);
        }
        fclose(f);
    }

    /* ---- canvas: the quantised image, with the kernels' slack behind the last row ---- */
    const int64_t pitch = check_size(usdu_canvas_pitch(W), "usdu_canvas_pitch");
    const int64_t canvas_bytes = check_size(usdu_canvas_bytes(B, H, W), "usdu_canvas_bytes");
    uint8_t* canvas = dev_alloc((size_t)canvas_bytes);
    {
        const size_t n = (size_t)B * H * W * 3;
        float* img = xmalloc(n * sizeof(float));
        read_file(argv[10], img, n * sizeof(float));
        float* img_dev = upload(img, n * sizeof(float));
        free(img);
        check(usdu_quantize_canvas(img_dev, canvas, B, H, W, pitch, NULL), "usdu_quantize_canvas");
        check_cuda(cudaDeviceSynchronize(), "quantize");
        check_cuda(cudaFree(img_dev), "cudaFree");
    }

    /* ---- plan tables and feather templates on the device ---- */
    int32_t* desc_dev = upload(desc, (size_t)T * USDU_TILE_WORDS * sizeof(int32_t));
    int32_t* tabs_dev = upload(tabs, (size_t)info[USDU_PI_TAB_WORDS] * sizeof(int32_t));
    uint8_t* mask_pool = dev_alloc((size_t)info[USDU_PI_MASK_POOL_BYTES]);
    {
        const int64_t scratch_bytes = check_size(usdu_mask_scratch_bytes(specs, n_cls), "usdu_mask_scratch_bytes");
        uint8_t* scratch = dev_alloc((size_t)scratch_bytes);
        check(usdu_build_feather_masks(specs, n_cls, mask_pool, scratch, NULL), "usdu_build_feather_masks");
        check_cuda(cudaDeviceSynchronize(), "feather masks");
        check_cuda(cudaFree(scratch), "cudaFree");
    }

    /* ---- the progressive job, wave by wave ---- */
    int32_t* order = xmalloc((size_t)T * sizeof(int32_t));
    int32_t* level = xmalloc((size_t)T * sizeof(int32_t));
    int32_t* ids = xmalloc((size_t)T * sizeof(int32_t));
    for (int i = 0; i < T; ++i) order[i] = i;
    const int n_waves = usdu_plan_waves(plan, order, T, level);
    check(n_waves, "usdu_plan_waves");
    g_geo = geo;
    for (int k = 0; k < n_waves; ++k) {
        int n = 0;
        for (int i = 0; i < T; ++i)
            if (level[i] == k) ids[n++] = order[i];
        qsort(ids, (size_t)n, sizeof(int32_t), by_shape);

        /* crop: canvas windows -> fp32 tiles at processing size, packed in list order */
        usdu_worklist* cw = NULL;
        check(usdu_plan_crop_worklist(plan, ids, n, B, 2, 0, 0, &cw), "usdu_plan_crop_worklist");
        int64_t ci[USDU_WL_INFO_WORDS];
        check(usdu_worklist_info(cw, ci), "usdu_worklist_info");
        const size_t citems_bytes = (size_t)(ci[USDU_WL_ITEMS] * ci[USDU_WL_ITEM_WORDS]) * sizeof(int32_t);
        int32_t* citems = xmalloc(citems_bytes);
        int64_t* slots = xmalloc((size_t)n * sizeof(int64_t));
        check(usdu_worklist_items(cw, citems), "usdu_worklist_items");
        check(usdu_worklist_slots(cw, slots), "usdu_worklist_slots");
        int32_t* citems_dev = upload(citems, citems_bytes);
        float* tiles_dev = dev_alloc((size_t)ci[USDU_WL_TOTAL] * sizeof(float));
        float* out_dev = dev_alloc((size_t)ci[USDU_WL_TOTAL] * sizeof(float));
        check(usdu_tile_crop_resize(canvas, B, H, W, pitch, desc_dev, tabs_dev, citems_dev, (int)ci[USDU_WL_GRID],
                                    (int)ci[USDU_WL_PATCH_W], (int)ci[USDU_WL_PATCH_H], tiles_dev, (int)ci[USDU_WL_FLAGS], NULL),
              "usdu_tile_crop_resize");

        /* sampler stand-in: one call per run of same-shape tiles */
        for (int i = 0; i < n;) {
            const int32_t* t = geo + (int64_t)ids[i] * USDU_PLAN_TILE_WORDS;
            const int ph = t[7], pw = t[6];
            int j = i + 1;
            while (j < n && geo[(int64_t)ids[j] * USDU_PLAN_TILE_WORDS + 7] == ph && geo[(int64_t)ids[j] * USDU_PLAN_TILE_WORDS + 6] == pw) ++j;
            const float* nd = NULL;
            for (int r = 0; r < n_noise; ++r)
                if (noise[r].ph == ph && noise[r].pw == pw) nd = noise[r].dev;
            if (!nd) {
                fprintf(stderr, "usdu_c_job: no noise record for processing size %dx%d\n", pw, ph);
                return 1;
            }
            const int64_t frame = (int64_t)B * ph * pw * 3;
            check(usdu_t0_denoise(tiles_dev + slots[i], nd, out_dev + slots[i], frame * (j - i), frame, one_minus_d, NULL),
                  "usdu_t0_denoise");
            i = j;
        }

        /* blend: the sampler output back into the canvas, in list order */
        usdu_worklist* bw = NULL;
        check(usdu_plan_blend_worklist(plan, ids, slots, n, 4, B, 2, 0, 0, 0, 0, &bw), "usdu_plan_blend_worklist");
        int64_t bi[USDU_WL_INFO_WORDS];
        check(usdu_worklist_info(bw, bi), "usdu_worklist_info");
        const size_t bitems_bytes = (size_t)(bi[USDU_WL_ITEMS] * bi[USDU_WL_ITEM_WORDS]) * sizeof(int32_t);
        const size_t cover_bytes = (size_t)bi[USDU_WL_COVER] * USDU_COVER_WORDS * sizeof(int32_t);
        int32_t* bitems = xmalloc(bitems_bytes);
        int32_t* cover = xmalloc(cover_bytes);
        check(usdu_worklist_items(bw, bitems), "usdu_worklist_items");
        if (cover_bytes) check(usdu_worklist_cover(bw, cover), "usdu_worklist_cover");
        int32_t* bitems_dev = upload(bitems, bitems_bytes);
        int32_t* cover_dev = cover_bytes ? upload(cover, cover_bytes) : NULL;
        if (bi[USDU_WL_ITEMS] > 0)
            check(usdu_tile_blend(canvas, B, H, W, pitch, desc_dev, tabs_dev, mask_pool, bitems_dev, (int)bi[USDU_WL_GRID], cover_dev,
                                  (int)bi[USDU_WL_PATCH_W], (int)bi[USDU_WL_PATCH_H], out_dev, 0, (int)bi[USDU_WL_FLAGS], NULL),
                  "usdu_tile_blend");
        check_cuda(cudaDeviceSynchronize(), "wave");

        check_cuda(cudaFree(citems_dev), "cudaFree");
        check_cuda(cudaFree(tiles_dev), "cudaFree");
        check_cuda(cudaFree(out_dev), "cudaFree");
        check_cuda(cudaFree(bitems_dev), "cudaFree");
        if (cover_dev) check_cuda(cudaFree(cover_dev), "cudaFree");
        free(citems);
        free(slots);
        free(bitems);
        free(cover);
        check(usdu_worklist_destroy(cw), "usdu_worklist_destroy");
        check(usdu_worklist_destroy(bw), "usdu_worklist_destroy");
    }

    /* ---- result: the u8 canvas rows ---- */
    {
        const size_t row = (size_t)W * 3, n = (size_t)B * H * row;
        uint8_t* out = xmalloc(n);
        check_cuda(cudaMemcpy2D(out, row, canvas, (size_t)pitch, row, (size_t)B * H, cudaMemcpyDeviceToHost), "cudaMemcpy2D");
        FILE* f = fopen(argv[12], "wb");
        if (!f) die(argv[12]);
        if (fwrite(out, 1, n, f) != n) die("short write");
        if (fclose(f) != 0) die("close");
        free(out);
    }

    for (int r = 0; r < n_noise; ++r) cudaFree(noise[r].dev);
    free(noise);
    cudaFree(canvas);
    cudaFree(desc_dev);
    cudaFree(tabs_dev);
    cudaFree(mask_pool);
    free(geo); free(desc); free(tabs); free(specs); free(order); free(level); free(ids);
    check(usdu_plan_destroy(plan), "usdu_plan_destroy");
    return 0;
}
