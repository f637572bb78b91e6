/*
 * usdu_b200.h -- C ABI of libusdu_b200.so: the H100-native (sm_90a) replacement for the
 * CPU/Pillow pixel path of ComfyUI-Distributed's Ultimate-SD-Upscale tile pipeline.
 *
 * The boundary is plain C: raw pointers, sizes, a CUDA stream handle passed as void*.
 * No torch types.  Device pointers are marked _dev; everything else is host memory.
 * Every entry point returns 0 on success or a negative usdu_status; the message of the
 * last failure on the calling thread is available from usdu_last_error().  There is no
 * CPU fallback: without a CUDA device every compute entry point fails with
 * USDU_ERR_CUDA.
 *
 * Reference interfaces replaced (file:line are relative to robertvoy/ComfyUI-Distributed
 * @ a91f9fb):
 *   utils/image.py:8-18                tensor_to_pil / pil_to_tensor
 *   upscale/tile_ops.py:34-155         extract_[batch_]tile_with_padding (crop + LANCZOS)
 *   upscale/tile_ops.py:289-308        create_tile_mask (rectangle + GaussianBlur)
 *   upscale/tile_ops.py:310-349        blend_tile (LANCZOS back + alpha composite)
 *   upscale/worker_comms.py:16-108     tile payload packing (PNG) -> usdu_pack_tiles_u8
 * The geometry (upscale/tile_ops.py:14-32, utils/usdu_utils.py:49-112) runs on the host, like
 * the reference, inside this library: the planner section at the end (usdu_plan_create ...)
 * builds the tile geometry, the descriptor and table arrays documented below, the dependency
 * waves and the work lists of every kernel, so a C/C++ host drives the whole tile path
 * without Python (csrc/tools/usdu_c_job.c is a complete single-GPU job).
 */
#ifndef USDU_B200_H
#define USDU_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library itself is built with -fvisibility=hidden */
#endif

#define USDU_ABI_VERSION 19

typedef enum usdu_status {
    USDU_OK = 0,
    USDU_ERR_INVALID = -1,   /* bad argument (null pointer, negative size, misaligned pitch ...) */
    USDU_ERR_CUDA = -2,      /* CUDA runtime error (no device, launch failure ...) */
    USDU_ERR_UNSUPPORTED = -3
} usdu_status;

/* ---- descriptor layouts (all int32, little endian, device-resident unless noted) ------
 *
 * Tile descriptor: USDU_TILE_WORDS int32 per tile position (geometry is identical for all
 * frames of a batch, upscale/tile_ops.py:108-138).
 */
#define USDU_TILE_WORDS 24
#define USDU_T_X1 0          /* crop window origin on the canvas */
#define USDU_T_Y1 1
#define USDU_T_EW 2          /* crop window ("extracted") size */
#define USDU_T_EH 3
#define USDU_T_PW 4          /* processing size handed to the sampler */
#define USDU_T_PH 5
#define USDU_T_MASK_OFF 6    /* byte offset of this tile's feather template in the mask pool */
#define USDU_T_MASK_PITCH 7  /* bytes per template row (>= EW) */
#define USDU_T_TAB_CROP_H 8  /* int32 offset of a resample table in the table pool (an identity table when the axis keeps its size; -1 is accepted by the generic kernels only) */
#define USDU_T_TAB_CROP_V 9  /*   crop:  EW->PW (H), EH->PH (V) */
#define USDU_T_TAB_BLEND_H 10 /*  blend: PW->EW (H), PH->EH (V) */
#define USDU_T_TAB_BLEND_V 11
#define USDU_T_SUP_X0 12     /* bbox of the template's non-zero alpha, window coordinates */
#define USDU_T_SUP_Y0 13
#define USDU_T_SUP_X1 14
#define USDU_T_SUP_Y1 15
#define USDU_T_FULL_X0 16    /* window-relative box inside which the template alpha is exactly 255 */
#define USDU_T_FULL_Y0 17
#define USDU_T_FULL_X1 18
#define USDU_T_FULL_Y1 19    /* words 20..23 reserved (0) */

/* Resample table at int32 offset o of the table pool:
 *   [o+0]=in_size [o+1]=out_size [o+2]=ksize [o+3]=max taps actually used by any output
 *   [o+4]=offset (from o) of the packed rows, 0 when the fast kernels cannot use this table
 *   [o+5]=max inputs read by USDU_FAST_GROUP consecutive outputs
 *   [o+6]=int32 per packed row: 8 (<= 7 taps) or 16 (<= 15 taps)  [o+7]=0
 *   [o+8 ...]            bounds: out_size x {first input index, tap count}
 *   [o+8+2*out_size ...] kk: out_size x ksize coefficients, 22-bit fixed point
 *   then packed rows: out_size x [o+6] = {first input index, k0..k6} or {first, k0..k14}, zero padded
 * (Pillow Resample.c precompute_coeffs + normalize_coeffs_8bpc.) */
#define USDU_TAB_HEADER 8
#define USDU_PACKED_ROW 8
#define USDU_FAST_TAPS 7     /* taps per output of the narrow fast path (packed rows of 8 int32) */
#define USDU_FAST_TAPS_WIDE 15 /* ... and of the wide one (packed rows of 16 int32): scales up to ~2.3 */
#define USDU_FAST_GROUP 8    /* table word 5 = inputs read by this many consecutive outputs (diagnostic) */

/* Crop work item: one block of one tile's processing-size output. */
#define USDU_CROP_ITEM_WORDS 6
/*   [0]=tile id [1]=ox0 [2]=oy0 [3]=out offset lo [4]=out offset hi [5]=block rows (fast path; <= 32)
 *   out offset: element offset of this tile's [B][PH][PW][3] block in `out`. */

/* Blend work item: one canvas block and the ordered list of tiles composited into it. */
#define USDU_BLEND_ITEM_WORDS 4
/*   [0]=block x0 [1]=block y0 [2]=first cover entry [3]=cover count */
#define USDU_COVER_WORDS 4
/*   [0]=tile id [1]=src offset lo [2]=src offset hi [3]=0
 *   src offset: element offset of the tile's [B][PH][PW][3] processed block in `src`.
 *   Entries of one item are applied in list order (ascending tile id reproduces
 *   upscale/modes/static.py:521-553). */

/* Fast-path job record (USDU_FLAG_FAST): USDU_JOB_WORDS int32, one per (block, tile), built by
 * the planner so that a CTA needs ONE dependent load before it can start streaming pixels.
 * With USDU_FLAG_FAST `items_dev` of the two tile kernels holds these records instead of the
 * generic work items (and `cover_dev` is ignored): the grid is the first n_items records;
 * further records of the same canvas block are chained through USDU_J_NEXT. */
#define USDU_JOB_WORDS 32
#define USDU_J_SRC_A 0     /* crop: canvas px of the first staged column (multiple of 4)
                              blend: element offset (low 32 bits) of the first staged element, frame 0 */
#define USDU_J_SRC_B 1     /* crop: canvas row of the first staged row; blend: high 32 bits */
#define USDU_J_LEAD 2      /* pixels between the staged column 0 and the first needed input pixel (0..3) */
#define USDU_J_COLS 3      /* needed input pixels */
#define USDU_J_ROWS 4      /* staged input rows */
#define USDU_J_IX0 5       /* first needed input pixel / row in axis coordinates */
#define USDU_J_IY0 6
#define USDU_J_ROWS_H 7    /* table-pool index of packed row 0 of the horizontal axis */
#define USDU_J_OX_BASE 8   /* output index of block column 0 (may be negative) */
#define USDU_J_N_OUT_H 9
#define USDU_J_ROWS_V 10
#define USDU_J_OY_BASE 11
#define USDU_J_N_OUT_V 12
#define USDU_J_DST_X 13    /* crop: output pixel of block column 0; blend: canvas pixel of block column 0 */
#define USDU_J_DST_Y 14
#define USDU_J_OFF_LO 15   /* crop: element offset of the tile's [B][PH][PW][3] block in out */
#define USDU_J_OFF_HI 16   /* blend: byte offset (signed 64 bit) of block pixel (0,0) in the mask pool */
#define USDU_J_ROWS_OUT 17 /* crop: valid output rows; blend: rows to run (= CY1) */
#define USDU_J_COLS_OUT 18 /* crop: valid output pixels */
#define USDU_J_CX0 19      /* blend: block-relative box outside which this tile leaves the canvas untouched */
#define USDU_J_CX1 20
#define USDU_J_CY0 21
#define USDU_J_CY1 22
#define USDU_J_FLAGS 23    /* bit 0: the whole block lies in the tile's opaque core (alpha == 255) */
#define USDU_J_MPITCH 24   /* blend: feather template pitch */
#define USDU_J_PITCH 25    /* elements per source row (blend) / per output row (crop): PW*3 */
#define USDU_J_FRAME_LO 26 /* elements per frame PH*PW*3 */
#define USDU_J_FRAME_HI 27
#define USDU_J_NEXT 28     /* blend: index of the next record of the same block, -1 = last */
#define USDU_J_TAPS_H 29   /* taps of the horizontal / vertical axis: 1..USDU_FAST_TAPS (packed rows of 8 int32; a value
                              <= 6 lets the kernel skip the unused last slot) or USDU_FAST_TAPS_WIDE (rows of 16) */
#define USDU_J_TAPS_V 30

/* Feather-mask spec (host array, USDU_MASK_WORDS int32 each). */
#define USDU_MASK_WORDS 16
/*   [0]=W [1]=H canvas; [2..5]=bx1,by1,bx2,by2 clipped inclusive-rectangle bbox (exclusive
 *   right/bottom); [6..9]=x1,y1,x2,y2 window; [10]=blur radius (mask_blur, 0 = none);
 *   [11]=out byte offset in the mask pool; [12]=out pitch; [13..15]=0 */

/* canvas block edge used by the blend / crop kernels (pixels) */
#define USDU_BLOCK_W 64
#define USDU_BLOCK_H 32
/* ... and by the fast kernels (USDU_FLAG_FAST): work items must be built with these */
#define USDU_FAST_BLOCK_W 128
#define USDU_FAST_BLOCK_H 32

/* ---- library ------------------------------------------------------------------------ */
int usdu_abi_version(void);
const char* usdu_last_error(void);
/* number of CUDA devices visible, or a negative usdu_status */
int usdu_device_count(void);
/* streaming multiprocessors of the current CUDA device, or a negative usdu_status */
int usdu_sm_count(void);

/* Resident CTAs per SM of a tensor-core kernel build at the dynamic shared memory its launcher requests for the patch
 * words of a work list (USDU_WL_PATCH_W / _H; block_rows: the blend's block height): kernel = USDU_KERNEL_CROP_LDG,
 * USDU_KERNEL_CROP_TMA (| USDU_KERNEL_LARGE: the 4-CTA build of launches of >= 8 CTAs per SM) or USDU_KERNEL_BLEND
 * (fp32 sources); two_ksteps: the USDU_FLAG_MMA_KS2 build.  use_device = 1: the current device's occupancy calculator;
 * 0: the table of the kernels' launch bounds and 228 KB of shared memory per SM.  0 = does not fit an SM. */
#define USDU_KERNEL_CROP_LDG 0
#define USDU_KERNEL_CROP_TMA 1
#define USDU_KERNEL_BLEND 2
#define USDU_KERNEL_LARGE 4
int usdu_mma_resident_ctas(int kernel, int two_ksteps, int patch_w, int patch_h, int block_rows, int use_device);

/* ---- host-side table builders (exact Pillow arithmetic, C double / C float) -------- */
/* taps per output for an in->out LANCZOS axis (Resample.c: ceil(3*max(in/out,1))*2+1) */
int usdu_resample_ksize(int in_size, int out_size);
/* number of int32 words of a table: USDU_TAB_HEADER + out*(2+ksize) */
int64_t usdu_resample_table_words(int in_size, int out_size);
/* fill `table` (host, usdu_resample_table_words() int32) */
int usdu_build_resample_table(int in_size, int out_size, int32_t* table);
/* The same for any of Pillow's separable filters used on the path: LANCZOS for the tiles
 * (upscale/tile_ops.py:88,148,329), BICUBIC for conditioning masks (utils/usdu_utils.py:424,435). */
#define USDU_FILTER_LANCZOS 0
#define USDU_FILTER_BICUBIC 1
int usdu_filter_ksize(int filter, int in_size, int out_size);
int64_t usdu_filter_table_words(int filter, int in_size, int out_size);
int usdu_build_filter_table(int filter, int in_size, int out_size, int32_t* table);
/* source index of every output sample of Image.resize(..., NEAREST) along one axis
 * (Geometry.c ImagingScaleAffine; used by pad_image2's edge strips, utils/usdu_utils.py:190-199) */
int usdu_nearest_index(int in_size, int out_size, int32_t* index_host);
/* table of an axis that keeps its size (size -> size): one tap of weight 2^22;
 * ((USDU_TAB_HEADER + 3*size + 3) & ~3) + size * USDU_PACKED_ROW int32.  Tables must start at a
 * multiple of 4 int32 in the pool (their packed rows are read with 128-bit loads). */
int usdu_build_identity_table(int size, int32_t* table);
/* ImageFilter.GaussianBlur(radius) -> extended-box parameters (BoxBlur.c, 3 passes) */
int usdu_box_blur_params(float radius, int32_t* rad, uint32_t* ww, uint32_t* fw);

/* ---- device kernels ----------------------------------------------------------------- */
/* `flags` of the two tile kernels: USDU_FLAG_FAST selects the register-window kernels
 * (usdu_fast.cu); the caller may set it only when every table referenced by the launch has
 * packed rows (table word 4 != 0) and no table offset is -1.  Without it the generic
 * kernels run (any scale, any tap count). */
#define USDU_FLAG_FAST 1
/* USDU_FLAG_MMA selects the tensor-core kernels (usdu_mma.cu: every LANCZOS tap runs as mma.sync.m16n8k32 on 8-bit
 * coefficient limbs, bit-identical results).  items_dev then holds job records in the TENSOR-CORE flavour: the same 32
 * words, with USDU_J_ROWS_H / _V = table-pool index of the axis' fragment section (built by usdu_plan_create;
 * {n_mtiles, ksteps, 0, 0} then per M-tile {k0, 0, 0, 0, per (k-step, limb) 32 lanes x 4 registers}),
 * USDU_J_TAPS_H / _V = k-steps (1 or 2), USDU_J_IX0 / _IY0 = first staged input column / row (multiples of 4),
 * USDU_J_COLS a multiple of 4, USDU_J_LEAD = 0, crop: USDU_J_SRC_A a multiple of 4 and USDU_J_CY1 = block rows (16 / 32).
 * patch_w = bytes a plane row must hold (staged pixels or the reach of the last K window, whichever is larger);
 * patch_h = plane rows (multiple of 8) in bits 0..15, rows of the intermediate the kernel allocates (multiple of 4, >= plane
 * rows) in bits 16..31; the byte planes lie right behind the intermediate in shared memory, so vertical K windows may reach
 * past the allocated rows (zero coefficients) as long as they stay inside the planes.
 * usdu_tile_blend: block height 16 or 32 in flags bits 8..15. */
#define USDU_FLAG_MMA 2
/* ... some record of the launch has USDU_J_TAPS_H or _V == 2 (an axis scaled by more than ~1.4): run the two-k-step build */
#define USDU_FLAG_MMA_KS2 4
/* usdu_tile_blend with USDU_FLAG_FAST: bits 8..15 of `flags` carry the canvas block height the
 * job records were built for (1..USDU_FAST_BLOCK_H); the canvas block travels by TMA. */
#define USDU_FLAG_BLOCK_ROWS(n) ((n) << 8)
/* generic kernels (no USDU_FLAG_FAST): optional block size the work items were built for, rows in
 * bits 8..15 (<= USDU_BLOCK_H), columns in bits 16..23 (<= USDU_BLOCK_W); 0 = the default block.
 * The planner shrinks blocks when an extreme down-scale would not fit shared memory. */
#define USDU_FLAG_BLOCK_COLS(n) ((n) << 16)
/* usdu_tile_blend (integer-pipe kernels): canvas_dev is ANOTHER device's memory mapped into this process (NVLink peer
 * access); the kernel then waits for its bulk stores to complete, not only to be read, and issues a system-scope fence
 * before a CTA exits.  Round 1's multi-GPU final blend stored into the master's canvas this way; since round 2 every rank
 * composites a slab of the final canvas in its OWN memory and the master gathers the slabs with peer loads
 * (usdu_gather_dequantize), so nothing in the package sets this flag any more. */
#define USDU_FLAG_REMOTE_CANVAS (1 << 24)
/* Q0: canvas_u8[b][y][x*3+c] = (uint8)(255.f * img[b][y][x][c])   (utils/image.py:8-10)
 * pitch = bytes per canvas row (>= 3*W, multiple of 16); frame stride = H*pitch.
 * The allocation behind a canvas must hold USDU_CANVAS_SLACK bytes more than B*H*pitch: the staging of the
 * integer-pipe kernels reads whole 12-byte chunks and, for widths that are not multiples of 4, may touch up to 4
 * bytes past the last row's pitch (the values are discarded).  usdu_canvas_bytes() gives the size to allocate. */
#define USDU_CANVAS_SLACK 16
/* bytes per canvas row the package uses: 3*W rounded up to 128 */
int64_t usdu_canvas_pitch(int W);
/* B*H*usdu_canvas_pitch(W) + USDU_CANVAS_SLACK */
int64_t usdu_canvas_bytes(int B, int H, int W);
int usdu_quantize_canvas(const float* img_dev, uint8_t* canvas_dev, int B, int H, int W,
                         int64_t pitch, void* stream);
/* canvas u8 -> fp32 image (u / 255.0f, utils/image.py:12-14) */
int usdu_dequantize_canvas(const uint8_t* canvas_dev, float* img_dev, int B, int H, int W,
                           int64_t pitch, void* stream);
/* The same two casts on canvas rows [y0, y1) of EVERY frame (img_dev / canvas_dev are the bases of the whole
 * [B][H][W][3] image and [B][H][pitch] canvas).  Multi-GPU jobs quantise, composite and dequantise the canvas slab by
 * slab: canvas_dev of usdu_dequantize_rows may be a PEER's canvas mapped over NVLink (the master gathers the final
 * slabs of all ranks while it dequantises, upscale/modes/static.py:556-564 'result tensor'). */
int usdu_quantize_rows(const float* img_dev, uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                       int y0, int y1, void* stream);
int usdu_dequantize_rows(const uint8_t* canvas_dev, float* img_dev, int B, int H, int W, int64_t pitch,
                         int y0, int y1, void* stream);
/* The same two casts as launches a captured CUDA graph can replay for any caller's tensors, meant to run in row bands
 * on a side stream beside the wave loop.  The fp32 image (quantise) and result (dequantise) are not launch arguments:
 * each kernel reads them from a DEVICE-resident usdu_stream_args block, which usdu_stream_args_set rewrites on `stream`
 * before the graph is replayed there (one 16-byte copy; the host array is staged by the driver before the call returns,
 * so back-to-back calls need no pinned buffer).  At most max_ctas CTAs stride over the band (1 <= max_ctas): a
 * bandwidth-bound pass that holds only a few CTA slots leaves the others to the latency-bound wave kernels.  Needs W % 4
 * == 0 and 16-byte aligned canvas, image and result (checked here and by usdu_stream_args_set). */
typedef struct usdu_stream_args {
    const float* img_dev;   /* [B][H][W][3] input of usdu_quantize_rows_streamed */
    float* out_dev;         /* [B][H][W][3] result of usdu_dequantize_rows_streamed */
} usdu_stream_args;
int usdu_stream_args_set(usdu_stream_args* args_dev, const float* img_dev, float* out_dev, void* stream);
int usdu_quantize_rows_streamed(const usdu_stream_args* args_dev, uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                                int y0, int y1, int max_ctas, void* stream);
int usdu_dequantize_rows_streamed(const uint8_t* canvas_dev, const usdu_stream_args* args_dev, int B, int H, int W,
                                  int64_t pitch, int y0, int y1, int max_ctas, void* stream);
/* Instantiate a captured graph (cudaGraph_t passed as void*) for replay.  high_priority != 0: every kernel node except
 * the two streamed casts above gets the device's greatest stream priority and the graph is instantiated with
 * cudaGraphInstantiateFlagUseNodePriority, so the wave kernels win CTA dispatch over a cast band running beside them.
 * *exec_out receives the cudaGraphExec_t; launch it with usdu_graph_launch, free it with usdu_graph_exec_destroy. */
int usdu_graph_instantiate(void* graph, int high_priority, void** exec_out);
int usdu_graph_launch(void* exec, void* stream);
int usdu_graph_exec_destroy(void* exec);
/* The master's gather of a multi-GPU job in ONE launch: canvas rows [slab_rows[q], slab_rows[q+1]) are read from
 * slab_canvas_dev[q] (host array of n_slabs device pointers, each the base of a whole [B][H][pitch] canvas: the local one
 * or a peer's mapped over NVLink) and dequantised into the local fp32 image.  slab_rows (host, n_slabs + 1 ints) must
 * start at 0 and end at H.  Replaces the master's drain loop + result conversion, upscale/result_collector.py:36-182 and
 * upscale/modes/static.py:556-564. */
#define USDU_MAX_SLABS 16
int usdu_gather_dequantize(const uint8_t* const* slab_canvas_dev, const int32_t* slab_rows, int n_slabs,
                           float* img_dev, int B, int H, int W, int64_t pitch, void* stream);
/* The all-gather of the quantised INPUT slabs in one launch (host path of a multi-GPU job): rows
 * [slab_rows[q], slab_rows[q+1]) of canvas_dev are copied from slab_canvas_dev[q]; the slab whose pointer IS canvas_dev
 * (this rank's own) is skipped.  Replaces every worker holding the whole canvas, upscale/modes/static.py:209-212. */
int usdu_gather_canvas(const uint8_t* const* slab_canvas_dev, const int32_t* slab_rows, int n_slabs,
                       uint8_t* canvas_dev, int B, int H, int W, int64_t pitch, void* stream);
/* Q1 for transport: dst[i] = (uint8)(255.f * src[i]); n elements (worker_comms.py:30-33) */
int usdu_pack_tiles_u8(const float* src_dev, uint8_t* dst_dev, int64_t n, void* stream);
/* receiving side of the transport: dst[i] = src[i] / 255.0f (api/job_routes.py:104-132) */
int usdu_unpack_tiles_f32(const uint8_t* src_dev, float* dst_dev, int64_t n, void* stream);

/* Collector worker transport (nodes/collector.py:84-119): each u8 frame [H, W, C] as the base64 text of one PNG,
 * what the reference's worker POSTs to /distributed/job_complete.  The PNG is stored (deflate level 0, filter None),
 * its bytes fixed by this layout (tests/png_model.py png_stored_b64 states it in numpy):
 *   8-byte signature; IHDR (W, H, depth 8, colour type 4 / 2 / 6 for C = 2 / 3 / 4, compression, filter, interlace 0);
 *   the raw stream R = per row a filter byte 0 and the row's W*C bytes, |R| = H*(1 + W*C), cut into stored deflate
 *   blocks of 65535 bytes (the last shorter); block k alone in IDAT chunk k, whose data is [78 01 if k == 0] +
 *   [BFINAL | BTYPE 00] + LEN (le16) + NLEN (le16) + the block; one IDAT chunk holding the big-endian Adler-32 of R;
 *   IEND.  Text: standard base64 alphabet, '=' padding, no line breaks, no terminator.
 * usdu_png_sizes: for one frame, the PNG length, the text length and the device staging bytes; USDU_ERR_INVALID
 * unless C is 2, 3 or 4 and H, W >= 1.
 * usdu_png_base64_u8: src_dev = B contiguous u8 frames [H, W, C]; staging_dev = B * staging bytes (16-byte aligned,
 * scratch); frame b's text goes to text_dev + b * text length (text_dev 4-byte aligned).  Three launches on `stream`,
 * no host synchronisation.  B <= 65535. */
int usdu_png_sizes(int H, int W, int C, int64_t* png_len, int64_t* text_len, int64_t* staging_bytes);
int usdu_png_base64_u8(const uint8_t* src_dev, int B, int H, int W, int C, uint8_t* staging_dev, char* text_dev,
                       void* stream);

/* Master side of the static-mode transport (upscale/payload_parsers.py:32-36): the level-0 PNG tiles workers post,
 * decoded to u8 RGB frames in one launch, one CTA per frame.  The host validates each file and cuts it into segments:
 * runs of the uploaded bytes that, in order, form the frame's filtered stream R (per row a filter byte 0..4, then the
 * row's W*C bytes; |R| = H*(1 + W*C)), chunk framing, zlib header and stored-block headers left out.
 * segs_dev: n_segs (src offset, raw start) int64 pairs -- the segment starting at R[raw start] lies at
 *   src_dev + src offset and runs to the next segment's raw start (the frame's last one to |R|); a frame's first raw
 *   start is 0.
 * descs_dev: n descriptors of USDU_PNG_DESC_WORDS int64: first segment, segment count, H, W, C (1 grey, 2 grey+alpha,
 *   3 RGB, 4 RGBA), byte offset of the frame's [H, W, 3] u8 output in dst_dev, 0, 0.
 * The rows are un-filtered (None / Sub / Up / Avg / Paeth) and converted as PIL's convert("RGB"): grey replicated,
 * alpha dropped.  max_row_bytes >= every frame's W*C and <= USDU_PNG_MAX_ROW_BYTES (16,384 px, ComfyUI's
 * MAX_RESOLUTION, at 4 channels).  Shared memory holds a ring of usdu_png_decode_warps(max_row_bytes) rows, one per
 * warp of the CTA: min(16, opt-in shared memory per block / max_row_bytes), 3 at the limit on an H100.
 * usdu_png_decode_warps returns that depth for the current device, or a negative usdu_status. */
#define USDU_PNG_DESC_WORDS 8
#define USDU_PNG_MAX_ROW_BYTES 65536
int usdu_png_decode_u8(const uint8_t* src_dev, const int64_t* segs_dev, int64_t n_segs, const int64_t* descs_dev,
                       int n, int max_row_bytes, uint8_t* dst_dev, void* stream);
int usdu_png_decode_warps(int max_row_bytes);

/* The same decode for every other PNG PIL's open().convert("RGB") opens: colour type 0 at 1/2/4/8/16 bits, 2 at 8/16,
 * 3 (palette) at 1/2/4/8, 4 and 6 at 8/16, interlaced (Adam7) or not.  The host inflates each file's zlib stream
 * (http_master.parse_png_general) and uploads the filtered stream R whole; a frame is one pass, or Adam7's seven
 * (the empty ones left out), each decoded by one CTA of the launch.
 * descs_dev: n pass descriptors of USDU_PNG_GENERAL_DESC_WORDS int64: offset in src_dev of the pass's R (per row a
 *   filter byte 0..4, then ceil(w * depth * C / 8) bytes), pass width w >= 1 and height h >= 1, x0, y0, dx, dy (pixel
 *   (i, j) of the pass is pixel (y0 + i*dy, x0 + j*dx) of the frame; 0, 0, 1, 1 without interlace), the frame's width,
 *   colour type, bit depth, byte offset of the frame's [H, W, 3] u8 output in dst_dev, offset in src_dev of a
 *   768-byte RGB palette (colour type 3: the PLTE's entries, zeros after them), then 0s.
 * The rows are un-filtered on PNG filter units of max(1, depth * C / 8) bytes and converted as PIL 12's
 * convert("RGB"): 1/2/4-bit grey times 255/85/17, 16-bit grey min(v, 255), other 16-bit samples their high byte,
 * palette indices through the palette (tRNS ignored), grey replicated, alpha dropped.  max_row_bytes >= every pass's
 * filtered row bytes and <= USDU_PNG_MAX_ROW_BYTES; the ring depth is usdu_png_decode_warps(max_row_bytes). */
#define USDU_PNG_GENERAL_DESC_WORDS 16
int usdu_png_decode_general_u8(const uint8_t* src_dev, const int64_t* descs_dev, int n, int max_row_bytes,
                               uint8_t* dst_dev, void* stream);

/* Baseline JPEGs at the masters' routes, decoded as PIL's open().convert("RGB") with libjpeg-turbo's defaults (islow
 * IDCT, fancy upsampling, table-driven YCbCr->RGB).  The entropy decode is serial and runs on the host
 * (csrc/usdu_jpeg.cpp); dequantisation, IDCT, upsampling and colour conversion run on the device.
 * Taken: SOF0/SOF1, 8-bit, one scan of every component, 1 component, or 3 with the first at h, v in {1, 2} and the
 * others 1x1; sides up to 65,500 (libjpeg's JPEG_MAX_DIMENSION); any DQT/DHT tables, DRI with RST0..7 in sequence,
 * APPn/COM skipped, except the APPn segments PIL's Python header parse raises on (short "JFIF" APP0, "Adobe" APP14 and
 * "ICC_PROFILE" APP2, a cut "Photoshop 3.0" 8BIM resource) and "MPF" APP2 (an MPO).  Everything else, and every file
 * whose markers, Huffman codes, MCU count, restart markers or EOI are not exactly right, fails with USDU_ERR_INVALID
 * and the reason in usdu_last_error (also where libjpeg would only warn).
 * usdu_jpeg_parse: data[n] (host) -> info (USDU_JPEG_INFO_WORDS int64, the USDU_JI_* words) and quant (3 * 64 int32:
 *   each component's quantisation table in natural order, zeros for absent components).
 * usdu_jpeg_decode_coefs: the Huffman decode of the same file into coefs (host, n_words = 64 * info[USDU_JI_BLOCKS]
 *   int16): per component in order, a raster of 8x8 blocks over the MCU-padded component (bw x bh blocks, bw = MCUX *
 *   h, bh = MCUY * v, h = v = 1 for components after the first and for a 1-component file), each block's 64
 *   coefficients in natural (row-major) order, not dequantised. */
#define USDU_JPEG_INFO_WORDS 16
#define USDU_JI_W 0
#define USDU_JI_H 1
#define USDU_JI_COMPONENTS 2 /* 1 or 3 */
#define USDU_JI_H0 3         /* sampling of the first component (1 for a 1-component file) */
#define USDU_JI_V0 4
#define USDU_JI_COLOUR 5     /* USDU_JPEG_GREY, _YCC or _RGB, as libjpeg's default_decompress_parms decides */
#define USDU_JI_RESTART 6    /* restart interval in MCUs, 0 without DRI */
#define USDU_JI_MCUX 7       /* MCUs across and down */
#define USDU_JI_MCUY 8
#define USDU_JI_BLOCKS 9     /* coefficient blocks of all components */
#define USDU_JI_SCAN 10      /* offset of the first entropy-coded byte */
#define USDU_JPEG_GREY 0
#define USDU_JPEG_YCC 1
#define USDU_JPEG_RGB 2
int usdu_jpeg_parse(const uint8_t* data, int64_t n, int64_t* info, int32_t* quant);
int usdu_jpeg_decode_coefs(const uint8_t* data, int64_t n, int16_t* coefs, int64_t n_words);

/* usdu_jpeg_decode_u8: n frames, one launch of n_ctas CTAs; a CTA decodes one tile of a frame, one MCU row by
 * USDU_JPEG_TILE_W pixels, into the frame's [H, W, 3] u8 output.
 * descs_dev: n descriptors of USDU_JPEG_DESC_WORDS int64: offset in src_dev of the frame's coefficients (the layout of
 *   usdu_jpeg_decode_coefs, 16-byte aligned), offset in src_dev of its 3 * 64 int32 quantisation tables (4-byte
 *   aligned), W, H, components, h0, v0, colour, MCUX, MCUY (the USDU_JI_* words), byte offset of the frame's output in
 *   dst_dev, index of the frame's first CTA (0 for the first frame, then the running sum of MCUY * ceil(W /
 *   USDU_JPEG_TILE_W)), then 0s.  n_ctas is the sum over all frames.
 * The stages restate libjpeg-turbo's: dequantisation and the islow IDCT as its x86 SIMD code computes them (16-bit
 * dequantised coefficients, its 16-bit sums and saturating packs, which equal jidctint.c's results wherever no
 * intermediate leaves 16 bits); h2v1, h1v2 and h2v2 fancy upsampling with its rounding biases and edge rows and
 * columns (replication when a subsampled chroma row is at most 2 samples wide, as jdsample.c chooses); ycc_rgb_convert's
 * fixed-point tables, or no conversion for RGB; a grey frame replicated into the 3 channels. */
#define USDU_JPEG_DESC_WORDS 16
#define USDU_JPEG_TILE_W 128
int usdu_jpeg_decode_u8(const uint8_t* src_dev, const int64_t* descs_dev, int n, int64_t n_ctas, uint8_t* dst_dev,
                        void* stream);

/* HTTP tile worker transport (upscale/worker_comms.py:30-34): each u8 RGB frame [H, W, 3] as the PNG Pillow writes with
 * compress_level=0, byte for byte.  At level 0 Pillow's file is a framing that depends on the shape alone, filled with
 * the filtered stream R and the checksums.  R is per row one filter byte and the row filtered with it (|R| = H*(1 + 3W));
 * the kernels choose each row's filter as Pillow does without `optimize`: for None (0), Up (2), Sub (1), Paeth (4) in
 * that order, the sum over the filtered bytes v of min(v, 256 - v), with the previous RAW row above (zeros above the
 * first); the first candidate with the smallest sum.  This library does not model zlib or Pillow's buffering: the
 * caller derives the framing from Pillow for the shape (one encoded probe) and passes it as a layout:
 *   template_dev: png_len bytes, a file of this shape (its stream bytes and checksums are overwritten);
 *   runs_dev: n_runs (file offset, stream offset, length) int64 triples, sorted by file offset: R[stream offset, + length)
 *     goes to file[file offset, + length);
 *   chunks_dev: n_chunks (file offset, data length) int64 pairs, sorted: every IDAT chunk, whose CRC-32 (over type and
 *     data) is recomputed; every file byte outside the chunks is copied from the template;
 *   adler_at (host): the 4 file offsets of the big-endian Adler-32 of R, most significant byte first.
 * The runs, the Adler bytes and the stored-block headers may fall anywhere in the chunks, split across two of them
 * included; runs and Adler bytes lie in chunk data and do not overlap.  src_dev = B contiguous u8 frames [H, W, 3];
 * scratch_dev (16-byte aligned) = B * (round_up(|R|, 16) + 8*H + 16) bytes; frame b's file goes to dst_dev + b *
 * png_len.  Three launches on `stream`, no host synchronisation.  USDU_ERR_INVALID unless C = 3, W*3 <=
 * USDU_PNG_MAX_ROW_BYTES, 0 <= B <= 65535, png_len > |R| and the Adler offsets lie in the file. */
int usdu_png_encode_u8(const uint8_t* src_dev, int B, int H, int W, int C, const uint8_t* template_dev, int64_t png_len,
                       const int64_t* runs_dev, int n_runs, const int64_t* chunks_dev, int n_chunks,
                       const int64_t* adler_at, uint8_t* scratch_dev, uint8_t* dst_dev, void* stream);

/* Collector master's assembly (nodes/collector.py:193-236 after api/job_routes.py:126-130): frame i of n, a u8 frame
 * of frame_elems bytes at frames_dev[i] (a device array of n device pointers), goes to dst + i * frame_elems as
 * k / 255.0f, bit-identical to usdu_unpack_tiles_f32.  dst (4-byte aligned) is device memory or pinned host memory
 * (cudaHostAlloc); the latter is written through its device alias, so one launch performs the conversion and the
 * device-to-host transfer. */
int usdu_gather_unpack_f32(const uint8_t* const* frames_dev, int n, int64_t frame_elems, float* dst, void* stream);

/* Collector master's job_complete checks (api/job_routes.py:104-139): the base64 text of a posted image decoded, and
 * the decoded PNG's O(bytes) checks, on the device; the host keeps the structural walk (http_collector.py).
 * usdu_b64_png_check: text (16-byte aligned; device or pinned host memory, read in place) holds n bytes, the image
 * field after its data-URL header; n < 2^31.  png_dev (device, 16-byte aligned) gets the decoded bytes and needs
 * 12 * ceil(n / 16) bytes.  table_dev (device) gets USDU_B64_TABLE_WORDS int64:
 *   head (USDU_B64_HEAD_WORDS): [0] 1 if a byte lies outside [A-Za-z0-9+/=]; [1] index of the first '=' (n if none);
 *     [2] index of the last other byte + 1 (0 if none); [3] decoded length m when Python's
 *     binascii.a2b_base64(text, strict_mode=True) (3.12) accepts the text, else -1 -- accepted exactly when [0] is 0,
 *     no other byte follows a '=' ([2] <= [1]), the text does not start with '=' and, with d = [1] data characters and
 *     p = n - d pads: d % 4 == 0, or d % 4 == 2 with p == 2, or d % 4 == 3 with p == 1; m = 3 * (d / 4) + (0, -, 1, 2)
 *     [d % 4]; the trailing bits of a short quad are ignored;
 *     [4] chunks recorded; [5] why the chunk walk stopped (USDU_B64_CHUNKS_*); [6] the first chunk's IHDR raw stream
 *     bytes H * (1 + W * C) (-1 unless it reads as IHDR of length 13, 8-bit, colour type 0/2/4/6, W * C <=
 *     USDU_PNG_MAX_ROW_BYTES); [7] the zlib header bytes CMF | FLG << 8 (-1 if the stream is shorter); [8] bytes of the
 *     IDAT stream; [9] stored blocks recorded; [10] why the block walk stopped (USDU_B64_BLOCKS_*); [11] the 4 bytes
 *     after the final block, big-endian (-1 if the stream is shorter); [12] Adler-32 of the stored blocks' data (-1
 *     unless the walk reached the final block); [13] the largest filter byte over the rows of [6] (-1 unless the blocks
 *     hold that many bytes); [14] data bytes of the recorded blocks; [15] stream position after the final block;
 *     [16] entry of the first IDAT chunk; [17] IDAT chunks;
 *   USDU_B64_MAX_CHUNKS chunk entries of 4 words: file offset, data length, type (big-endian), IDAT stream start (-1);
 *   USDU_B64_MAX_BLOCKS block entries of 4 words: stream offset of the block header, BFINAL/BTYPE byte | LEN << 8 |
 *     NLEN << 24, offset of its data in the concatenated data of the blocks, Adler partials (s1 | s2 << 32);
 *   the file's first min(m, USDU_B64_PREFIX_BYTES) bytes.
 * The chunk walk goes from byte 8 through consecutive chunk headers, as http_master.parse_png does, and stops after
 * the first chunk that is not IDAT following an IDAT, after an IEND before any IDAT, after a chunk whose length exceeds
 * 2^31 - 1 or which runs past the end, when the next header does not fit, or at the table's end.  When it stopped
 * after IDATs, the block walk follows the zlib stream of stored blocks through the IDAT chunks until the final block, a
 * compressed block, a LEN/NLEN mismatch, a block or header past the stream's end, or the table's end.  Four launches on
 * `stream`, no host synchronisation. */
#define USDU_B64_HEAD_WORDS 24
#define USDU_B64_MAX_CHUNKS 4096
#define USDU_B64_MAX_BLOCKS 4096
#define USDU_B64_PREFIX_BYTES 4096
#define USDU_B64_TABLE_WORDS \
    (USDU_B64_HEAD_WORDS + 4 * USDU_B64_MAX_CHUNKS + 4 * USDU_B64_MAX_BLOCKS + USDU_B64_PREFIX_BYTES / 8)
enum { USDU_B64_CHUNKS_NONE = 0, USDU_B64_CHUNKS_SHORT = 1, USDU_B64_CHUNKS_PAST_END = 2, USDU_B64_CHUNKS_AFTER_IDAT = 3,
       USDU_B64_CHUNKS_IEND = 4, USDU_B64_CHUNKS_FULL = 5 };
enum { USDU_B64_BLOCKS_NONE = 0, USDU_B64_BLOCKS_SHORT = 1, USDU_B64_BLOCKS_ZLIB = 2, USDU_B64_BLOCKS_COMPRESSED = 3,
       USDU_B64_BLOCKS_LEN = 4, USDU_B64_BLOCKS_FINAL = 5, USDU_B64_BLOCKS_FULL = 6 };
int usdu_b64_png_check(const char* text, int64_t n, uint8_t* png_dev, int64_t* table_dev, void* stream);

/* TEST DOUBLE, not part of the reference path: the deterministic T0 sampler stand-in used by the
 * parity tests and bench.py (BASELINE.md section 3) as one fused pass,
 * out[i] = clamp(tiles[i]*one_minus_d + noise_scaled[i % frame], 0, 1), each step rounded. */
int usdu_t0_denoise(const float* tiles_dev, const float* noise_scaled_dev, float* out_dev, int64_t n,
                    int64_t frame, float one_minus_d, void* stream);

/* Feather templates: n_specs masks into mask_pool_dev.  scratch_dev needs
 * usdu_mask_scratch_bytes(specs, n) bytes. */
int64_t usdu_mask_scratch_bytes(const int32_t* specs_host, int n_specs);
int usdu_build_feather_masks(const int32_t* specs_host, int n_specs, uint8_t* mask_pool_dev,
                             uint8_t* scratch_dev, void* stream);

/* Tile crop + LANCZOS resize: canvas u8 -> fp32 tiles (values k/255).
 * grid = n_items x B blocks.  out_dev holds [B][PH][PW][3] fp32 per tile at the item's
 * out offset.  patch_w x patch_h (pixels) is the largest input patch any item reads (the
 * planner knows it from the resample tables); it sizes the shared-memory staging. */
int usdu_tile_crop_resize(const uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                          const int32_t* tiles_dev, const int32_t* tabs_dev,
                          const int32_t* items_dev, int n_items, int patch_w, int patch_h,
                          float* out_dev, int flags, void* stream);

/* The same crop straight from the fp32 IMAGE [B][H][W][3] (tensor-core job records only, W % 4 == 0): the truncating
 * cast of utils/image.py:8-10 happens while the window is staged, the tiles are bit-identical to cropping the
 * quantised canvas.  For participants whose tiles never overlap (a conflict-free static partition: every crop of
 * upscale/modes/static.py:242-280 then sees the ORIGINAL image), which therefore never need the quantised canvas. */
int usdu_tile_crop_resize_f32(const float* image_dev, int B, int H, int W, const int32_t* tabs_dev,
                              const int32_t* items_dev, int n_items, int patch_w, int patch_h,
                              float* out_dev, int flags, void* stream);

/* Seam blend: for every item (canvas block) apply its cover list in order:
 * quantise (fp32 source) -> LANCZOS back to the crop size -> integer alpha composite
 * with the tile's feather template, in place on the canvas.
 * src_is_u8 = 0: src_dev is fp32 sampler output in [0,1]; 1: src_dev is u8 (already Q1).
 * patch_w x patch_h: largest processed-tile patch any (item, cover entry) reads.
 * Tiles whose crop windows overlap must not be blended by different items of one launch
 * unless they appear in the same item's cover list (items own disjoint canvas blocks, so
 * any cover list is race-free; ORDER across overlapping tiles is the cover-list order). */
int usdu_tile_blend(uint8_t* canvas_dev, int B, int H, int W, int64_t pitch,
                    const int32_t* tiles_dev, const int32_t* tabs_dev,
                    const uint8_t* mask_pool_dev, const int32_t* items_dev, int n_items,
                    const int32_t* cover_dev, int patch_w, int patch_h, const void* src_dev,
                    int src_is_u8, int flags, void* stream);

/* ---- one-channel u8 planes: per-tile conditioning masks (utils/usdu_utils.py:415-442) ---------
 * Window of a separable 8bpc resize of n planes src[n][src_h][src_w] (Image.resize semantics:
 * horizontal pass first, u8 intermediate, then vertical): dst[p][j][i] = resized[p][oy+j][ox+i]
 * for j < oh, i < ow.  tab_h_dev / tab_v_dev are tables from usdu_build_filter_table for
 * (src_w -> full output width) / (src_h -> full output height), or NULL when that axis keeps its
 * size (Pillow skips the pass).  Only the window is computed, which gives exactly the
 * pixels of "resize the whole mask to the canvas size, then crop" (crop_mask).
 * The intermediate holds input rows mid_y0 .. mid_y0+mid_rows-1 (what the vertical taps of output
 * rows oy..oy+oh-1 read: usdu_table_input_span on the HOST copy of the vertical table), layout
 * [n][mid_rows][(ow+3)&~3] bytes; unused (may be NULL) unless both passes run. */
int usdu_table_input_span(const int32_t* table_host, int first_out, int n_out, int* first_in, int* n_in);
int usdu_plane_resample_u8(const uint8_t* src_dev, int n, int src_h, int src_w, int64_t src_pitch, int64_t src_plane,
                           const int32_t* tab_h_dev, int ox, int ow, const int32_t* tab_v_dev, int oy, int oh,
                           int mid_y0, int mid_rows, uint8_t* mid_dev,
                           uint8_t* dst_dev, int64_t dst_pitch, int64_t dst_plane, void* stream);
/* pad_image2(img, hp, hp, vp, vp, fill=True) (utils/usdu_utils.py:169-203) on n planes [h][w] ->
 * [h+2vp][w+2hp]: left/right strips = edge column rows 1+row_index[y], then top/bottom strips =
 * edge row columns 1+col_index[x] (they overwrite the corners).  row_index_dev = usdu_nearest_index
 * (h-2 -> h+2vp), col_index_dev = usdu_nearest_index(w-2 -> w+2hp); either may be NULL when its
 * pad is 0. */
int usdu_plane_pad_fill_u8(const uint8_t* src_dev, int n, int h, int w, int64_t src_pitch, int64_t src_plane,
                           int hp, int vp, const int32_t* row_index_dev, const int32_t* col_index_dev,
                           uint8_t* dst_dev, int64_t dst_pitch, int64_t dst_plane, void* stream);

/* ---- host-side planner (no device needed) -------------------------------------------------
 * A plan is one job geometry: usdu_plan_create(W, H, tile_width, tile_height, padding, mask_blur,
 * uniform) applies round_to_multiple (ties to even, upscale/tile_ops.py:14-16), calculate_tiles
 * (:18-32), the crop window and expand_crop (utils/usdu_utils.py:49-112) and, for uniform = 0,
 * the multiple-of-8 target size; then it builds the table pool (tables of every crop and blend
 * axis, each followed by its tensor-core fragment section while the plan qualifies for the
 * tensor-core kernels; every section starts at a multiple of 4 int32), the feather-mask specs,
 * the tile descriptors and the overlap graph.  A tile size that rounds to zero, an empty canvas
 * and feather templates of 2 GiB or more are rejected with USDU_ERR_INVALID.  The plan is
 * immutable; the query calls copy into caller-allocated arrays sized from usdu_plan_info. */
typedef struct usdu_plan usdu_plan;
int usdu_plan_create(int W, int H, int tile_width, int tile_height, int padding, int mask_blur, int uniform,
                     usdu_plan** plan);
int usdu_plan_destroy(usdu_plan* plan);
#define USDU_PLAN_INFO_WORDS 16    /* int64 words of usdu_plan_info */
#define USDU_PI_TW 0               /* tile size after round_to_multiple */
#define USDU_PI_TH 1
#define USDU_PI_TILES 2            /* tile positions (row-major grid) */
#define USDU_PI_TAB_WORDS 3        /* int32 words of the table pool */
#define USDU_PI_TABLES 4           /* resample tables in the pool (rows of usdu_plan_table_index) */
#define USDU_PI_MASK_CLASSES 5     /* feather-mask specs (rows of usdu_plan_mask_specs) */
#define USDU_PI_MASK_POOL_BYTES 6  /* bytes of the mask pool usdu_build_feather_masks fills */
#define USDU_PI_FAST 7             /* 1: every table has packed rows (integer-pipe kernels usable) */
#define USDU_PI_MMA 8              /* 1: ... and tensor-core fragments, windows on 4-pixel columns */
#define USDU_PI_PATH 9             /* best kernel path: 0 generic, 1 integer-pipe (USDU_FLAG_FAST), 2 tensor-core */
#define USDU_PI_NEIGHBOR_WORDS 10  /* entries of usdu_plan_neighbors' list */
int usdu_plan_info(const usdu_plan* plan, int64_t* info);
/* per tile USDU_PLAN_TILE_WORDS int32: {x, y} grid origin, {x1, y1} crop window origin, {ew, eh} window size,
 * {pw, ph} processing size, {bx2, by2} exclusive far corner of the clipped mask rectangle (which starts at x, y),
 * feather-mask class, 0 */
#define USDU_PLAN_TILE_WORDS 12
int usdu_plan_tiles(const usdu_plan* plan, int32_t* tiles);
/* tiles x USDU_TILE_WORDS descriptors (upload for the tile kernels) */
int usdu_plan_tile_desc(const usdu_plan* plan, int32_t* desc);
/* the table pool, USDU_PI_TAB_WORDS int32 (upload for the tile kernels) */
int usdu_plan_tables(const usdu_plan* plan, int32_t* pool);
/* per table USDU_PLAN_TABLE_WORDS int32: {in size, out size, pool offset, pool index of packed row 0, pool index of
 * the fragment section (-1 = none), k-steps, staged taps of the integer-pipe kernels, taps the job records carry} */
#define USDU_PLAN_TABLE_WORDS 8
int usdu_plan_table_index(const usdu_plan* plan, int32_t* index);
/* USDU_PI_MASK_CLASSES x USDU_MASK_WORDS specs for usdu_mask_scratch_bytes / usdu_build_feather_masks */
int usdu_plan_mask_specs(const usdu_plan* plan, int32_t* specs);
/* tiles whose crop windows intersect: tile i's list is list[first[i] .. first[i+1]); first has tiles + 1 entries */
int usdu_plan_neighbors(const usdu_plan* plan, int32_t* first, int32_t* list);
/* Level schedule of the tiles order[0..n) (distinct ids) under progressive semantics (upscale/modes/single_gpu.py:40-64):
 * wave[i] = level of order[i]; tiles of one level have disjoint windows and run as one crop / sampler / blend step,
 * levels in ascending order.  Returns the number of levels, or a negative usdu_status. */
int usdu_plan_waves(const usdu_plan* plan, const int32_t* order, int n, int32_t* wave);

/* Work lists: one kernel launch each, built for
 *   path: 0 generic kernels, 1 integer-pipe (USDU_FLAG_FAST), 2 tensor-core (USDU_FLAG_MMA); lowered to what the plan
 *         supports (USDU_WL_PATH tells which);
 *   sm_count: SMs of the block-height model, 0 = query the current device (132 when there is none);
 *   mma_block_rows: tensor-core block height to force (16 or 32), 0 = the model's choice.
 * Crop: the tiles' [B][PH][PW][3] fp32 outputs are packed in list order (usdu_worklist_slots: element offset per tile,
 * USDU_WL_TOTAL elements in all).  Blend: src_offsets[i] = element offset of tile_ids[i]'s processed block in the
 * source, src_bytes = 4 (fp32) or 1 (u8); the list order is the blend order.  part_n > 0 restricts the launch to the
 * part_i-th of part_n horizontal slabs of canvas block rows (USDU_WL_ROW0 / _ROW1).
 * Launch: items = usdu_worklist_items, grid = USDU_WL_GRID, flags = USDU_WL_FLAGS, patch = USDU_WL_PATCH_W / _H, and for
 * the generic blend cover_dev = usdu_worklist_cover. */
typedef struct usdu_worklist usdu_worklist;
int usdu_plan_crop_worklist(const usdu_plan* plan, const int32_t* tile_ids, int n, int B, int path, int sm_count,
                            int mma_block_rows, usdu_worklist** wl);
int usdu_plan_blend_worklist(const usdu_plan* plan, const int32_t* tile_ids, const int64_t* src_offsets, int n,
                             int src_bytes, int B, int path, int part_i, int part_n, int sm_count,
                             int mma_block_rows, usdu_worklist** wl);
int usdu_worklist_destroy(usdu_worklist* wl);
/* Work lists of one dependency wave of the split schedule, which runs the crop jobs that read no pixel the previous
 * wave's blend changes ("early") beside that wave's sampler and blend, and the rest ("late") on the chain
 * crop -> sampler -> blend.  prev_ids[0..n_prev) = the previous wave (n_prev = 0: the first wave, every job is late);
 * src_offsets as for the blend (fp32 sources).  The tensor-core path sizes each list for its role: late jobs in short
 * blocks (16 rows), early jobs in the tallest the crop's 48-row box allows (usdu_plan_crop_worklist with 32 rows), a
 * tall job that reads pixels of the previous wave's feather supports falls back to its short jobs, each late or early
 * by its own rectangle; the blend block height minimises rounds of resident CTAs (usdu_mma_resident_ctas) times the
 * rows a CTA stages and writes.  The integer-pipe path splits one list built as usdu_plan_crop_worklist does.  Early
 * and late cover every crop output element exactly once and share the output layout (usdu_worklist_slots of either);
 * `early` may have no items.  path >= 1 (job records). */
int usdu_plan_split_worklists(const usdu_plan* plan, const int32_t* tile_ids, const int64_t* src_offsets, int n,
                              const int32_t* prev_ids, int n_prev, int B, int path, int sm_count, usdu_worklist** late,
                              usdu_worklist** early, usdu_worklist** blend);
#define USDU_WL_INFO_WORDS 16      /* int64 words of usdu_worklist_info */
#define USDU_WL_ITEMS 0            /* rows of usdu_worklist_items */
#define USDU_WL_ITEM_WORDS 1       /* int32 per row: USDU_JOB_WORDS, USDU_CROP_ITEM_WORDS or USDU_BLEND_ITEM_WORDS */
#define USDU_WL_COVER 2            /* rows (USDU_COVER_WORDS) of usdu_worklist_cover (generic blend) */
#define USDU_WL_PATCH_W 3
#define USDU_WL_PATCH_H 4
#define USDU_WL_ALGO_BYTES 5       /* algorithmic HBM bytes of the launch per frame */
#define USDU_WL_N_LAUNCH 6         /* blend job records: chain heads (the grid); -1 = one CTA per row */
#define USDU_WL_BLOCK_ROWS 7
#define USDU_WL_BLOCK_COLS 8
#define USDU_WL_ROW0 9             /* part_n > 0: canvas rows [ROW0, ROW1) of the slab; else -1 */
#define USDU_WL_ROW1 10
#define USDU_WL_PATH 11
#define USDU_WL_KS2 12             /* tensor-core records with a two-k-step axis (set USDU_FLAG_MMA_KS2) */
#define USDU_WL_TOTAL 13           /* crop: fp32 elements of the packed output */
#define USDU_WL_FLAGS 14           /* the `flags` argument of the launch */
#define USDU_WL_GRID 15            /* the `n_items` argument of the launch */
int usdu_worklist_info(const usdu_worklist* wl, int64_t* info);
int usdu_worklist_items(const usdu_worklist* wl, int32_t* items);
int usdu_worklist_cover(const usdu_worklist* wl, int32_t* cover);
int usdu_worklist_slots(const usdu_worklist* wl, int64_t* offsets);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* USDU_B200_H */
