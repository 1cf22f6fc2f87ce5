/* blinky_b200 — C ABI of the H100-native Blinky lens-warp path.
 *
 * This is the thin boundary a C host (TyrQuake's fisheye seams, or a headless
 * harness) calls into.  It replaces, for the lens-warp path only, what the
 * reference keeps inside one statically linked translation unit,
 * the reference's engine/NQ/fisheye.c (public surface: engine/include/fisheye.h:4-9).
 * Plain pointers and sizes only; no C++ or torch types.
 *
 * Mapping to the reference (file:line are in the reference's engine/NQ/fisheye.c):
 *
 *   blinky_create / blinky_destroy      F_Init :642-676 / F_Shutdown :678-681 (state + Lua VM)
 *   blinky_set_palette                  create_palmap :857-908 (from host_basepal)
 *   blinky_command                      the console commands registered at :651-665
 *                                       (fisheye, f_lens, f_globe, f_fov, f_vfov, f_cover,
 *                                        f_contain, f_rubix, f_rubixgrid, f_help)
 *   blinky_load_lens[_source]           cmd_lens :1061-1103 / LUA_load_lens :1659-1750
 *   blinky_load_globe[_source]          cmd_globe :1138-1161 / LUA_load_globe :1752-1875
 *   blinky_set_zoom                     cmd_fov/vfov/cover/contain :955-965, :1032-1058
 *   blinky_set_rubix / _rubixgrid       cmd_rubix :933-937 / cmd_rubixgrid :939-953
 *   blinky_build_lensmap                the rebuild branch of F_RenderView :730-743 ->
 *                                       create_lensmap :2367-2397 (inverse :2084-2124,
 *                                       forward :2126-2338), one shot instead of time-sliced
 *   blinky_warp_*                       render_lensmap :2406-2424 (THE hot loop) on the GPU
 *   blinky_write_config                 F_WriteConfig :683-696
 *   blinky_save_globe                   save_globe / WritePCXplate :1396-1486
 *
 * Conventions: every function returns BLINKY_OK (0) or a negative BLINKY_E_*
 * code; blinky_last_error() has the message.  Nothing ever calls exit() (the
 * reference does on OOM, :723-726).  A context is single-threaded: calls on
 * one context must be serialised by the caller; use one context per GPU.
 */
#ifndef BLINKY_B200_H
#define BLINKY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BLINKY_MAX_PLATES 6 /* MAX_PLATES, fisheye.c:352 */

enum {
    BLINKY_OK = 0,
    BLINKY_E_INVALID = -1,   /* bad argument / call order */
    BLINKY_E_SCRIPT = -2,    /* lens or globe script failed to load or run */
    BLINKY_E_ZOOM = -3,      /* calc_zoom failed (fisheye.c:1293-1386) */
    BLINKY_E_NODEVICE = -4,  /* context has no GPU (created with device < 0) */
    BLINKY_E_CUDA = -5,      /* CUDA runtime error */
    BLINKY_E_NOMEM = -6,
    BLINKY_E_STATE = -7      /* lens/globe invalid or lensmap not built */
};

/* zoom.type, fisheye.c:457 */
enum { BLINKY_ZOOM_NONE = 0, BLINKY_ZOOM_FOV = 1, BLINKY_ZOOM_VFOV = 2, BLINKY_ZOOM_COVER = 3, BLINKY_ZOOM_CONTAIN = 4 };
/* lens.map_type, fisheye.c:391 */
enum { BLINKY_MAP_NONE = 0, BLINKY_MAP_INVERSE = 1, BLINKY_MAP_FORWARD = 2 };

/* Packed device lensmap entry (one per screen pixel, 4 bytes):
 *   bit 31      valid (reference: lens.pixels[i] != NULL)
 *   bits 28-30  rubix tint index 0..5, or 7 = none (reference: pixel_tints[i], 255 = none)
 *   bits 0-27   texel offset into the globe: plate*ps*ps + py*ps + px (GLOBEPIXEL, :349) */
#define BLINKY_LM_VALID 0x80000000u
#define BLINKY_LM_TINT_SHIFT 28
#define BLINKY_LM_TINT_NONE 7u
#define BLINKY_LM_INDEX_MASK 0x0FFFFFFFu

/* kernel variants (blinky_set_kernel) */
enum {
    BLINKY_KERNEL_AUTO = 0,    /* pick per lensmap from the tile classification */
    BLINKY_KERNEL_GATHER = 1,  /* direct global gather, vectorised coalesced stores */
    BLINKY_KERNEL_TMA = 2      /* ring kernel: TMA-staged face tiles in shared memory where tiles are coherent (what AUTO picks) */
};

typedef struct blinky_ctx blinky_ctx;
typedef void (*blinky_print_fn)(const char *text, void *user);   /* Con_Printf sink */
typedef void (*blinky_exec_fn)(const char *command, void *user); /* Cmd_ExecuteString hook for `onload` */

/* ---- lifecycle --------------------------------------------------------- */
/* device >= 0: CUDA device ordinal.  device < 0: host-only context (lensmap
 * build, palette, console surface work; every blinky_warp_* call fails with
 * BLINKY_E_NODEVICE — there is no CPU fallback for the hot path). */
int blinky_create(int device, blinky_ctx **out);
void blinky_destroy(blinky_ctx *ctx);
const char *blinky_last_error(blinky_ctx *ctx);
const char *blinky_version(void);

/* messages the reference sends to Con_Printf; default sink keeps them in a log */
void blinky_set_print_callback(blinky_ctx *ctx, blinky_print_fn fn, void *user);
/* where a lens script's `onload` command goes (fisheye.c:1087-1095); default:
 * this library's own blinky_command */
void blinky_set_exec_callback(blinky_ctx *ctx, blinky_exec_fn fn, void *user);
const char *blinky_log(blinky_ctx *ctx);
void blinky_log_clear(blinky_ctx *ctx);

/* ---- configuration (host side) ----------------------------------------- */
/* directory that contains lua-scripts/{globes,lenses}/ (com_basedir, :1666) */
int blinky_set_basedir(blinky_ctx *ctx, const char *basedir);
/* host_basepal: 256 RGB triplets -> six rubix tint LUTs */
int blinky_set_palette(blinky_ctx *ctx, const uint8_t palette[768]);
/* executes one console command line, e.g. "f_lens panini", "f_fov 170",
 * "f_globe cube", "f_rubix", "f_rubixgrid 10 4 1", "f_cover", "fisheye 1" */
int blinky_command(blinky_ctx *ctx, const char *text);

int blinky_load_globe(blinky_ctx *ctx, const char *name);
int blinky_load_lens(blinky_ctx *ctx, const char *name);
/* same, from source text instead of <basedir>/lua-scripts/...; the text is
 * kept and re-run on every rebuild exactly like the file would be (:737) */
int blinky_load_globe_source(blinky_ctx *ctx, const char *name, const char *lua_source);
int blinky_load_lens_source(blinky_ctx *ctx, const char *name, const char *lua_source);
int blinky_set_zoom(blinky_ctx *ctx, int zoom_type, int fov_degrees);
int blinky_set_rubix(blinky_ctx *ctx, int enabled);
int blinky_set_rubixgrid(blinky_ctx *ctx, int numcells, double cell_size, double pad_size);

/* ---- lensmap build ("InitLensMap") -------------------------------------- */
/* Builds the lensmap for a width x height view and square plates of
 * `platesize` pixels (the reference forces platesize = min(w,h), :707; pass
 * platesize <= 0 for that behaviour).
 *   threads == 1  the lens script is interpreted in the reference's own order on one
 *                 script state;
 *   threads  > 1  rows are split over that many cloned script states (requires
 *                 lens_inverse to be a pure function of x,y — true for every shipped lens);
 *   threads  < 0  as above with every CPU the process may use;
 *   threads == 0  GPU build: the lens function is translated to CUDA, compiled for sm_90a
 *                 with NVRTC and evaluated by one kernel — lens_inverse for every screen
 *                 pixel, or, for forward-only lenses, lens_forward for every plate grid point
 *                 followed by the quad rasterisation in the reference's writer order.
 *                 Results that are not provably the host's (error bounds on every libm call)
 *                 are re-evaluated by the interpreter, so the map is the same as the host
 *                 build's.  Lenses outside the translatable subset, globes with a
 *                 globe_plate script and CPU-only contexts fall back to threads < 0.
 * blinky_build_info() says which way the last build went.
 * On a GPU context the packed map, tile table and tint LUTs are uploaded too. */
int blinky_build_lensmap(blinky_ctx *ctx, int width, int height, int platesize, int threads);
/* e.g. "device: 12 of 8294400 pixels re-evaluated by the interpreter; NVRTC 310 ms, kernel 1.9 ms"
 * or "host (line 22: nil values are not supported here)" */
const char *blinky_build_info(blinky_ctx *ctx);
/* Translate + NVRTC-compile the current lens_inverse (forward = 0) or lens_forward (forward = 1)
 * kernel without running it (works without a GPU). */
int blinky_compile_lens(blinky_ctx *ctx, int forward, size_t *cubin_bytes);
/* 1 if a lens/globe/zoom/rubixgrid/size change since the last build requires a rebuild (:730) */
int blinky_needs_rebuild(blinky_ctx *ctx, int width, int height, int platesize);

/* ---- state queries ------------------------------------------------------ */
int blinky_fisheye_enabled(blinky_ctx *ctx);          /* fisheye_enabled, :293 */
int blinky_lens_valid(blinky_ctx *ctx);
int blinky_globe_valid(blinky_ctx *ctx);
const char *blinky_lens_name(blinky_ctx *ctx);
const char *blinky_globe_name(blinky_ctx *ctx);
const char *blinky_lens_onload(blinky_ctx *ctx);      /* "" when nil */
int blinky_map_type(blinky_ctx *ctx);
int blinky_zoom_type(blinky_ctx *ctx);
int blinky_zoom_fov(blinky_ctx *ctx);
int blinky_max_fov(blinky_ctx *ctx);
int blinky_max_vfov(blinky_ctx *ctx);
double blinky_lens_width(blinky_ctx *ctx);
double blinky_lens_height(blinky_ctx *ctx);
double blinky_scale(blinky_ctx *ctx);                 /* lens.scale after a build */
int blinky_rubix_enabled(blinky_ctx *ctx);
int blinky_numplates(blinky_ctx *ctx);
int blinky_platesize(blinky_ctx *ctx);
int blinky_width(blinky_ctx *ctx);
int blinky_height(blinky_ctx *ctx);
/* per plate: forward[3] right[3] up[3] fov dist as 11 floats; returns numplates */
int blinky_get_plates(blinky_ctx *ctx, float *out, int max_plates);
/* globe.plates[i].display after a build (:1976): which plates the lens uses */
int blinky_get_display(blinky_ctx *ctx, int out[BLINKY_MAX_PLATES]);
double blinky_plate_fov(blinky_ctx *ctx, int plate);  /* radians: fisheye_plate_fov source, :769 */
/* six 256-entry tint LUTs (globe.plates[i].palette) */
int blinky_get_palmaps(blinky_ctx *ctx, uint8_t out[BLINKY_MAX_PLATES * 256]);
/* lensmap in the reference's terms: idx = pointer - globe.pixels or -1; tint 0..5 or 255 */
int blinky_get_lensmap(blinky_ctx *ctx, int32_t *idx, uint8_t *tint);
/* the packed 32-bit entries the kernels read */
int blinky_get_lensmap_packed(blinky_ctx *ctx, uint32_t *out);
int64_t blinky_mapped_pixels(blinky_ctx *ctx);        /* M in the 5*W*H + M byte count */
/* direct script probes (LUAtoC_lens_inverse/_forward before float narrowing):
 * return 1 = values, 0 = nil, negative = error */
int blinky_lens_inverse(blinky_ctx *ctx, double x, double y, double ray_out[3]);
int blinky_lens_forward(blinky_ctx *ctx, double rx, double ry, double rz, double *x, double *y);
/* The current lens function translated to C++ / CUDA C++ — what the device lensmap builder
 * compiles (SURVEY 8f).  flavour: bit 0 = CUDA (else plain C++), bit 1 = lens_forward (else
 * lens_inverse), bit 2 = append the fixed kernel (the per-pixel / per-grid-point tail) — with
 * bits 0 and 2 this is exactly what NVRTC is given.  Returns the bytes needed (excluding NUL), or BLINKY_E_SCRIPT when the lens is
 * outside the translatable subset (reason: blinky_last_error). */
int blinky_lens_source(blinky_ctx *ctx, int flavour, char *buf, size_t bufsize);
/* F_WriteConfig text; returns bytes needed (excluding NUL) */
int blinky_write_config(blinky_ctx *ctx, char *buf, size_t bufsize);

/* f_saveglobe (fisheye.c:1120-1136, 1396-1486): the console command arms a request;
 * the frame driver asks blinky_saveglobe_pending() after rendering the plates and then
 * passes them to blinky_save_globe(), which writes <directory>/<name><i>.pcx per plate
 * (the reference's COM_WriteFile target is com_gamedir) and prints "Wrote ...". */
int blinky_saveglobe_pending(blinky_ctx *ctx);
int blinky_save_globe(blinky_ctx *ctx, const uint8_t *faces_host, const char *directory);

/* ---- hot path ("RenderLensMap") — GPU only ------------------------------- */
int blinky_set_kernel(blinky_ctx *ctx, int kernel_variant);
/* Frame shown where the lens maps nothing (what Draw_TileClear left in
 * vid.buffer, :802).  [height][width] bytes, NULL = all zero.  Uploaded once. */
int blinky_set_background(blinky_ctx *ctx, const uint8_t *background_host);

/* Device-resident batch: d_faces -> d_out on `stream` (a cudaStream_t; NULL is
 * CUDA's default stream).  d_faces: nframes x [numplates][ps][ps]
 * bytes, frame stride face_stride bytes; d_out: nframes x [height][width]
 * bytes, stride out_stride.  Asynchronous.  One kernel launch per call. */
int blinky_warp_device(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out, size_t out_stride,
                       int nframes, void *stream);

/* End to end from HOST buffers: pinned-staged cudaMemcpyAsync of each frame's
 * displayed plates, the warp, and the copy back, software-pipelined over
 * internal streams.  faces_host: nframes x [numplates][ps][ps].  dst_host: nframes
 * screens of dst_rowbytes pitch; the view rectangle starts at (x0,y0) inside
 * each (scr_vrect, VBUFFER macro :634).  If keep_unmapped != 0 only mapped
 * pixels are written into dst (exact reference semantics, :2413); otherwise
 * unmapped pixels receive the background set above.  Synchronous. */
int blinky_warp_host(blinky_ctx *ctx, const uint8_t *faces_host, size_t face_stride, uint8_t *dst_host,
                     size_t dst_frame_stride, int dst_rowbytes, int x0, int y0, int nframes, int keep_unmapped);

/* bytes blinky_warp_host copies host->device per frame for the current lensmap: for
 * every plate the lens shows, the texel rectangle it samples */
int64_t blinky_upload_bytes_per_frame(blinky_ctx *ctx);

/* pinned host memory helpers for callers that want zero staging copies */
int blinky_alloc_pinned(blinky_ctx *ctx, size_t bytes, void **out);
int blinky_free_pinned(blinky_ctx *ctx, void *ptr);
int blinky_sync(blinky_ctx *ctx);

/* ---- peer memory: fused warp + gather over NVLink ------------------------------
 * The kernels write through whatever device-accessible pointer d_out is.  To fuse the
 * reference topology's final gather into the warp, rank 0 allocates the gather buffer,
 * exports it, every other rank (one process per GPU) opens it and passes
 * `peer_base + its frame offset` as d_out: finished pixels then travel to rank 0 as
 * NVLink stores issued by the warp kernel itself, no separate collective.
 * handle: 64 opaque bytes (cudaIpcMemHandle_t), moved between processes by the caller. */
int blinky_alloc_device(blinky_ctx *ctx, size_t bytes, void **out);
int blinky_free_device(blinky_ctx *ctx, void *ptr);
int blinky_ipc_export(blinky_ctx *ctx, void *device_ptr, unsigned char handle[64]);
int blinky_ipc_open(blinky_ctx *ctx, const unsigned char handle[64], void **peer_ptr);
int blinky_ipc_close(blinky_ctx *ctx, void *peer_ptr);

/* ---- sharded batches: frames over N GPUs, finished frames gathered on rank 0 -----------------
 * One process per GPU, one context per process.  A batch of total_frames independent frames is cut
 * into contiguous blocks (blinky_shard_range, sizes differ by at most one); every rank builds the same
 * lensmap and warps its own block; there is NO collective on the data path.  The reference topology's
 * last step — finished frames reach the one display (the reference writes vid.buffer,
 * engine/NQ/fisheye.c:802-803, 2406-2424) — is a gather to rank 0, done chunk by chunk so that the
 * transfer of chunk k overlaps the warp of chunk k+1 (a compute and a communication stream per rank).
 *   BLINKY_GATHER_NCCL        ncclSend / ncclRecv of finished chunks (NCCL only for the final gather)
 *   BLINKY_GATHER_PEER_COPY   copy engines push finished chunks into rank 0's buffer (CUDA-IPC peer memory over NVLink)
 *   BLINKY_GATHER_PEER_STORE  the warp kernels store straight into rank 0's buffer (fused warp + gather)
 * NCCL is loaded at run time (libnccl.so.2, or the path in BLINKY_NCCL_LIB); the 128-byte id made by
 * blinky_shard_unique_id on one rank is carried to the others by the caller (MPI, a file, torch.distributed ...).
 * Calls marked collective must be made by every rank. */
enum { BLINKY_GATHER_NCCL = 0, BLINKY_GATHER_PEER_COPY = 1, BLINKY_GATHER_PEER_STORE = 2 };
/* pure arithmetic (no context): frames [*first, *first + *count) belong to `rank` */
int blinky_shard_range(int total_frames, int rank, int world, int *first, int *count);
int blinky_shard_unique_id(unsigned char id[128]);
/* collective: joins the group (ncclCommInitRank) */
int blinky_shard_init(blinky_ctx *ctx, int rank, int world, const unsigned char id[128]);
/* collective: rank 0 allocates the gather buffer (total_frames x [height][width] bytes, frame f at
 * f*width*height) and shares it; *root_buffer is that device pointer on rank 0 and NULL elsewhere.
 * Needs a built lensmap.  The buffer lives until the next call or blinky_shard_close. */
int blinky_shard_buffer(blinky_ctx *ctx, int total_frames, void **root_buffer);
/* collective: d_faces = this rank's block of frames (device memory, frame stride face_stride).
 * Stream-ordered: the work starts after what `stream` holds and `stream` then waits for it; on rank 0
 * the gathered batch is complete when `stream` reaches that point. */
int blinky_shard_warp_gather(blinky_ctx *ctx, const void *d_faces, size_t face_stride, int total_frames, int mode,
                             int chunk_frames, void *stream);
int blinky_shard_sync(blinky_ctx *ctx);
int blinky_shard_close(blinky_ctx *ctx);

/* Fused 8-bit -> 32-bit palette expansion (engine/common/vid_sdl.c:539-546,
 * d_8to24table): same warp, output one uint32 per pixel.  table: 256 entries. */
int blinky_set_rgba_table(blinky_ctx *ctx, const uint32_t table[256]);
int blinky_warp_device_rgba(blinky_ctx *ctx, const void *d_faces, size_t face_stride, void *d_out_rgba,
                            size_t out_stride, int nframes, void *stream);

/* one-line description of how the current lensmap was tiled for the TMA kernel
 * (tile counts per class, staged bytes per pixel); "" before a build */
const char *blinky_plan_summary(blinky_ctx *ctx);
/* The tile plan the kernels read (DESIGN.md section 3): 16-byte tile descriptors
 * {u32 entry_offset; i16 box_x, box_y; u8 plate (bits 0-2) | tile tint << 3 (0-5, 7 = no pixel tinted),
 * type (0 empty, 1 box, 2 gather, 3 box fully mapped), box_w/16, box_h/8; u16 px, py} — the upper six bits of
 * `type` are the index of the box shape (one TMA descriptor per shape, at most 64) — ordered BOX tiles, GATHER
 * tiles, EMPTY tiles, and the entry blocks in the same order, fixed sizes: BOX 2176 bytes = [4][32 lanes][8]
 * uint16 {bit 15 valid, bits 0-13 offset inside the box} in the ring kernel's lane order (lane l, entry i ->
 * tile row (l>>3) + 4*(i>>2), column 4*(l&7) + (i&3)) followed by [32 lanes] uint32 tint flags (bit i: the
 * lane's pixel i carries the tile's tint; tiles whose tinted pixels disagree are GATHER tiles); GATHER 4096
 * bytes = [32][32] packed 32-bit lensmap entries.  Pass NULL buffers to query the sizes.  Works on CPU-only contexts;
 * the tests interpret the plan on the CPU to pin this layout (tests/test_tile_plan.py). */
int blinky_get_tile_plan(blinky_ctx *ctx, void *tiles_out, size_t tiles_cap, void *entries_out, size_t entries_cap, size_t *ntiles,
                         size_t *entry_bytes);
/* FNV-1a digest of the tile table + entry blocks planned on `threads` host threads (the plan
 * must not depend on the thread count; used by the tests) */
uint64_t blinky_plan_digest(blinky_ctx *ctx, int threads);
/* number of kernel launches issued by this context so far */
int64_t blinky_launch_count(blinky_ctx *ctx);
/* last warp kernel's name and launch geometry, for reports */
const char *blinky_last_kernel(blinky_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* BLINKY_B200_H */
