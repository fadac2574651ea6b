/* halide_b200_runtime.h — the C ABI boundary of the H100-native Halide apps library.
 *
 * This header re-declares (it does not copy) the binary layout a Halide AOT filter and its
 * harness agree on, so that `apps/<app>/process.cpp|filter.cpp|test.cpp` of the reference link
 * against libhalide_b200.so unchanged.  Every declaration cites the reference interface it
 * replaces; all paths are relative to /root/reference.
 *
 *   halide_buffer_t            src/runtime/HalideRuntime.h:1710-1737   (56 bytes, LP64)
 *   halide_dimension_t         src/runtime/HalideRuntime.h:1657-1685   (16 bytes)
 *   halide_type_t              src/runtime/HalideRuntime.h:521-545     (4 bytes: code, bits, reserved)
 *   halide_device_interface_t  src/runtime/HalideRuntime.h:875-899     (15 function pointers + impl)
 *   halide_error_code_t        src/runtime/HalideRuntime.h:1152-1357
 *   halide_filter_metadata_t   src/runtime/HalideRuntime.h:1937-1977
 *   halide_cuda_* entry points src/runtime/HalideRuntimeCuda.h:40-81
 *
 * If the reference's own HalideRuntime.h was included first (harness builds), the type
 * re-declarations below are skipped and only the function prototypes remain, so both headers
 * can coexist in one translation unit.
 */
#ifndef HALIDE_B200_RUNTIME_H
#define HALIDE_B200_RUNTIME_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef HALIDE_HALIDERUNTIME_H /* the reference header's include guard */
#define HALIDE_B200_OWNS_ABI_TYPES 1

/* Element type codes (HalideRuntime.h:492-503). */
enum {
    halide_type_int = 0,
    halide_type_uint = 1,
    halide_type_float = 2,
    halide_type_handle = 3,
    halide_type_bfloat = 4
};

/* 4-byte type word: code@0, bits@1, 16 reserved bits@2 (HalideRuntime.h:521-545). */
struct halide_type_t {
    uint8_t code;
    uint8_t bits;
    uint16_t reserved;
};

/* One dimension: coordinates [min, min+extent), stride in ELEMENTS (HalideRuntime.h:1657-1685). */
typedef struct halide_dimension_t {
    int32_t min, extent, stride;
    uint32_t flags;
} halide_dimension_t;

/* Dirty bits in halide_buffer_t::flags (HalideRuntime.h:1699-1702). */
enum {
    halide_buffer_flag_host_dirty = 1,
    halide_buffer_flag_device_dirty = 2
};

struct halide_device_interface_t;

/* The image handle crossing the boundary (HalideRuntime.h:1710-1737).  `host` addresses the element
 * whose coordinates are the per-dimension mins; caller owns host memory and the dim[] array. */
typedef struct halide_buffer_t {
    uint64_t device;                                          /* @0  device handle (CUdeviceptr) or 0 */
    const struct halide_device_interface_t *device_interface; /* @8  */
    uint8_t *host;                                            /* @16 */
    uint64_t flags;                                           /* @24 */
    struct halide_type_t type;                                /* @32 */
    int32_t dimensions;                                       /* @36 */
    halide_dimension_t *dim;                                  /* @40 */
    void *padding;                                            /* @48 */
} halide_buffer_t;

struct halide_device_interface_impl_t;

/* Function table every buffer with a device allocation points at (HalideRuntime.h:875-899).
 * Halide::Runtime::Buffer calls copy_to_host / device_sync / device_free through it
 * (src/runtime/HalideBuffer.h:352-358,1810-1815). */
struct halide_device_interface_t {
    int (*device_malloc)(void *user_context, struct halide_buffer_t *buf,
                         const struct halide_device_interface_t *device_interface);
    int (*device_free)(void *user_context, struct halide_buffer_t *buf);
    int (*device_sync)(void *user_context, struct halide_buffer_t *buf);
    void (*device_release)(void *user_context, const struct halide_device_interface_t *device_interface);
    int (*copy_to_host)(void *user_context, struct halide_buffer_t *buf);
    int (*copy_to_device)(void *user_context, struct halide_buffer_t *buf,
                          const struct halide_device_interface_t *device_interface);
    int (*device_and_host_malloc)(void *user_context, struct halide_buffer_t *buf,
                                  const struct halide_device_interface_t *device_interface);
    int (*device_and_host_free)(void *user_context, struct halide_buffer_t *buf);
    int (*buffer_copy)(void *user_context, struct halide_buffer_t *src,
                       const struct halide_device_interface_t *dst_device_interface, struct halide_buffer_t *dst);
    int (*device_crop)(void *user_context, const struct halide_buffer_t *src, struct halide_buffer_t *dst);
    int (*device_slice)(void *user_context, const struct halide_buffer_t *src, int slice_dim, int slice_pos,
                        struct halide_buffer_t *dst);
    int (*device_release_crop)(void *user_context, struct halide_buffer_t *buf);
    int (*wrap_native)(void *user_context, struct halide_buffer_t *buf, uint64_t handle,
                       const struct halide_device_interface_t *device_interface);
    int (*detach_native)(void *user_context, struct halide_buffer_t *buf);
    int (*compute_capability)(void *user_context, int *major, int *minor);
    const struct halide_device_interface_impl_t *impl;
};

/* Return codes (HalideRuntime.h:1152-1357); only the ones this library can produce are named. */
enum halide_error_code_t {
    halide_error_code_success = 0,
    halide_error_code_generic_error = -1,
    halide_error_code_explicit_bounds_too_small = -2,
    halide_error_code_bad_type = -3,
    halide_error_code_access_out_of_bounds = -4,
    halide_error_code_buffer_allocation_too_large = -5,
    halide_error_code_buffer_extents_too_large = -6,
    halide_error_code_constraints_make_required_region_smaller = -7,
    halide_error_code_constraint_violated = -8,
    halide_error_code_param_too_small = -9,
    halide_error_code_param_too_large = -10,
    halide_error_code_out_of_memory = -11,
    halide_error_code_buffer_argument_is_null = -12,
    halide_error_code_copy_to_host_failed = -14,
    halide_error_code_copy_to_device_failed = -15,
    halide_error_code_device_malloc_failed = -16,
    halide_error_code_device_sync_failed = -17,
    halide_error_code_device_free_failed = -18,
    halide_error_code_no_device_interface = -19,
    halide_error_code_unimplemented = -20,
    halide_error_code_internal_error = -22,
    halide_error_code_device_run_failed = -23,
    halide_error_code_buffer_extents_negative = -28,
    halide_error_code_gpu_device_error = -29,
    halide_error_code_device_wrap_native_failed = -32,
    halide_error_code_device_detach_native_failed = -33,
    halide_error_code_host_is_null = -34,
    halide_error_code_host_and_device_dirty = -37,
    halide_error_code_buffer_is_null = -38,
    halide_error_code_device_buffer_copy_failed = -39,
    halide_error_code_device_crop_unsupported = -40,
    halide_error_code_incompatible_device_interface = -42,
    halide_error_code_bad_dimensions = -43,
    halide_error_code_device_dirty_with_no_device_support = -44
};

/* Scalar value cell used by the metadata tables (HalideRuntime.h:1880-1900). */
struct halide_scalar_value_t {
    union {
        uint8_t b;
        int8_t i8;
        int16_t i16;
        int32_t i32;
        int64_t i64;
        uint8_t u8;
        uint16_t u16;
        uint32_t u32;
        uint64_t u64;
        float f32;
        double f64;
        void *handle;
    } u;
};

enum halide_argument_kind_t {
    halide_argument_kind_input_scalar = 0,
    halide_argument_kind_input_buffer = 1,
    halide_argument_kind_output_buffer = 2
};

/* Per-argument metadata record (HalideRuntime.h:1937-1951). */
struct halide_filter_argument_t {
    const char *name;
    int32_t kind;
    int32_t dimensions;
    struct halide_type_t type;
    const struct halide_scalar_value_t *scalar_def, *scalar_min, *scalar_max, *scalar_estimate;
    int64_t const *const *buffer_estimates;
};

/* What F_metadata() returns (HalideRuntime.h:1954-1977); apps/blur/test.cpp:158 reads ->target. */
struct halide_filter_metadata_t {
    int32_t version;
    int32_t num_arguments;
    const struct halide_filter_argument_t *arguments;
    const char *target;
    const char *name;
};

typedef void (*halide_error_handler_t)(void *, const char *);
typedef void *(*halide_malloc_t)(void *, size_t);
typedef void (*halide_free_t)(void *, void *);
typedef void (*halide_print_t)(void *, const char *);

#endif /* HALIDE_HALIDERUNTIME_H */

/* ---- runtime shim: the subset of the Halide runtime the filters and harnesses call ---- */

/* Error reporting (HalideRuntime.h:173-195; default handler prints "Error: ..." and aborts,
 * src/runtime/posix_error_handler.cpp:9-41).  halide_set_error_handler returns the old handler. */
void halide_error(void *user_context, const char *msg);
halide_error_handler_t halide_set_error_handler(halide_error_handler_t handler);

/* Host allocator hooks (HalideRuntime.h; installed by tools/halide_malloc_trace.h in apps/camera_pipe/process.cpp). */
halide_malloc_t halide_set_custom_malloc(halide_malloc_t user_malloc);
halide_free_t halide_set_custom_free(halide_free_t user_free);
/* The rest of the host-side hooks tools/RunGenMain.cpp links (HalideRuntime.h:170-181,434-465,2343). */
void *halide_default_malloc(void *user_context, size_t x);
void halide_default_free(void *user_context, void *ptr);
void *halide_malloc(void *user_context, size_t x);
void halide_free(void *user_context, void *ptr);
halide_print_t halide_set_custom_print(halide_print_t print);
void halide_print(void *user_context, const char *msg);
void *halide_get_symbol(const char *name);
#ifdef __cplusplus
int halide_reuse_device_allocations(void *user_context, bool enable);
#else
int halide_reuse_device_allocations(void *user_context, _Bool enable);
#endif

/* Device bookkeeping (src/runtime/device_interface.cpp:30-56,154-205). */
int halide_device_malloc(void *user_context, struct halide_buffer_t *buf,
                         const struct halide_device_interface_t *device_interface);
int halide_device_free(void *user_context, struct halide_buffer_t *buf);
int halide_device_sync(void *user_context, struct halide_buffer_t *buf);
int halide_copy_to_host(void *user_context, struct halide_buffer_t *buf);
/* Copy the region `dst` describes out of `src` (HalideRuntime.h halide_buffer_copy; src/runtime/device_interface.cpp:154-205):
 * to dst's device side when dst_device_interface is halide_cuda_device_interface(), to its host side when it is NULL. */
int halide_buffer_copy(void *user_context, struct halide_buffer_t *src,
                       const struct halide_device_interface_t *dst_device_interface, struct halide_buffer_t *dst);
int halide_copy_to_device(void *user_context, struct halide_buffer_t *buf,
                          const struct halide_device_interface_t *device_interface);
void halide_device_release(void *user_context, const struct halide_device_interface_t *device_interface);

/* CUDA device API (src/runtime/HalideRuntimeCuda.h:21,40-81). */
const struct halide_device_interface_t *halide_cuda_device_interface(void);
int halide_cuda_wrap_device_ptr(void *user_context, struct halide_buffer_t *buf, uint64_t device_ptr);
int halide_cuda_detach_device_ptr(void *user_context, struct halide_buffer_t *buf);
uintptr_t halide_cuda_get_device_ptr(void *user_context, struct halide_buffer_t *buf);
int halide_cuda_release_unused_device_allocations(void *user_context);

/* ---- library extensions (no reference equivalent; plain pointers and sizes only) ---- */

/* Stream every kernel and copy of this thread's subsequent filter calls is issued on
 * (a cudaStream_t passed as void*; NULL = the legacy default stream, which is also torch's
 * default current stream).  Replaces halide_set_cuda_get_stream (HalideRuntimeCuda.h:66-81). */
void halide_b200_set_stream(void *cuda_stream);
void *halide_b200_get_stream(void);
/* A non-blocking stream for a caller thread that pipelines frames (one stream per thread: copies of
 * one thread's frame overlap kernels and copies of another's); destroy synchronises first. */
void *halide_b200_stream_create(void);
int halide_b200_stream_destroy(void *cuda_stream);
/* Select the CUDA device for this process (replaces HL_GPU_DEVICE, src/runtime/gpu_device_selection.cpp). */
int halide_b200_set_device(int ordinal);
/* Number of kernels this library has launched since process start (bench.py's gpu_launches). */
uint64_t halide_b200_kernel_launch_count(void);
/* Library/target identification string, e.g. "x86-64-linux-cuda-cuda_capability_90-h100_native". */
const char *halide_b200_target(void);
/* Bracket the kernels of one filter call with CUDA events on the library stream and report the
 * device time of the most recent call in milliseconds (negative if timing is disabled). */
void halide_b200_set_timing(int enable);
float halide_b200_last_kernel_ms(void);
/* Per-kernel profile: when enabled, every kernel launch is bracketed by CUDA events on its
 * stream.  The report is text, one "name count total_ms" line per kernel; returns bytes needed. */
void halide_b200_profile_enable(int enable);
void halide_b200_profile_reset(void);
int halide_b200_profile_report(char *out, int out_size);


/* ---- multi-GPU (one process per GPU; the reference has no counterpart, SURVEY.md §8e) ---- */

/* NCCL bootstrap: rank 0 obtains a 128-byte id, the host's control plane broadcasts it, every rank
 * joins.  Ranks are ordered top to bottom over the frame's rows. */
int halide_b200_dist_unique_id(char *out128);
int halide_b200_dist_init(int rank, int nranks, const char *id128);
/* In-process loopback group: each of nranks host threads of one process calls this with its rank and from then on
 * is that rank (a thread-local binding, checked before the NCCL communicator); messages are device-to-device copies
 * on the one device.  Every host wait is bounded (about 20 s; then the call returns halide_error_code_generic_error).
 * halide_b200_dist_shutdown on the thread ends its membership. */
int halide_b200_dist_init_loopback(int rank, int nranks);
int halide_b200_dist_shutdown(void);
int halide_b200_dist_rank(void);
int halide_b200_dist_size(void);

/* local_laplacian on this rank's row band of a frame whose rows are [frame_y_min, frame_y_min +
 * frame_y_extent): `input`/`output` hold the band's rows (all columns/channels) with dim[1].min in
 * frame coordinates; ranks are ordered top to bottom.  Communication per call: one exchange of input halo rows with
 * the two row neighbours (every pyramid row a band needs beyond itself is recomputed from them) and one all-to-all
 * gather of a coarse pyramid level.  Bit-identical to the single-GPU filter on the whole frame. */
int halide_b200_local_laplacian_sharded(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                        struct halide_buffer_t *output, int32_t frame_y_min, int32_t frame_y_extent);

/* local_laplacian on every frame of a 4-D (x, y, c, n) uint16 buffer: output frame n = local_laplacian(input frame n,
 * levels, alpha, beta), bit for bit, with repeat_edge acting on x, y, c of the input per frame.  The input must cover
 * the output's region in all four dimensions (else halide_error_code_access_out_of_bounds); a bounds query answers
 * with the output's region.  All frames share one launch sequence: every kernel spreads the batch's work over the
 * whole GPU, and the coarse pyramid levels of all frames run in one cooperative launch. */
int halide_b200_local_laplacian_batch(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                      struct halide_buffer_t *output);

/* local_laplacian on 3-D (x, y, c) uint8 buffers: output = to_u8(local_laplacian(to_u16(input), levels, alpha, beta)),
 * bit for bit, with the element conversions of the reference's image I/O (tools/halide_image_io.h, Internal::convert):
 * to_u16(v) = v * 257 and to_u8(w) = ((w + 128) * 255 + 255) >> 16 in 32-bit arithmetic.  Both happen inside the kernels
 * that read and write the frame, so no uint16 copy of either frame exists.  Bounds, repeat_edge, channel crops, error
 * codes and the bounds query are those of local_laplacian; both buffers must be uint8 (else halide_error_code_bad_type). */
int halide_b200_local_laplacian_u8(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                   struct halide_buffer_t *output);

/* halide_b200_local_laplacian_u8 on every frame of a 4-D (x, y, c, n) uint8 buffer, with the frame rules of
 * halide_b200_local_laplacian_batch: output frame n = halide_b200_local_laplacian_u8(input frame n), bit for bit. */
int halide_b200_local_laplacian_u8_batch(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                         struct halide_buffer_t *output);

/* The four local_laplacian entry points above (uint16 / uint8, one frame / batch) on pixel-interleaved buffers (RGBRGB...,
 * RGBA...): every buffer must have dim[2].stride == 1, dim[0].stride (the pixel pitch) >= dim[2].extent, and positive
 * dim[1].stride (and dim[3].stride), else halide_error_code_constraint_violated — a planar buffer included.  The result
 * is, bit for bit, what the matching planar entry point gives on planar copies of the same buffers; output samples the
 * buffer's channels do not cover (an RGBA frame's alpha under an output of channels [0, 3)) are left untouched.  A
 * bounds query proposes dense interleaved strides (C, W*C, 1[, W*H*C]). */
int halide_b200_local_laplacian_interleaved(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                            struct halide_buffer_t *output);
int halide_b200_local_laplacian_interleaved_batch(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                  struct halide_buffer_t *output);
int halide_b200_local_laplacian_u8_interleaved(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                               struct halide_buffer_t *output);
int halide_b200_local_laplacian_u8_interleaved_batch(struct halide_buffer_t *input, int32_t levels, float alpha, float beta,
                                                     struct halide_buffer_t *output);

/* The seven entry points above (batch, 8-bit and interleaved, in every combination) with the pyramid_levels J of
 * halide_b200_local_laplacian_pyramid_levels (below) as an argument, 1 <= J <= 20.  Buffers, layout rules, error codes
 * and the bounds query are those of the fixed-depth entry point of the same suffix, and J is checked as
 * halide_b200_local_laplacian_pyramid_levels checks it.  Frame n of the output is, bit for bit,
 * halide_b200_local_laplacian_pyramid_levels(J) on a planar uint16 copy of input frame n (8-bit frames converted as
 * halide_b200_local_laplacian_u8 converts them); at J == 8 each is its fixed-depth counterpart, with the same launches. */
int halide_b200_local_laplacian_pyramid_levels_batch(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                     float alpha, float beta, struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_u8(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels, float alpha,
                                                  float beta, struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_u8_batch(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                        float alpha, float beta, struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_interleaved(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                           float alpha, float beta, struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_interleaved_batch(struct halide_buffer_t *input, int32_t pyramid_levels,
                                                                 int32_t levels, float alpha, float beta,
                                                                 struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_u8_interleaved(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels,
                                                              float alpha, float beta, struct halide_buffer_t *output);
int halide_b200_local_laplacian_pyramid_levels_u8_interleaved_batch(struct halide_buffer_t *input, int32_t pyramid_levels,
                                                                    int32_t levels, float alpha, float beta,
                                                                    struct halide_buffer_t *output);

/* camera_pipe on raw bursts and into pixel-interleaved RGB.  Matrices and scalars are camera_pipe's, in the same order,
 * and shared by every frame; the tables they give are computed once per call, and every frame runs in one launch.
 *   halide_b200_camera_pipe_batch:             input uint16 (x, y, n), processed uint8 (x, y, c, n), planar;
 *   halide_b200_camera_pipe_interleaved:       input uint16 (x, y),    processed uint8 (x, y, c), interleaved;
 *   halide_b200_camera_pipe_interleaved_batch: input uint16 (x, y, n), processed uint8 (x, y, c, n), interleaved.
 * Output frame n (absolute coordinate) is, byte for byte, camera_pipe(input frame n), and the same bytes the planar entry
 * point gives on planar copies.  Checks, in camera_pipe's order: types (else halide_error_code_bad_type) and dimension
 * counts (else halide_error_code_bad_dimensions); the bounds query; the layout rules; an empty output (W, H, C or N 0)
 * returns 0; the input must cover, in x and y, the raw region camera_pipe reads for the output's x and y region and, in n,
 * the output's frames, and the output's channels must lie in [0, 3) (else halide_error_code_access_out_of_bounds).
 * Layout: the raw input and a planar output keep camera_pipe's dim[0].stride == 1; an interleaved output must have
 * dim[2].stride == 1, dim[0].stride (the pixel pitch) >= dim[2].extent and positive dim[1].stride (and dim[3].stride),
 * else halide_error_code_constraint_violated.  Samples an interleaved output's channels do not cover (an RGBA frame's
 * alpha under channels [0, 3)) keep their bytes.  A bounds query proposes the raw region over the output's frames with
 * dense strides, and an interleaved output dense interleaved strides (C, W*C, 1[, W*H*C]). */
int halide_b200_camera_pipe_batch(struct halide_buffer_t *input, struct halide_buffer_t *matrix_3200,
                                  struct halide_buffer_t *matrix_7000, float color_temp, float gamma, float contrast,
                                  float sharpen_strength, int32_t blackLevel, int32_t whiteLevel,
                                  struct halide_buffer_t *processed);
int halide_b200_camera_pipe_interleaved(struct halide_buffer_t *input, struct halide_buffer_t *matrix_3200,
                                        struct halide_buffer_t *matrix_7000, float color_temp, float gamma, float contrast,
                                        float sharpen_strength, int32_t blackLevel, int32_t whiteLevel,
                                        struct halide_buffer_t *processed);
int halide_b200_camera_pipe_interleaved_batch(struct halide_buffer_t *input, struct halide_buffer_t *matrix_3200,
                                              struct halide_buffer_t *matrix_7000, float color_temp, float gamma,
                                              float contrast, float sharpen_strength, int32_t blackLevel, int32_t whiteLevel,
                                              struct halide_buffer_t *processed);

/* bilateral_grid with its s_sigma GeneratorParam (the grid cell size in pixels, 8 in bilateral_grid) as an argument:
 * the result is what the generator built with s_sigma computes.  s_sigma must be in [1, 128] (else
 * halide_error_code_param_too_small / _too_large, checked after the buffer checks and the bounds query, before any CUDA
 * call); r_sigma, buffers, error codes and the bounds query follow bilateral_grid, which s_sigma == 8 runs, bit for bit. */
int halide_b200_bilateral_grid_s_sigma(struct halide_buffer_t *input, int32_t s_sigma, float r_sigma,
                                       struct halide_buffer_t *output);

/* The float pipelines bilateral_grid and nl_means on 8-bit frames (a decoded photo, a uint8 torch tensor):
 *   halide_b200_bilateral_grid_u8(in8, r_sigma, out8) == to_u8(bilateral_grid(to_f32(in8), r_sigma))
 *   halide_b200_nl_means_u8(in8, patch_size, search_area, sigma, out8)
 *       == to_u8(nl_means(to_f32(in8), patch_size, search_area, sigma))
 * byte for byte, with the element conversions of the reference's image I/O (tools/halide_image_io.h, Internal::convert):
 * to_f32(v) = v / 255.0f (an IEEE division) and to_u8(f) = (uint8_t)lround(f * 255.0f) (the product rounded to float, then
 * halves away from zero).  Both happen inside the kernels that read and write the frame, so no float copy of either frame
 * exists.  Both buffers must be uint8 (else halide_error_code_bad_type); the float entry points keep refusing uint8.
 * Dimensions, the input's coverage of the output (bilateral_grid), the output's channels [0, 3) (nl_means), the parameter
 * checks and their order, empty outputs, size limits, error codes and the bounds query are those of the float entry
 * point.  bilateral_grid_u8 runs s_sigma = 8. */
int halide_b200_bilateral_grid_u8(struct halide_buffer_t *input, float r_sigma, struct halide_buffer_t *output);
int halide_b200_nl_means_u8(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                            struct halide_buffer_t *output);

/* bilateral_grid, halide_b200_bilateral_grid_u8 and halide_b200_bilateral_grid_s_sigma on video clips: 3-D (x, y, n)
 * float32 (bilateral_grid_batch, _s_sigma_batch) or uint8 (_u8_batch) buffers, e.g. an (N, H, W) tensor.  Output frame n
 * is, bit for bit, what the one-frame entry point gives on input frame n with the same arguments; frames are independent
 * (nothing is clamped or shared across n).  The input must cover the output's x/y region and its frames (else
 * halide_error_code_access_out_of_bounds, naming dimension 2 for the frames); output->dim[2].min selects the input frame
 * each output frame reads.  A bounds query gives the input the output's (x, y, n) region with dense strides.  Strides: as
 * halide_b200_nl_means_batch's (dim[0].stride == 1; rows may be padded, frames may be crops of a larger array, and frame
 * strides may be negative or, on the input, zero).  The frames run in groups whose two scratch grids together stay within
 * 256 MiB, three launches a group; frames so large that fewer than 3 fit (7680 x 4320 at r_sigma 0.1) run one at a time
 * through the one-frame kernels, on one pair of grids.  Everything else follows the one-frame entry points:
 * element types (the float entry points refuse uint8 and the reverse), the argument checks and their order, s_sigma in
 * [1, 128], r_sigma > 0, the bins limit, size limits and error codes; an empty output (W, H or N of 0) returns 0 before
 * any CUDA call.  _u8_batch runs s_sigma = 8, as _u8 does. */
int halide_b200_bilateral_grid_batch(struct halide_buffer_t *input, float r_sigma, struct halide_buffer_t *output);
int halide_b200_bilateral_grid_u8_batch(struct halide_buffer_t *input, float r_sigma, struct halide_buffer_t *output);
int halide_b200_bilateral_grid_s_sigma_batch(struct halide_buffer_t *input, int32_t s_sigma, float r_sigma,
                                             struct halide_buffer_t *output);

/* nl_means and halide_b200_nl_means_u8 on video clips and pixel-interleaved frames, with nl_means' arguments:
 *   halide_b200_nl_means_batch / _u8_batch:                   4-D (x, y, c, n) float32 / uint8 buffers, planar;
 *   halide_b200_nl_means_interleaved / _u8_interleaved:       3-D (x, y, c), interleaved;
 *   halide_b200_nl_means_interleaved_batch / _u8_interleaved_batch: 4-D, interleaved.
 * Batch: output frame n is, bit for bit, what nl_means (nl_means_u8) gives on input frame n, with x, y and c clamped
 * inside each frame as nl_means clamps them; every frame runs in one launch.  The input's frames must cover the output's
 * (else halide_error_code_access_out_of_bounds); a bounds query gives the input the output's x/y region, channels [0, 3)
 * and the output's frames.
 * Interleaved: the result is, bit for bit, what the planar entry point gives on planar copies of the same buffers.  Every
 * buffer must have dim[2].stride == 1, dim[0].stride (the pixel pitch) >= dim[2].extent and positive dim[1].stride (and
 * dim[3].stride), else halide_error_code_constraint_violated, a planar buffer included.  The output keeps nl_means'
 * channels [0, 3); the samples of an output pixel it does not cover (an RGBA frame's alpha) keep their values, and an
 * RGBA input's alpha is never read.  A bounds query proposes dense interleaved strides (C, W*C, 1[, W*H*C]).
 * Everything else is nl_means' (nl_means_u8's): element types (float32 entry points refuse uint8 and the reverse), the
 * argument checks and their order, the patch_size / search_area ranges and codes, empty outputs (0, before any CUDA
 * call), size limits, the 8-bit conversions and halide_b200_nl_means_variant.  nl_means and nl_means_u8 themselves keep
 * refusing 4-D and interleaved buffers. */
int halide_b200_nl_means_batch(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                               struct halide_buffer_t *output);
int halide_b200_nl_means_interleaved(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                     struct halide_buffer_t *output);
int halide_b200_nl_means_interleaved_batch(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                           float sigma, struct halide_buffer_t *output);
int halide_b200_nl_means_u8_batch(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma,
                                  struct halide_buffer_t *output);
int halide_b200_nl_means_u8_interleaved(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                        float sigma, struct halide_buffer_t *output);
int halide_b200_nl_means_u8_interleaved_batch(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area,
                                              float sigma, struct halide_buffer_t *output);

/* conv_layer (3x3 convolution + bias + relu, float32) at any shape: the generator's algorithm without its set_bounds /
 * set_stride constraints,
 *   relu(co, x, y, n) = max(0, bias(co) + sum over ky, kx, ci of filter(co, kx, ky, ci) * input(ci, x + kx, y + ky, n)).
 * CO, W, H, N and the mins (c0, x0, y0, n0) are relu's; CI is filter's extent in dimension 3 (input's in dimension 0 when
 * filter is the buffer of a bounds query).  Nothing is edge-clamped: input must cover [0, CI) x [x0, x0 + W + 2) x
 * [y0, y0 + H + 2) x [n0, n0 + N), filter [c0, c0 + CO) x [0, 3) x [0, 3) x [0, CI) and bias [c0, c0 + CO), else
 * halide_error_code_access_out_of_bounds; buffers may be larger, mins need not be 0, and every stride but dim[0].stride
 * (1, else halide_error_code_constraint_violated) is free, so rows may be padded and buffers may be crops of larger
 * tensors; elements of relu's memory outside its region are not written.  Types and dimension counts are conv_layer's.  A
 * bounds query answers with the regions above and dense strides; a relu with a zero extent does nothing and returns 0.  At
 * conv_layer's shape the result equals conv_layer's byte for byte. */
int halide_b200_conv_layer_any_shape(struct halide_buffer_t *input, struct halide_buffer_t *filter,
                                     struct halide_buffer_t *bias, struct halide_buffer_t *relu);

/* local_laplacian with its pyramid_levels GeneratorParam J (the pyramid depth, 8 in local_laplacian) as an argument: the
 * result is what the generator built with pyramid_levels = J computes, bit for bit.  J must be in [1, 20] (else
 * halide_error_code_param_too_small / _too_large, checked after the buffer checks, the bounds query and the levels check,
 * before any CUDA call); buffers (3-D, planar, uint16), levels, alpha, beta, error codes and the bounds query follow
 * local_laplacian, which J == 8 runs.  J does not change the input region required: it is the output's. */
int halide_b200_local_laplacian_pyramid_levels(struct halide_buffer_t *input, int32_t pyramid_levels, int32_t levels, float alpha,
                                               float beta, struct halide_buffer_t *output);
/* Host-only probe for tests: the last pyramid level halide_b200_local_laplacian_pyramid_levels gives launches of its own
 * on a frame_w x frame_h frame (the levels above it share one cooperative launch); -1 for arguments out of range. */
int halide_b200_ll_last_own_level(int32_t frame_w, int32_t frame_h, int32_t pyramid_levels);

/* stencil_chain with its stencils GeneratorParam S (the number of chained 5x5 stages, 32 in stencil_chain) as an argument:
 * the result is what the generator built with stencils = S computes, bit for bit.  Stage s + 1 is the 5x5 stencil with
 * weights (i+3)(j+3) in Z/2^16 applied to stage s; stage 0 is repeat_edge(input).  S must be in [1, 100] (else
 * halide_error_code_param_too_small / _too_large, checked after the buffer checks, the bounds query and the empty-buffer
 * handling, before any CUDA call); buffers (2-D uint16), error codes and the bounds query follow stencil_chain, which
 * S == 32 runs.  The device scratch grows with S: two (W + 4S - 16) x (H + 4S - 16) uint16 planes from S = 9 up (one
 * from S = 5 to 8, none below 5). */
int halide_b200_stencil_chain_stencils(struct halide_buffer_t *input, int32_t stencils, struct halide_buffer_t *output);

/* halide_blur, stencil_chain and halide_b200_stencil_chain_stencils on video clips: 3-D (x, y, n) uint16 buffers, e.g.
 * an (N, H, W) tensor.  Output frame n is, bit for bit, what the one-frame entry point gives on input frame n with the
 * same arguments; frames are independent (stencil_chain's repeat_edge applies in x and y within each frame, and nothing
 * is clamped or shared across n).  output->dim[2].min selects the input frame each output frame reads, and the input's
 * frames must cover the output's (else halide_error_code_access_out_of_bounds, naming dimension 2).  In x and y:
 * blur_batch needs [ox, ox + W + 1] x [oy, oy + H + 1] of every output frame, as halide_blur does; the stencil_chain
 * batches need a non-empty input, as stencil_chain does.  A bounds query gives the input that region (stencil_chain: the
 * output's), extended by the output's frame range, with dense strides.  Strides: as halide_b200_bilateral_grid_batch's
 * (dim[0].stride == 1; rows may be padded, frames may be crops of a larger array, and frame strides may be negative or,
 * on the input, zero).  blur_batch is one launch for any N.  The stencil_chain batches run the launch plan once per group
 * of frames, ceil(S / 4) launches a group; a group holds as many frames as their scratch planes fit in 256 MiB, at most
 * 65 535, and a group of one frame runs the one-frame kernels.  Everything else follows the one-frame entry points: the
 * argument checks and their order, stencils in [1, 100] with the same message, size limits and error codes; an empty
 * output (W, H or N of 0) returns 0 before the parameter checks and any CUDA call.  stencil_chain_batch runs S = 32. */
int halide_b200_blur_batch(struct halide_buffer_t *input, struct halide_buffer_t *blur_y);
int halide_b200_stencil_chain_batch(struct halide_buffer_t *input, struct halide_buffer_t *output);
int halide_b200_stencil_chain_stencils_batch(struct halide_buffer_t *input, int32_t stencils, struct halide_buffer_t *output);

/* Host-only probe of the band geometry for tests: with level jr gathered, out[j*8..j*8+7] = {own.lo, own.hi, d.lo, d.hi,
 * u.lo, u.hi, S.lo, S.hi} per pyramid level j = 0..7 (rows owned in the gather partition / Gaussian-side rows computed and
 * held / outGPyramid rows needed / the level's rows on the whole frame), out[64..65] = input rows read. */
int halide_b200_ll_band_geometry(int32_t frame_w, int32_t frame_h, int32_t band_lo, int32_t band_hi, int32_t first,
                                 int32_t last, int32_t jr, int32_t *out);
/* Row-sharded local_laplacian: pyramid level gathered all-to-all so that the coarser levels are computed
 * redundantly on every rank without further exchange.  0 = chosen by size (default), n >= 2 = level n.
 * Collective setting: all ranks must agree. */
void halide_b200_ll_shard_coarse_level(int level);
/* The level the sharded call gathers for a frame_w x frame_h frame over nranks ranks; host-only. */
int halide_b200_ll_shard_plan_level(int32_t frame_w, int32_t frame_h, int32_t nranks);
/* Test hook: bitmask routing levels==8 calls through the generic kernels (1 down, 2 up, 4 final,
 * 8 no fused coarse launch, 16 general-layout final kernel, 64 no TMA frame tile in the final
 * kernel) so every code path stays covered by the parity tests. */
void halide_b200_ll_force_generic(int mask);
/* Test hook: take (hold = 1) or drop (hold = 0) one hold on local_laplacian's cached remap table of (levels, alpha), as a
 * call does from its lookup to its last launch; taking builds the table if it is missing.  A held table is never evicted
 * from the cache.  0, or a negative halide_error_code_t (dropping a table that is not held: generic_error). */
int halide_b200_ll_lut_hold(int32_t levels, float alpha, int32_t hold);
/* halide_blur (and halide_b200_blur_batch) test hook: 1 = route 4-byte-aligned frames through the general (any alignment)
 * kernel as well;
 * >= 8 = aligned kernel with strips of that many rows (0 restores the defaults). */
void halide_b200_blur_force_general(int enable);
/* nl_means test hook: 1 = generic kernel for every patch / search size, so it can be checked on the sizes the
 * register-window kernel takes by default (patch 3 or 7, search 7); any other value restores the default. */
void halide_b200_nl_means_variant(int variant);
/* Device self-test of the fast kernels' arithmetic shortcuts; returns mismatches vs div.rn / cvt, or -1. */
long long halide_b200_selftest_arith(unsigned long long n, unsigned long long seed);
/* Device evaluation of one scalar primitive of the float pipelines (hl_math.cuh) over n elements of device arrays,
 * out[i] = f(a[i] [, b ...]); returns 0 or a negative halide_error_code_t.  fn, with the element types of a, b and out:
 *   0 halide_exp, 1 halide_log, 2 fast_exp, 3 clamp01        a float, out float
 *   4 halide_pow(a[i], b[i])                                a, b float, out float
 *   5 clampf(a[i], b[2i], b[2i+1]), 6 lerpf(a[i], b[2i], b[2i+1])  a float, b float pairs, out float
 *   7, 8, 9 evaluate_polynomial with 8, 10 and 7 coefficients (halide_exp's, halide_log's, and an odd-count set)
 *   10 frame_to_f32<uint8_t>                                a uint8, out float
 *   11 frame_from_f32<uint8_t>                              a float, out uint8
 *   12 frame_val<uint8_t> (u8 -> u16 value, as float)        a uint8, out float
 *   13 frame_narrow<uint8_t> (u16 -> u8)                    a uint16, out uint8
 *   14 pair_u16<uint8_t> (two u8 -> two u16 in one word)    a uint16, out uint32
 * The CPU oracle's oracle_math_vec takes the same numbers 0 .. 9. */
int halide_b200_selftest_math(int fn, const void *a, const void *b, void *out, long long n);
/* camera_pipe's per-call tables for n scalar sets, as its tables kernel computes them: m3200 / m7000 are dense 3x4 float
 * matrices on the device (x fastest); scalars holds n host records {color_temp, gamma, contrast, sharpen_strength} and
 * levels n host records {blackLevel, whiteLevel}.  Writes, on the device, matrix[n][12] (int16 Q8.8, x fastest),
 * curve[n][1024] (uint8) and s32[n] (uint8 sharpen strength x 32).  0 or a negative halide_error_code_t. */
int halide_b200_camera_pipe_tables(const float *m3200, const float *m7000, const float *scalars, const int32_t *levels, int n,
                                   int16_t *matrix, uint8_t *curve, uint8_t *s32);

#ifdef __cplusplus
}
#endif

#endif /* HALIDE_B200_RUNTIME_H */
