// hb_common.h — internal helpers shared by the filter translation units of libhalide_b200.so.
//
// Host side of the drop-in boundary, owned here once for every filter: the call sequence of a
// Halide-generated filter prologue over the buffer arguments (reference:
// src/AddImageChecks.cpp:311-347,404-476,560-686), bounds-query mode (src/AddImageChecks.cpp:477-496,
// 710-716), host/device residency (src/InjectHostDevBufferCopies.cpp,
// src/runtime/device_interface.cpp:154-205), the F_argv / F_metadata / F_auto_schedule exports
// (HB_EXPORT_FILTER, HB_EXPORT_AUTO_SCHEDULE) and the kernel-launch bookkeeping.  The argument
// records the checks read are the filter's metadata (halide_filter_argument_t).  A filter adds only
// its required regions, its own parameter checks and its launches.  Nothing here computes pixels.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <type_traits>
#include <utility>

#include "../../include/halide_b200_runtime.h"

namespace hb {

// ---- error reporting -------------------------------------------------------------------------
// Formats a message, hands it to the (replaceable) halide_error handler and returns `code`,
// mirroring the halide_error_* helpers in src/runtime/errors.cpp:5-80.
int fail(int code, const char *fmt, ...) __attribute__((format(printf, 2, 3)));

// ---- stream / launch accounting --------------------------------------------------------------
cudaStream_t stream();
void count_launch(const char *name, cudaStream_t s);
void profile_begin(const char *name, cudaStream_t s);  // event bracket only (closed by after_launch), not counted as a launch
void after_launch(cudaStream_t s);
int check_cuda(cudaError_t e, const char *what, int code);

// RAII bracket around the kernels of one filter call (halide_b200_set_timing).
struct CallTimer {
    explicit CallTimer(cudaStream_t s);
    ~CallTimer();
    cudaStream_t s;
};

// ---- once-per-device set-up (function attributes are per device / context; keyed by the CURRENT device, and safe
// to race: two threads at worst both run `fn`, which must be idempotent) -----------------------------------------
struct PerDeviceOnce {
    unsigned long long done = 0;  // bit d = device d set up (devices >= 64: always run fn)
    template<typename F>
    void run(F fn) {
        int dev = 0;
        cudaGetDevice(&dev);
        const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
        if (bit && (__atomic_load_n(&done, __ATOMIC_ACQUIRE) & bit)) return;
        fn();
        if (bit) __atomic_fetch_or(&done, bit, __ATOMIC_RELEASE);
    }
};

// ---- device scratch (callee-owned intermediates; pooled, src/runtime/cuda.cpp:760-870 analogue) ---
void *scratch_alloc(size_t bytes);  // returns nullptr on failure (caller maps to -16)
void scratch_free(void *p);         // stream-ordered: safe to call right after the last launch

struct Scratch {  // frees everything it handed out when the filter call returns
    static constexpr int kMax = 48;
    void *ptrs[kMax];
    int n = 0;
    ~Scratch() {
        for (int i = 0; i < n; i++) scratch_free(ptrs[i]);
    }
    template<typename T>
    T *get(size_t count) {
        if (n >= kMax) return nullptr;
        void *p = scratch_alloc(count * sizeof(T));
        if (p) ptrs[n++] = p;
        return (T *)p;
    }
};

// ---- the call boundary of a filter ------------------------------------------------------------
// A filter entry point runs, in this order: check_args; answer_bounds_query (return 0 if it did);
// check_shapes; its required-region and parameter checks (check_required + its own); acquire; its
// launches; finish.  Every step before acquire returns before any CUDA call.
constexpr const char *kTarget = "x86-64-linux-cuda-cuda_capability_90-h100_native";

// One buffer argument: the caller's buffer, its record in the filter's metadata (name, type,
// dimensions, input or output) and, once acquired, the device address of its element at the mins.
struct Arg {
    halide_buffer_t *b;
    const halide_filter_argument_t &meta;
    void *dev = nullptr;
};

// The part of a buffer a call touches: proposed by a bounds query, and required of the caller's
// buffer when must_cover (reads without a boundary condition).
struct Region {
    int min[4], extent[4];
    bool must_cover;
};
Region region_of(const halide_buffer_t *b, bool must_cover);  // the buffer's own min/extent

// null → -12, type → -3, dimensions → -43, buffer by buffer in argument order.
int check_args(const Arg *a, int n);
// Bounds-query mode (HalideRuntime.h:1851-1853): every buffer with neither host nor device memory
// gets need[i] with dense strides (src/AddImageChecks.cpp:386-436,477-496).  True if any did.
bool answer_bounds_query(Arg *a, const Region *need, int n);
// negative extent → -28, |extent*stride| and extent product limits → -5/-6, stride[0] != 1 → -8.
int check_shapes(const Arg *a, int n);
// every must_cover region must lie inside its buffer, dimension by dimension → else -4.
int check_required(const Arg *a, const Region *need, int n);
// Inputs: device allocation + H2D when host-dirty or not yet on the device; outputs: allocation
// only.  Sets a[i].dev.  Returns 0 or a negative halide_error_code_t.
int acquire(Arg *a, int n);
// After the launches: a launch error → device_run_failed naming `what`; else the outputs become
// device-dirty.
int finish(const Arg *a, int n, const char *what);

// Metadata default of a scalar argument: all 8 bytes zero but the member set.
halide_scalar_value_t scalar_i32(int32_t v);
halide_scalar_value_t scalar_f32(float v);

// F_argv: a pointer parameter receives args[i], a scalar parameter *(T *)args[i].
template<typename T>
T argv_slot(void *p) {
    if constexpr (std::is_pointer_v<T>) return static_cast<T>(p);
    else return *static_cast<T *>(p);
}
template<typename... A, size_t... I>
int call_argv(int (*f)(A...), void **args, std::index_sequence<I...>) {
    return f(argv_slot<A>(args[I])...);
}
template<typename... A>
int call_argv(int (*f)(A...), void **args) {
    return call_argv(f, args, std::index_sequence_for<A...>{});
}

inline size_t elem_bytes(const halide_buffer_t *b) {
    return (b->type.bits + 7) / 8;
}

}  // namespace hb

// The exports of a Halide AOT filter F besides F itself: F_argv and F_metadata, whose record lists
// ARGS (the filter's halide_filter_argument_t array).
#define HB_METADATA(NAME, ARGS)                                                                       \
    extern "C" const halide_filter_metadata_t *NAME##_metadata(void) {                               \
        static const halide_filter_metadata_t m = {1, (int32_t)(sizeof(ARGS) / sizeof(ARGS[0])), ARGS, \
                                                   hb::kTarget, #NAME};                               \
        return &m;                                                                                    \
    }
#define HB_EXPORT_FILTER(F, ARGS)                                      \
    extern "C" int F##_argv(void **args) { return hb::call_argv(F, args); } \
    HB_METADATA(F, ARGS)
// The harnesses' second AOT variant (apps/*/process.cpp link F_auto_schedule too): the same code
// under the other names.
#define HB_EXPORT_AUTO_SCHEDULE(F, ARGS)                                                 \
    extern "C" decltype(F) F##_auto_schedule __attribute__((alias(#F)));                \
    extern "C" int F##_auto_schedule_argv(void **) __attribute__((alias(#F "_argv"))); \
    HB_METADATA(F##_auto_schedule, ARGS)

// Launch macro: counts the launch, optionally brackets it with events for the per-kernel
// profile (halide_b200_profile_*), and surfaces launch-configuration errors immediately.
#define HB_LAUNCH(NAME, KERNEL, GRID, BLOCK, SMEM, STREAM, ...)        \
    do {                                                               \
        hb::count_launch(NAME, STREAM);                                \
        KERNEL<<<(GRID), (BLOCK), (SMEM), (STREAM)>>>(__VA_ARGS__);    \
        hb::after_launch(STREAM);                                      \
    } while (0)

extern "C" {
// Per-kernel profile: when enabled every HB_LAUNCH is bracketed by CUDA events on its stream.
void halide_b200_profile_enable(int enable);
void halide_b200_profile_reset(void);
// Writes lines "name count total_ms\n" into out (NUL-terminated); returns bytes needed.
int halide_b200_profile_report(char *out, int out_size);
}
