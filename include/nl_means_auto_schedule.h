/* nl_means_auto_schedule.h — stands in for the header Halide's AOT compiler emits for this filter
 * (src/CodeGen_C.cpp:1083-1108 argument order: generator inputs in declaration order, then outputs;
 *  src/CodeGen_C.cpp:675-721 for the _argv and _metadata companions).
 * Generator: /root/reference/apps/nl_means/nl_means_generator.cpp:9-18,162
 * `nl_means_auto_schedule` is the second AOT variant the harness links (the app harness, when built without
 * -DNO_AUTO_SCHEDULE calls it); here it is the same sm_90a implementation under the second name.
 * Returns 0 or a negative halide_error_code_t (include/halide_b200_runtime.h).
 */
#ifndef HALIDE_B200_NL_MEANS_AUTO_SCHEDULE_H
#define HALIDE_B200_NL_MEANS_AUTO_SCHEDULE_H

#include <stdint.h>

struct halide_buffer_t;
struct halide_filter_metadata_t;

#ifdef __cplusplus
extern "C" {
#endif

int nl_means_auto_schedule(struct halide_buffer_t *input, int32_t patch_size, int32_t search_area, float sigma, struct halide_buffer_t *non_local_means);
int nl_means_auto_schedule_argv(void **args);
const struct halide_filter_metadata_t *nl_means_auto_schedule_metadata(void);

#ifdef __cplusplus
}
#endif

#endif /* HALIDE_B200_NL_MEANS_AUTO_SCHEDULE_H */
