/* ggml-b200-backend.h — entry points of the ggml backend plug-in libggml-b200.so (layer 2 of ggml-b200.h).
 *
 * Same shape as the reference's per-backend public headers (include/ggml-cuda.h:23-45); needs ggml's own
 * headers (ggml.h, ggml-backend.h) on the include path, exactly like those.
 *
 *   dynamic:  GGML_BACKEND_PATH=/path/to/libggml-b200.so  (ggml_backend_load_all, src/ggml-backend-reg.cpp:554-582)
 *             or ggml_backend_load("/path/to/libggml-b200.so") -> exported ggml_backend_init / ggml_backend_score
 *   static:   ggml_backend_register(ggml_backend_b200_reg())  (src/ggml-backend-impl.h:210), or two lines in the
 *             registry constructor under #ifdef GGML_USE_B200 (src/ggml-backend-reg.cpp:155-186)
 *   -DGGML_USE_CUDA programs: the library also exports the ggml_backend_cuda_* symbols of include/ggml-cuda.h.
 */
#ifndef GGML_B200_BACKEND_H
#define GGML_B200_BACKEND_H

#include "ggml.h"
#include "ggml-backend.h"
#include "ggml-b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define GGML_B200_NAME "B200"

GGML_B200_API ggml_backend_reg_t         ggml_backend_b200_reg(void);
GGML_B200_API ggml_backend_t             ggml_backend_b200_init(int device);
GGML_B200_API bool                       ggml_backend_is_b200(ggml_backend_t backend);
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_buffer_type(int device);
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_host_buffer_type(void);
/* weights split by rows over every visible GPU (tensor_split: relative shares per device, NULL = equal), MUL_MAT only; the same thing is
 * returned by ggml_backend_reg_get_proc_address(reg, "ggml_backend_split_buffer_type") (reference: ggml_backend_cuda_split_buffer_type,
 * src/ggml-cuda/ggml-cuda.cu:1000) */
GGML_B200_API ggml_backend_buffer_type_t ggml_backend_b200_split_buffer_type(int main_device, const float * tensor_split);
GGML_B200_API int                        ggml_backend_b200_get_device_count(void);

/* dynamic-loading entry points (typedefs ggml_backend_init_t / ggml_backend_score_t, src/ggml-backend-impl.h:214-218) */
GGML_B200_API ggml_backend_reg_t         ggml_backend_init(void);
GGML_B200_API int                        ggml_backend_score(void);

#ifdef __cplusplus
}
#endif
#endif /* GGML_B200_BACKEND_H */
