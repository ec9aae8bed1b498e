// op_checks_emu.cpp — TEST INFRASTRUCTURE ONLY: the acceptance rules of ggml_b200/csrc/b200_op_checks.h, which both the ggml_b200_op_*
// launchers and the plug-in's supports_op apply, compiled for the host and exported with a C ABI for tests/test_op_checks.py.  Each entry
// takes its launcher's arguments without the stream and returns the status the launcher returns; a refusal without a reason returns 1.
#include "../../ggml_b200/csrc/b200_op_checks.h"

using namespace b200;
typedef ggml_b200_tensor T;

static int code(const op_check & r) { return r.ok() || r.reason ? r.code : 1; }

extern "C" {

int emu_get_rows(const T * a, const T * ids, const T * d) { return code(check_get_rows(a, ids, d)); }
int emu_bin_bcast(int32_t op, const T * a, const T * b, const T * d) { return code(check_bin_bcast(op, a, b, d)); }
int emu_norm(const T * s, const T * d) { return code(check_norm(s, d)); }
int emu_norm_affine(const T * s, const T * d1, const float * gain, const T * d2, const float * bias, const T * d3) {
    return code(check_norm_affine(s, d1, gain, d2, bias, d3));
}
int emu_cpy(const T * s, const T * d) { return code(check_cpy(s, d)); }
int emu_cpy2(const T * s, const T * d, const T * s2, const T * d2) { return code(check_cpy2(s, d, s2, d2)); }
int emu_flash_attn_ext(const T * q, const T * k, const T * v, const T * mask, const T * d) { return code(check_flash_attn_ext(q, k, v, mask, d)); }
int emu_mul_mat_f(const T * a, const T * b, const T * d) { return code(check_mul_mat_f(a, b, d)); }
int emu_rope(const T * s, const T * pos, const T * ff, const T * d, const ggml_b200_rope_params * p) { return code(check_rope(s, pos, ff, d, p)); }
int emu_argsort(const T * s, const T * d, int32_t order) { return code(check_argsort(s, d, order)); }
int emu_sum_rows(const T * s, const T * d) { return code(check_sum_rows(s, d)); }
int emu_concat(const T * a, const T * b, const T * d, int32_t dim) { return code(check_concat(a, b, d, dim)); }
int emu_ssm_conv(const T * sx, const T * c, const T * d) { return code(check_ssm_conv(sx, c, d)); }
int emu_ssm_scan(const T * s, const T * x, const T * dt, const T * A, const T * B, const T * C, const T * d) {
    return code(check_ssm_scan(s, x, dt, A, B, C, d));
}

} // extern "C"
