// op_checks_emu.cpp — TEST INFRASTRUCTURE ONLY: the acceptance rules of ggml_b200/csrc/b200_op_checks.h, which both the ggml_b200_op_*
// launchers and the plug-in's supports_op apply, compiled for the host and exported with a C ABI: emu_check_<op> for every public
// check_<op>.  Each entry takes its launcher's arguments without the stream and returns the status the launcher returns (check_code.h).
#include "check_code.h"

using namespace b200;
typedef ggml_b200_tensor T;

extern "C" {

int emu_check_get_rows(const T * a, const T * ids, const T * d) { return code(check_get_rows(a, ids, d)); }
int emu_check_bin_bcast(int32_t op, const T * a, const T * b, const T * d) { return code(check_bin_bcast(op, a, b, d)); }
int emu_check_norm(const T * s, const T * d) { return code(check_norm(s, d)); }
int emu_check_norm_affine(const T * s, const T * d1, const T * gain, const T * d2, const T * bias, const T * d3) {
    return code(check_norm_affine(s, d1, gain, d2, bias, d3));
}
int emu_check_scale(const T * s, const T * d) { return code(check_scale(s, d)); }
int emu_check_diag_mask_inf(const T * s, const T * d) { return code(check_diag_mask_inf(s, d)); }
int emu_check_unary(int32_t uop, const T * s, const T * d) { return code(check_unary(uop, s, d)); }
int emu_check_soft_max(const T * s, const T * mask, const T * d) { return code(check_soft_max(s, mask, d)); }
int emu_check_cpy(const T * s, const T * d) { return code(check_cpy(s, d)); }
int emu_check_cpy2(const T * s, const T * d, const T * s2, const T * d2) { return code(check_cpy2(s, d, s2, d2)); }
int emu_check_flash_attn_ext(const T * q, const T * k, const T * v, const T * mask, const T * d) { return code(check_flash_attn_ext(q, k, v, mask, d)); }
int emu_check_mul_mat_f(const T * a, const T * b, const T * d) { return code(check_mul_mat_f(a, b, d)); }
int emu_check_rope(const T * s, const T * pos, const T * ff, const T * d, const ggml_b200_rope_params * p) { return code(check_rope(s, pos, ff, d, p)); }
int emu_check_argsort(const T * s, const T * d, int32_t order) { return code(check_argsort(s, d, order)); }
int emu_check_sum_rows(const T * s, const T * d) { return code(check_sum_rows(s, d)); }
int emu_check_concat(const T * a, const T * b, const T * d, int32_t dim) { return code(check_concat(a, b, d, dim)); }
int emu_check_ssm_conv(const T * sx, const T * c, const T * d) { return code(check_ssm_conv(sx, c, d)); }
int emu_check_ssm_scan(const T * s, const T * x, const T * dt, const T * A, const T * B, const T * C, const T * d) {
    return code(check_ssm_scan(s, x, dt, A, B, C, d));
}
int emu_check_rwkv_wkv6(const T * k, const T * v, const T * r, const T * tf, const T * td, const T * s, const T * d) {
    return code(check_rwkv_wkv6(k, v, r, tf, td, s, d));
}
int emu_check_gated_linear_attn(const T * k, const T * v, const T * q, const T * g, const T * s, const T * d) {
    return code(check_gated_linear_attn(k, v, q, g, s, d));
}
int emu_check_im2col(const T * k, const T * x, const T * d, const ggml_b200_im2col_params * p) { return code(check_im2col(k, x, d, p)); }
int emu_check_pool_2d(const T * s, const T * d, const ggml_b200_pool_params * p) { return code(check_pool_2d(s, d, p)); }
int emu_check_upscale(const T * s, const T * d) { return code(check_upscale(s, d)); }
int emu_check_leaky_relu(const T * s, const T * d) { return code(check_leaky_relu(s, d)); }
int emu_check_repeat(const T * s, const T * d) { return code(check_repeat(s, d)); }
int emu_check_win_part(const T * s, const T * d, int32_t npx, int32_t npy, int32_t w) { return code(check_win_part(s, d, npx, npy, w)); }
int emu_check_win_unpart(const T * s, const T * d, int32_t w) { return code(check_win_unpart(s, d, w)); }
int emu_check_get_rel_pos(const T * s, const T * d) { return code(check_get_rel_pos(s, d)); }
int emu_check_add_rel_pos(const T * a, const T * pw, const T * ph, const T * d) { return code(check_add_rel_pos(a, pw, ph, d)); }
int emu_check_conv_transpose_2d(const T * k, const T * x, const T * d, int32_t stride) { return code(check_conv_transpose_2d(k, x, d, stride)); }
int emu_check_out_prod(const T * a, const T * b, const T * d) { return code(check_out_prod(a, b, d)); }
int emu_check_cross_entropy_loss(const T * x, const T * l, const T * d) { return code(check_cross_entropy_loss(x, l, d)); }
int emu_check_cross_entropy_loss_back(const T * g, const T * x, const T * l, const T * d) { return code(check_cross_entropy_loss_back(g, x, l, d)); }
int emu_check_opt_step_adamw(const T * w, const T * g, const T * m, const T * v, const T * p) { return code(check_opt_step_adamw(w, g, m, v, p)); }
int emu_check_argmax(const T * s, const T * d) { return code(check_argmax(s, d)); }
int emu_check_count_equal(const T * a, const T * b, const T * d) { return code(check_count_equal(a, b, d)); }
int emu_check_sum(const T * s, const T * d) { return code(check_sum(s, d)); }
int emu_check_repeat_back(const T * s, const T * d) { return code(check_repeat_back(s, d)); }

} // extern "C"
