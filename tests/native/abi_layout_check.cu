// Prints the layout of every struct of include/b200gsr.h that the Python binding mirrors as a ctypes.Structure
// (dreamscene_b200/_lib.py): one "<struct> sizeof <n>" line per struct and one "<struct> <field> <offset>" line per
// field.  Built with nvcc and run on the CPU by tests/test_abi_binding_cpu.py, which compares the numbers with the
// ctypes offsets and sizes (no GPU needed).
#include <cstddef>
#include <cstdio>
#include "b200gsr.h"

#define SIZE(s) std::printf(#s " sizeof %zu\n", sizeof(s))
#define FIELD(s, f) std::printf(#s " " #f " %zu\n", offsetof(s, f))

int main() {
    SIZE(b200gsr_params);
    FIELD(b200gsr_params, P); FIELD(b200gsr_params, M); FIELD(b200gsr_params, sh_degree);
    FIELD(b200gsr_params, image_height); FIELD(b200gsr_params, image_width); FIELD(b200gsr_params, tanfovx);
    FIELD(b200gsr_params, tanfovy); FIELD(b200gsr_params, scale_modifier); FIELD(b200gsr_params, prefiltered);
    FIELD(b200gsr_params, score_flag); FIELD(b200gsr_params, bg); FIELD(b200gsr_params, viewmatrix);
    FIELD(b200gsr_params, projmatrix); FIELD(b200gsr_params, campos);

    SIZE(b200gsr_view_inputs);
    FIELD(b200gsr_view_inputs, means3D); FIELD(b200gsr_view_inputs, shs); FIELD(b200gsr_view_inputs, colors_precomp);
    FIELD(b200gsr_view_inputs, opacities); FIELD(b200gsr_view_inputs, scales); FIELD(b200gsr_view_inputs, rotations);
    FIELD(b200gsr_view_inputs, cov3D_precomp);

    SIZE(b200gsr_view_grads);
    FIELD(b200gsr_view_grads, d_means3D); FIELD(b200gsr_view_grads, d_means2D); FIELD(b200gsr_view_grads, d_shs);
    FIELD(b200gsr_view_grads, d_colors); FIELD(b200gsr_view_grads, d_opacities); FIELD(b200gsr_view_grads, d_scales);
    FIELD(b200gsr_view_grads, d_rotations); FIELD(b200gsr_view_grads, d_cov3D); FIELD(b200gsr_view_grads, accumulate);

    SIZE(b200gsr_group);
    FIELD(b200gsr_group, xyz); FIELD(b200gsr_group, opacity); FIELD(b200gsr_group, scaling);
    FIELD(b200gsr_group, rotation); FIELD(b200gsr_group, f_dc); FIELD(b200gsr_group, f_rest); FIELD(b200gsr_group, n);

    SIZE(b200gsr_group_grad);
    FIELD(b200gsr_group_grad, xyz); FIELD(b200gsr_group_grad, opacity); FIELD(b200gsr_group_grad, scaling);
    FIELD(b200gsr_group_grad, rotation); FIELD(b200gsr_group_grad, f_dc); FIELD(b200gsr_group_grad, f_rest);

    SIZE(b200gsr_adam_tensor);
    FIELD(b200gsr_adam_tensor, param); FIELD(b200gsr_adam_tensor, grad); FIELD(b200gsr_adam_tensor, exp_avg);
    FIELD(b200gsr_adam_tensor, exp_avg_sq); FIELD(b200gsr_adam_tensor, n); FIELD(b200gsr_adam_tensor, lerp_weight);
    FIELD(b200gsr_adam_tensor, beta2); FIELD(b200gsr_adam_tensor, one_minus_beta2); FIELD(b200gsr_adam_tensor, eps);
    FIELD(b200gsr_adam_tensor, step_size); FIELD(b200gsr_adam_tensor, bc2_sqrt);

    SIZE(b200gsr_saved_layout);
    FIELD(b200gsr_saved_layout, header); FIELD(b200gsr_saved_layout, tile_start); FIELD(b200gsr_saved_layout, work_order);
    FIELD(b200gsr_saved_layout, n_contrib); FIELD(b200gsr_saved_layout, keys); FIELD(b200gsr_saved_layout, geom);
    FIELD(b200gsr_saved_layout, dgeom); FIELD(b200gsr_saved_layout, bwd_items); FIELD(b200gsr_saved_layout, total);

    SIZE(b200gsr_scratch_layout);
    FIELD(b200gsr_scratch_layout, counters); FIELD(b200gsr_scratch_layout, tile_count);
    FIELD(b200gsr_scratch_layout, tile_cursor); FIELD(b200gsr_scratch_layout, rectdepth);
    FIELD(b200gsr_scratch_layout, ms_hist); FIELD(b200gsr_scratch_layout, total);
    return 0;
}
