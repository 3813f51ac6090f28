// TEST INFRASTRUCTURE ONLY -- host launchers for the reference's frustum query kernels.  oracle/build_ref_frustum.py writes the
// reference's CUDA string to oracle/_ref/frustum_ref_kernels.cu and compiles this file with it; oracle/record_ref_frustum.py calls
// these launchers from ctypes with the arguments of query_point_indices.py:615-770, in the same order and with the same block size.
#include "frustum_ref_kernels.cu"

#define LAUNCH_RET                                   \
    do {                                             \
        cudaError_t e = cudaGetLastError();          \
        if (e == cudaSuccess) e = cudaDeviceSynchronize(); \
        return (int)e;                               \
    } while (0)

extern "C" int ref_get_occ_vox(int grid, int block, const float* in_data, const int* n_actual, int B, int N, const float* shift,
                               const float* vsize, const int* gsize, const int* ksize, int pixel_size, int grid_size_vol,
                               uint8_t* coor_occ, int8_t* loc_coor_counter, int* near_id, int* far_id, int inverse) {
    get_occ_vox<<<grid, block>>>(in_data, n_actual, B, N, shift, vsize, gsize, ksize, pixel_size, grid_size_vol, coor_occ,
                                 loc_coor_counter, near_id, far_id, inverse);
    LAUNCH_RET;
}

extern "C" int ref_near_vox_full(int grid, int block, int B, int SR, const int* pixel_idx, int R, const int* vscale, const int* gsize,
                                 int pixel_size, int grid_size_vol, const int* ksize, uint8_t* pixel_map, int8_t* ray_mask,
                                 const uint8_t* coor_occ, int8_t* loc_coor_counter, const int* near_id, const int* far_id,
                                 short* voxel_to_coorz_idx) {
    near_vox_full<<<grid, block>>>(B, SR, pixel_idx, R, vscale, gsize, pixel_size, grid_size_vol, ksize, pixel_map, ray_mask,
                                   coor_occ, loc_coor_counter, near_id, far_id, voxel_to_coorz_idx);
    LAUNCH_RET;
}

extern "C" int ref_insert_vox_points(int grid, int block, float* in_data, int* n_actual, int B, int N, int P, int max_o,
                                     int pixel_size, int grid_size_vol, const float* shift, const int* gsize, const float* vsize,
                                     const int8_t* loc_coor_counter, short* voxel_pnt_counter, int* voxel_to_pntidx,
                                     unsigned long seconds, int inverse) {
    insert_vox_points<<<grid, block>>>(in_data, n_actual, B, N, P, max_o, pixel_size, grid_size_vol, shift, gsize, vsize,
                                       loc_coor_counter, voxel_pnt_counter, voxel_to_pntidx, seconds, inverse);
    LAUNCH_RET;
}

extern "C" int ref_query_layered(int grid, int block, const float* in_data, int B, int SR, int R, int max_o, int P, int K,
                                 int pixel_size, int grid_size_vol, float radius_limit2, float depth_limit2, const float* shift,
                                 const int* gsize, const float* vsize, const float* ray_vsize, const int* vscale, const int* ksize,
                                 const int* pixel_idx, const int8_t* loc_coor_counter, const short* voxel_to_coorz_idx,
                                 const short* voxel_pnt_counter, const int* voxel_to_pntidx, int* sample_pidx, float* sample_loc,
                                 unsigned long seconds, int NN, int inverse) {
    query_neigh_along_ray_layered<<<grid, block>>>(in_data, B, SR, R, max_o, P, K, pixel_size, grid_size_vol, radius_limit2,
                                                   depth_limit2, shift, gsize, vsize, ray_vsize, vscale, ksize, pixel_idx,
                                                   loc_coor_counter, voxel_to_coorz_idx, voxel_pnt_counter, voxel_to_pntidx,
                                                   sample_pidx, sample_loc, seconds, NN, inverse);
    LAUNCH_RET;
}
