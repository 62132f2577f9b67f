// match_common.cuh -- types shared by the two Hamming knn2 kernels (match.cu: XOR/POPC, match_tc.cu: wgmma) and their epilogue.
#pragma once
#include "common.cuh"
#include <climits>

struct PairDesc {          // one (left,right) image pair
    int q_row, nq;         // rows of the left image inside the descriptor array
    int t_row, nt;         // rows of the right image
    int64_t out_row;       // first row of this pair in the flattened [sum nq] arrays
    int q_blk, t_blk;      // first 256-row block of the left / right image in the expanded operand store (tensor-core path)
};

struct Top2 { int d0, i0, d1, i1; };

// ordering of cv::batchDistance (K=2): lexicographic on (distance, trainIdx) when candidates arrive in ascending index
__device__ __forceinline__ void top2_insert(Top2& b, int d, int j) {
    if (d < b.d0) { b.d1 = b.d0; b.i1 = b.i0; b.d0 = d; b.i0 = j; }
    else if (d < b.d1) { b.d1 = d; b.i1 = j; }
}

// tensor-core path (match_tc.cu): Hamming on 32-byte descriptors, L2 on u8-valued descriptors of dimension <= 128
int match_tc_splits(int sm_count, int n_pairs, int nq_max, int nt_max);
size_t match_tc_block_bytes(bool l2);
int match_tc_block_rows();
int match_tc_expand(sfmb200_ctx* ctx, const uint32_t* d_desc, const int2* d_blocks, int n_blocks, uint8_t* d_E);
int match_tc_expand_l2(sfmb200_ctx* ctx, const float* d_desc, int dim, const int2* d_blocks, int n_blocks, uint8_t* d_E, int32_t* d_norms, int* d_bad);
int match_tc_launch(sfmb200_ctx* ctx, bool l2, const uint8_t* d_E, const int32_t* d_norms, const PairDesc* d_pairs, int n_pairs, int nq_max, int splits,
                    int4* d_partial, int* d_error_flag);
