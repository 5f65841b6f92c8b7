// Host-side operator builders (ops.cu).
#pragma once
#include "kernels.h"

namespace mgb {

// Pixel rectangle of one conv output tile: tile_w x tile_h == 128, tile_w a power of two, fewest tiles over the image.
void conv_tile_shape(int Hout, int Wout, int* tile_w, int* tile_h);

// A [M, K] bf16 row-major, W [N, K] bf16 row-major.
int fill_linear_params(GemmParams* p, const bf16* a, const bf16* w, int M, int N, int K, int block_n, int splits,
                       int stages, const bf16* a2 = nullptr, int K2 = 0);
// x NHWC bf16 ([NB, Hout, Wout, Cin] for kind 0/1, [NB, 4, Hout, Wout, Cin] parity planes for kind 2/3);
// w [Cout, taps * Cin] bf16 tap-major.
int fill_conv_params(GemmParams* p, const bf16* x, const bf16* w, int NB, int Hout, int Wout, int Cin, int Cout,
                     int kind, int block_n, int splits, int stages, int Hsrc = 0, int Wsrc = 0, const bf16* x2 = nullptr,
                     int Cin2 = 0);
int effective_splits(const GemmParams& p);
// Makes a filled conv (one image, no split-K, no second operand) run tile rows [ty0, ty0 + tiles) of its image with
// tmap_a's row 0 at image row src_y0 and the output's row 0 at image row out_y0 (GemmParams::ty0).
int set_conv_band(GemmParams* p, int ty0, int tiles, int src_y0, int out_y0);
// Launch (plus the deferred epilogue when split-K is active). p.epi must be filled by the caller. Rejects, before any
// launch, a special epilogue with block_n != 16, N > 16 (N != 3 for depth / normals) or missing epilogue inputs.
int run_gemm(GemmParams& p, int block_n, float* splitk_ws, cudaStream_t stream);
// Tile width, split-K factor and pipeline depth of a GEMM with m_tiles 128-row tiles, N columns and num_kb K blocks of 64,
// for epilogue flags `flags` (EPI_GEGLU: widths that are multiples of 64; a special epilogue: width 16, no split-K).
void choose_tile(int m_tiles, int N, int num_kb, int flags, bool allow_split, int* block_n, int* splits,
                 int* stages);

}  // namespace mgb
