// ssim_tile.cuh — the SSIM map of one 16x16 tile, shared by the image loss (losses.cu) and the evaluation metrics (metrics.cu).
//
// A 256-thread block loads the tile and its 5-pixel halo of both images into sx / sy (26 x 26, zero outside the image, as
// F.conv2d(padding=5) pads), then ssim_tile_horizontal and ssim_tile_vertical form the five window sums of loss_utils.py's _ssim
// (mu1, mu2, E[x^2], E[y^2], E[xy]) with a separable 11-tap convolution in fp32, and ssim_terms the map's value.  Both kernels take
// their SSIM from here, so a tile's map is the same in either.
#pragma once
#include "sgr_common.cuh"

namespace sgr {

constexpr int kSsimTile = 16, kSsimHalo = 5, kSsimExt = kSsimTile + 2 * kSsimHalo;  // 26

// horizontal pass: 26 rows x 16 columns x 5 quantities
__device__ __forceinline__ void ssim_tile_horizontal(const float (&sx)[kSsimExt][kSsimExt + 1], const float (&sy)[kSsimExt][kSsimExt + 1],
                                                     float (&h)[5][kSsimExt][kSsimTile + 1], const GaussWin &win) {
	for (int e = threadIdx.x; e < kSsimExt * kSsimTile; e += 256) {
		const int r = e / kSsimTile, q = e - r * kSsimTile;
		float m1 = 0.f, m2 = 0.f, s11 = 0.f, s22 = 0.f, s12 = 0.f;
#pragma unroll
		for (int k = 0; k < kSsimWin; k++) {
			const float a = sx[r][q + k], b = sy[r][q + k], w = win.w[k];
			m1 += w * a; m2 += w * b; s11 += w * a * a; s22 += w * b * b; s12 += w * a * b;
		}
		h[0][r][q] = m1; h[1][r][q] = m2; h[2][r][q] = s11; h[3][r][q] = s22; h[4][r][q] = s12;
	}
}

struct SsimSums {
	float m1, m2, s11, s22, s12;
};
// vertical pass for the pixel (tx, ty) of the tile
__device__ __forceinline__ SsimSums ssim_tile_vertical(const float (&h)[5][kSsimExt][kSsimTile + 1], const GaussWin &win, int tx, int ty) {
	SsimSums s{0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
	for (int k = 0; k < kSsimWin; k++) {
		const float w = win.w[k];
		s.m1 += w * h[0][ty + k][tx]; s.m2 += w * h[1][ty + k][tx]; s.s11 += w * h[2][ty + k][tx]; s.s22 += w * h[3][ty + k][tx];
		s.s12 += w * h[4][ty + k][tx];
	}
	return s;
}

// S = A1 A2 / (B1 B2) with C1 = 0.01^2, C2 = 0.03^2 and sigma = E[x^2] - mu^2, the reciprocal inv = 1 / (B1 B2) kept for the gradient
struct SsimTerms {
	float A1, A2, B1, B2, inv, S;
};
__device__ __forceinline__ SsimTerms ssim_terms(const SsimSums &s) {
	const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
	const float mu1_sq = s.m1 * s.m1, mu2_sq = s.m2 * s.m2, mu12 = s.m1 * s.m2;
	const float sig1 = s.s11 - mu1_sq, sig2 = s.s22 - mu2_sq, sig12 = s.s12 - mu12;
	SsimTerms t;
	t.A1 = 2.f * mu12 + C1;
	t.A2 = 2.f * sig12 + C2;
	t.B1 = mu1_sq + mu2_sq + C1;
	t.B2 = sig1 + sig2 + C2;
	t.inv = 1.0f / (t.B1 * t.B2);
	t.S = t.A1 * t.A2 * t.inv;
	return t;
}

}  // namespace sgr
