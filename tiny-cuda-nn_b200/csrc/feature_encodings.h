// feature_encodings.h -- the parameter-free encodings (Identity, Frequency, TriangleWave, OneBlob, SphericalHarmonics) as stand-alone
// kernels, and the segment table that describes a Composite encoding (encodings/composite.h:135-215): which input dimensions each
// nested encoding reads and which output columns it writes.
#pragma once
#include "common.cuh"

namespace tcnnb {

enum FeatureType : uint32_t { FEAT_IDENTITY = 0, FEAT_FREQUENCY = 1, FEAT_TRIANGLE_WAVE = 2, FEAT_ONEBLOB = 3, FEAT_SPHERICAL_HARMONICS = 4, FEAT_GRID = 5, FEAT_EMPTY = 6 };

struct FeatureSegment {
	uint32_t type;
	uint32_t in_begin, n_in;     // input dimensions [in_begin, in_begin + n_in)
	uint32_t out_begin;          // first output column
	uint32_t n_out;              // features (without padding)
	uint32_t n_pad;              // padding columns, all ONE (the grid pads with zeros): behind the features, IN FRONT for SphericalHarmonics
	                             // (FEAT_EMPTY: no features, only its padding; the kernels write nothing else for it)
	uint32_t param;              // n_frequencies / log2(n_bins) / degree
	float scale, offset;         // Identity
};

constexpr uint32_t MAX_FEATURE_SEGMENTS = 8;
struct FeatureSegments {
	uint32_t n;
	FeatureSegment s[MAX_FEATURE_SEGMENTS];
};

// encoded rows [n][row_stride] fp16 <- positions rows [n][x_stride] fp32, all non-grid segments of the table in one launch
cudaError_t launch_feature_forward(cudaStream_t stream, const FeatureSegments& segs, uint32_t n, const float* x, uint32_t x_stride, __half* encoded, uint32_t row_stride);
// dL_dx rows [n][x_stride] fp32 (only the segments' own input columns are written) <- dL_dy rows [n][row_stride] fp16
cudaError_t launch_feature_input_gradient(cudaStream_t stream, const FeatureSegments& segs, uint32_t n, const float* x, uint32_t x_stride, const __half* dL_dy, uint32_t row_stride,
                                          float* dL_dx);

}  // namespace tcnnb
