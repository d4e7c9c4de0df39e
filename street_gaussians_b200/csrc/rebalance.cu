// rebalance.cu — the copies of sgr_rebalance_pack / sgr_rebalance_splice (include/sgr.h): moving row ranges of every sub-model's
// parameters, Adam moments and densification statistics between a rank's tensors and its send / receive buffers.  Every row range of a
// contiguous [n, w] tensor is one flat span of floats, so both entries reduce to ONE launch over a table of spans (built and checked in
// capi.cu): each block copies up to kSpanFloats consecutive floats of one span, 8 loads in flight per thread, coalesced.  The copies
// are pure data movement: the bits of every moved float are kept.
#include "sgr_common.cuh"

#include <vector>

namespace sgr {

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 8;
constexpr int kSpanFloats = kThreads * kPerThread;  // floats per block

// span of block b (block_start[] ascending, block_start[n] = number of blocks; spans with no floats are never in the table)
__device__ __forceinline__ int find_span(const int32_t *block_start, int n, int b) {
	int lo = 0, hi = n - 1;
	while (lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if (block_start[mid] <= b) lo = mid; else hi = mid - 1;
	}
	return lo;
}

__global__ void __launch_bounds__(kThreads) copy_spans_kernel(const RebalanceSpan *__restrict__ spans, const int32_t *__restrict__ block_start,
                                                              int nspans) {
	const int s = find_span(block_start, nspans, blockIdx.x);
	const RebalanceSpan sp = spans[s];
	const long long e0 = (long long)(blockIdx.x - block_start[s]) * kSpanFloats;
	const int n = (int)min((long long)kSpanFloats, sp.n - e0);
	const float *__restrict__ src = sp.src + e0;
	float *__restrict__ dst = sp.dst + e0;
	float v[kPerThread];
#pragma unroll
	for (int j = 0; j < kPerThread; j++) {
		const int e = threadIdx.x + j * kThreads;
		if (e < n) v[j] = src[e];
	}
#pragma unroll
	for (int j = 0; j < kPerThread; j++) {
		const int e = threadIdx.x + j * kThreads;
		if (e < n) dst[e] = v[j];
	}
}

}  // namespace

size_t rebalance_scratch_bytes(long long nspans) {
	return align_up(sizeof(RebalanceSpan) * (size_t)(nspans > 0 ? nspans : 1)) + align_up(sizeof(int32_t) * (size_t)(nspans + 1));
}

long long rebalance_blocks(const RebalanceSpan *spans, int nspans) {
	long long blocks = 0;
	for (int i = 0; i < nspans; i++) blocks += (spans[i].n + kSpanFloats - 1) / kSpanFloats;
	return blocks;
}

// spans: HOST, every n > 0, rebalance_blocks(spans) < 2^31; scratch: rebalance_scratch_bytes(nspans) device bytes
cudaError_t launch_rebalance_copy(const RebalanceSpan *spans, int nspans, void *scratch, cudaStream_t st) {
	if (nspans == 0) return cudaSuccess;
	const size_t off = align_up(sizeof(RebalanceSpan) * (size_t)nspans);
	std::vector<char> h(off + sizeof(int32_t) * (size_t)(nspans + 1), 0);
	memcpy(h.data(), spans, sizeof(RebalanceSpan) * nspans);
	int32_t *bstart = reinterpret_cast<int32_t *>(h.data() + off);
	long long blocks = 0;
	for (int i = 0; i < nspans; i++) {
		bstart[i] = (int32_t)blocks;
		blocks += (spans[i].n + kSpanFloats - 1) / kSpanFloats;
	}
	bstart[nspans] = (int32_t)blocks;
	char *d = reinterpret_cast<char *>(scratch);
	cudaError_t e = cudaMemcpyAsync(d, h.data(), h.size(), cudaMemcpyHostToDevice, st);
	if (e != cudaSuccess) return e;
	count_launch();
	copy_spans_kernel<<<(unsigned)blocks, kThreads, 0, st>>>(reinterpret_cast<const RebalanceSpan *>(d), reinterpret_cast<const int32_t *>(d + off),
	                                                        nspans);
	return cudaGetLastError();
}

}  // namespace sgr
