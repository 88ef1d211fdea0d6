// common.cuh -- shared device/host helpers for libcalm_b200 (sm_90a only).
#pragma once

#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

// Same failure behaviour as the reference backend (infer.cu:12-20): report and abort.
#define CUDA_CHECK(x)                                                                                         \
	do {                                                                                                      \
		cudaError_t err_ = (x);                                                                               \
		if (err_ != cudaSuccess) {                                                                            \
			fprintf(stderr, "calm_b200: CUDA error in %s at %s:%d: %s (%s=%d)\n", __FUNCTION__, __FILE__, \
			        __LINE__, cudaGetErrorString(err_), cudaGetErrorName(err_), (int)err_);                   \
			abort();                                                                                          \
		}                                                                                                     \
	} while (0)

#define CALM_FATAL(...)                       \
	do {                                      \
		fprintf(stderr, "calm_b200: " __VA_ARGS__); \
		fprintf(stderr, "\n");                \
		abort();                              \
	} while (0)

// Per-token scalars.  Lives in device memory so that a captured CUDA graph can
// be replayed for every token: the host (forward_cuda) or the device
// (k_advance, greedy decode) rewrites it between replays.
struct TokenParams {
	int token;   // input token id
	int pos;     // absolute position
	int kv_pos;  // cache slot written this step  (reference infer.c:330-332)
	int kv_len;  // cache slots attended this step
	int kv_sink; // 0, or KV_SINKS once the cache rolls over
	int step;    // index into out_tokens (greedy decode)
	int seq_len;
	int tp_seq;  // tokens started so far (tensor parallelism: epoch base of the peer-memory exchange; same on every rank)
};

// ---------------------------------------------------------------- programmatic dependent launch
// Every staged kernel starts with pdl_enter(): it lets the NEXT kernel of the stream be launched right away
// (its CTAs park in their own pdl_enter until this grid has completed and flushed), which takes the launch
// latency off the critical path between the ~160 kernels of a token.  No-ops when launched without the attribute.
__device__ __forceinline__ void pdl_enter() {
	asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
	asm volatile("griddepcontrol.wait;" ::: "memory");
}
// The two halves, for kernels that request their first weight vectors (immutable data, independent of the previous
// grid) between them: the loads are in flight while the previous kernel drains and while the activations are staged.
__device__ __forceinline__ void pdl_launch_next() {
	asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
__device__ __forceinline__ void pdl_wait_prev() {
	asm volatile("griddepcontrol.wait;" ::: "memory");
}
// L2 prefetch of a contiguous range (<= 16 KB, multiple of 16), issued by one thread; fire-and-forget (SASS UBLKPF)
__device__ __forceinline__ void l2_prefetch(const void* p, uint32_t bytes) {
	asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void l2_prefetch_row(const void* row, int rowbytes) {
	for (int off = 0; off < rowbytes; off += 16384) l2_prefetch((const char*)row + off, (uint32_t)min(16384, rowbytes - off));
}

// f32 -> (hi, lo) f16 pair with x = hi + lo up to 2^-22 |x|
__device__ __forceinline__ void split_hl(float x, __half& hi, __half& lo) {
	hi = __float2half_rn(x);
	lo = __float2half_rn(x - __half2float(hi));
}

// ---------------------------------------------------------------- bulk async copies (TMA, 1-D) and mbarriers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
	return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make freshly initialised barriers visible to the async proxy (the TMA unit) before the first copy names them
__device__ __forceinline__ void mbar_init_fence() {
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
	uint32_t ok;
	asm volatile(
	    "{\n\t.reg .pred p;\n\t"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
	    "selp.u32 %0, 1, 0, p;\n\t}"
	    : "=r"(ok)
	    : "r"(smem_u32(bar)), "r"(parity)
	    : "memory");
	return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	while (!mbar_try_wait(bar, parity)) {
	}
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completion is counted on `bar` (SASS UBLKCP)
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
	             "r"(smem_u32(bar))
	             : "memory");
}
__device__ __forceinline__ void tma_load_1d_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t policy) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
	             "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
	             : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
	uint64_t p;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
	return p;
}

// ---------------------------------------------------------------- in-kernel stage stamps (perf_cuda)
// The reference times its stages INSIDE the running kernel with %globaltimer (infer.cu:390-402) so that the
// table describes the production path.  Same here: when a kernel is handed a stamp slot, one thread per CTA
// folds the time it passed the dependency wait into slot[0] (min) and the time it finished into slot[1] (max).
// The production graph passes NULL; the profiling graph (CALM_B200_PERF=1) is the same graph with slots.
__device__ __forceinline__ unsigned long long globaltimer_ns() {
	unsigned long long t;
	asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
	return t;
}
__device__ __forceinline__ void stamp_begin(unsigned long long* slot) {
	if (slot && threadIdx.x == 0) atomicMin(slot, globaltimer_ns());
}
__device__ __forceinline__ void stamp_end(unsigned long long* slot) {
	if (slot) { // uniform over the CTA
		__syncthreads();
		if (threadIdx.x == 0) atomicMax(slot + 1, globaltimer_ns());
	}
}

// ---------------------------------------------------------------- warp / block reductions

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
	for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
	return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
	for (int m = 16; m > 0; m >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, m));
	return v;
}

// Sum over the whole CTA; every thread gets the result.  `red` is >= 32 floats of shared memory.
__device__ __forceinline__ float block_sum(float v, float* red) {
	int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
	v = warp_sum(v);
	__syncthreads(); // protect `red` from a previous use
	if (lane == 0) red[warp] = v;
	__syncthreads();
	float r = lane < nwarps ? red[lane] : 0.f;
	return warp_sum(r);
}

// ---------------------------------------------------------------- streaming loads

// 16-byte weight load: read-only path, no L1 allocation (every weight byte is used once per token).
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
	uint4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
	return r;
}

__device__ __forceinline__ uint2 ldg_stream8(const uint2* p) {
	uint2 r;
	asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
	return r;
}

// ---------------------------------------------------------------- weight formats
//
// A weight row is consumed in 16-byte vectors.  VW = weights per vector.  The
// activation vector is staged in shared memory in a layout that makes the
// matching reads conflict-free 16-byte loads: for vector v = 32*c + lane the
// VW activations are stored as VW/4 float4 "quads", quad q at float4 index
// (c*(VW/4) + q)*32 + (lane ^ xs_swz(q)).  xs_index() maps an activation index to that slot.
// The XOR makes the STAGING stores conflict-free too: consecutive threads stage consecutive float4s of x (coalesced
// loads), i.e. the quads q = 0..Q-1 of one vector, whose slots are 512 bytes apart -- without the swizzle the 8 lanes of a
// 16-byte store phase hit 8/Q bank groups (fp8: 4-way, gf4: 8-way conflicts: 1800 of the w2 kernel's cycles for the
// 57 KB Llama-3 hidden vector, r02 ncu capture: 212 K store conflicts).  Readers XOR their lane with the same constant.

template <int DBITS>
struct WFmt;
template <>
struct WFmt<16> {
	static constexpr int VW = 8;
};
template <>
struct WFmt<8> {
	static constexpr int VW = 16;
};
template <>
struct WFmt<4> {
	static constexpr int VW = 32;
};

template <int DBITS>
__host__ __device__ __forceinline__ constexpr int xs_swz(int q) { // lane permutation of quad q: 8 distinct 16-byte bank groups for the 8 lanes of a store phase
	return (q * (8 / (WFmt<DBITS>::VW / 4))) & 31;
}

template <int DBITS>
__device__ __forceinline__ int xs_index(int j) {
	constexpr int VW = WFmt<DBITS>::VW, Q = VW / 4;
	int v = j / VW, w = j % VW;
	int c = v >> 5, lane = v & 31, q = w >> 2;
	return (((c * Q + q) << 5) + (lane ^ xs_swz<DBITS>(q))) * 4 + (w & 3);
}

// number of floats of the staged activation vector (whole 32-vector chunks, zero padded)
template <int DBITS>
__host__ __device__ __forceinline__ int xs_floats(int n) {
	constexpr int VW = WFmt<DBITS>::VW;
	int nvec = n / VW;
	return ((nvec + 31) & ~31) * VW;
}

// gf4 only: behind the staged vector sit the group sums the decode needs, 3 * (x_8g + ... + x_8g+7) for every group g of 8
// activations (one gf4 word), in plain order: lane l of 32-vector chunk c reads its vector's four sums as ONE float4 at
// index 32 c + l.  They used to be recomputed from the activations by every warp for every row pair (7 FADD per word).
template <int DBITS>
__host__ __device__ __forceinline__ int xs_aux_floats(int n) {
	return DBITS == 4 ? xs_floats<DBITS>(n) / 8 : 0;
}
template <int DBITS>
__host__ __device__ __forceinline__ int xs_all_floats(int n) {
	return xs_floats<DBITS>(n) + xs_aux_floats<DBITS>(n);
}

// e5m2 pair (two bytes) -> two floats.  An e5m2 byte is the high byte of a half
// (reference infer.c:28-35, helpers.cuh:65-98), so a byte permute builds the half2.
__device__ __forceinline__ float2 e5m2x2_lo(uint32_t w) {
	uint32_t h = __byte_perm(w, 0, 0x1404);
	return __half22float2(*reinterpret_cast<__half2*>(&h));
}
__device__ __forceinline__ float2 e5m2x2_hi(uint32_t w) {
	uint32_t h = __byte_perm(w, 0, 0x3424);
	return __half22float2(*reinterpret_cast<__half2*>(&h));
}
__device__ __forceinline__ float e5m2_to_float(uint8_t b) {
	return __half2float(__ushort_as_half((unsigned short)(b << 8)));
}

// float -> e5m2, round to nearest even, saturating to the largest finite value: the same
// conversion the reference's KVT(float) = __nv_fp8_e5m2(float) constructor performs (infer.cu:476-481).
__device__ __forceinline__ uint8_t float_to_e5m2(float f) {
	return (uint8_t)__nv_cvt_float_to_fp8(f, __NV_SATFINITE, __NV_E5M2);
}

// Dot of one 16-byte weight vector with its VW activations (already in registers); g3 = the vector's four group sums (gf4; unused otherwise).
template <int DBITS>
__device__ __forceinline__ float dot_vec(const uint4& w, const float4 (&xv)[WFmt<DBITS>::VW / 4], const float4& g3, float acc);

template <>
__device__ __forceinline__ float dot_vec<16>(const uint4& w, const float4 (&xv)[2], const float4&, float acc) {
	float2 a = __half22float2(*reinterpret_cast<const __half2*>(&w.x));
	float2 b = __half22float2(*reinterpret_cast<const __half2*>(&w.y));
	float2 c = __half22float2(*reinterpret_cast<const __half2*>(&w.z));
	float2 d = __half22float2(*reinterpret_cast<const __half2*>(&w.w));
	acc = fmaf(a.x, xv[0].x, acc);
	acc = fmaf(a.y, xv[0].y, acc);
	acc = fmaf(b.x, xv[0].z, acc);
	acc = fmaf(b.y, xv[0].w, acc);
	acc = fmaf(c.x, xv[1].x, acc);
	acc = fmaf(c.y, xv[1].y, acc);
	acc = fmaf(d.x, xv[1].z, acc);
	acc = fmaf(d.y, xv[1].w, acc);
	return acc;
}

__device__ __forceinline__ float dot_e5m2x4(uint32_t w, const float4& x, float acc) {
	float2 lo = e5m2x2_lo(w), hi = e5m2x2_hi(w);
	acc = fmaf(lo.x, x.x, acc);
	acc = fmaf(lo.y, x.y, acc);
	acc = fmaf(hi.x, x.z, acc);
	acc = fmaf(hi.y, x.w, acc);
	return acc;
}

template <>
__device__ __forceinline__ float dot_vec<8>(const uint4& w, const float4 (&xv)[4], const float4&, float acc) {
	acc = dot_e5m2x4(w.x, xv[0], acc);
	acc = dot_e5m2x4(w.y, xv[1], acc);
	acc = dot_e5m2x4(w.z, xv[2], acc);
	acc = dot_e5m2x4(w.w, xv[3], acc);
	return acc;
}

// gf4 word: bits 0..7 e5m2 scale s, then eight 3-bit codes; w_k = (q_k - 4) * s / -4 (reference infer.c:37-40).
// A code is dropped into the top mantissa bits of 1.0f (0x3F800000 | q << 20 == 1 + q/8, exact): one shift and
// one logic op per weight, no int->float conversion.  With S = sum_k (1 + q_k/8) x_k and X = sum_k x_k:
//   sum_k w_k x_k = (-s/4) (sum_k q_k x_k - 4 X) = (-s/4) (8 S - 12 X) = s (3 X - 2 S).
// `x3` = 3 X of this group of 8 activations (staged once per vector by stage_vector, shared by all rows and warps).
__device__ __forceinline__ float gf4_code(uint32_t w, int k) { // 1 + q_k / 8
	const int sh = 8 + 3 * k - 20; // field k sits at bits 8+3k..10+3k; move it to bits 20..22
	uint32_t f = sh >= 0 ? (w >> sh) : (w << -sh), r;
	asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(f), "r"(0x00700000u), "r"(0x3F800000u)); // (f & mask) | one: a single LOP3
	return __uint_as_float(r);
}
__device__ __forceinline__ float dot_gf4_word(uint32_t w, const float4& x0, const float4& x1, float x3, float acc) {
	float S = gf4_code(w, 0) * x0.x;
	S = fmaf(gf4_code(w, 1), x0.y, S);
	S = fmaf(gf4_code(w, 2), x0.z, S);
	S = fmaf(gf4_code(w, 3), x0.w, S);
	S = fmaf(gf4_code(w, 4), x1.x, S);
	S = fmaf(gf4_code(w, 5), x1.y, S);
	S = fmaf(gf4_code(w, 6), x1.z, S);
	S = fmaf(gf4_code(w, 7), x1.w, S);
	const float sc = e5m2_to_float((uint8_t)(w & 0xff));
	return fmaf(sc, fmaf(-2.f, S, x3), acc);
}

template <>
__device__ __forceinline__ float dot_vec<4>(const uint4& w, const float4 (&xv)[8], const float4& g3, float acc) {
	acc = dot_gf4_word(w.x, xv[0], xv[1], g3.x, acc);
	acc = dot_gf4_word(w.y, xv[2], xv[3], g3.y, acc);
	acc = dot_gf4_word(w.z, xv[4], xv[5], g3.z, acc);
	acc = dot_gf4_word(w.w, xv[6], xv[7], g3.w, acc);
	return acc;
}

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
	return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

// single weight decode (embedding row)
template <int DBITS>
__device__ __forceinline__ float weight_at(const void* w, size_t idx);
template <>
__device__ __forceinline__ float weight_at<16>(const void* w, size_t idx) {
	return __half2float(reinterpret_cast<const __half*>(w)[idx]);
}
template <>
__device__ __forceinline__ float weight_at<8>(const void* w, size_t idx) {
	return e5m2_to_float(reinterpret_cast<const uint8_t*>(w)[idx]);
}
template <>
__device__ __forceinline__ float weight_at<4>(const void* w, size_t idx) {
	uint32_t word = reinterpret_cast<const uint32_t*>(w)[idx >> 3];
	float sf = e5m2_to_float((uint8_t)(word & 0xff)) / -4.f;
	return (float)((int)((word >> (8 + (idx & 7) * 3)) & 7) - 4) * sf;
}

// ---------------------------------------------------------------- KV cache element access

__device__ __forceinline__ void kv_store(__half* p, float v) {
	*p = __float2half_rn(v);
}
__device__ __forceinline__ void kv_store(uint8_t* p, float v) {
	*p = float_to_e5m2(v);
}
__device__ __forceinline__ float kv_load(const __half* p) {
	return __half2float(*p);
}
__device__ __forceinline__ float kv_load(const uint8_t* p) {
	return e5m2_to_float(*p);
}

// 8 consecutive cache elements -> 8 floats
__device__ __forceinline__ void kv_load8(const __half* p, float (&o)[8]) {
	uint4 r = *reinterpret_cast<const uint4*>(p);
	float2 a = __half22float2(*reinterpret_cast<__half2*>(&r.x));
	float2 b = __half22float2(*reinterpret_cast<__half2*>(&r.y));
	float2 c = __half22float2(*reinterpret_cast<__half2*>(&r.z));
	float2 d = __half22float2(*reinterpret_cast<__half2*>(&r.w));
	o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y, o[4] = c.x, o[5] = c.y, o[6] = d.x, o[7] = d.y;
}
__device__ __forceinline__ void kv_load8(const uint8_t* p, float (&o)[8]) {
	uint2 r = *reinterpret_cast<const uint2*>(p);
	float2 a = e5m2x2_lo(r.x), b = e5m2x2_hi(r.x), c = e5m2x2_lo(r.y), d = e5m2x2_hi(r.y);
	o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y, o[4] = c.x, o[5] = c.y, o[6] = d.x, o[7] = d.y;
}
