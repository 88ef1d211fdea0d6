// stages.cuh -- one kernel per stage of calm's per-token forward() ("staged" engine).
//
// Stage list per layer (reference CPU order, infer.c:349-458; CUDA stages infer.cu:441-620):
//   k_qkv       RMSNorm -> q,k,v matvec (+bias, clip) -> RoPE -> q vector / KV-cache append
//   k_attn      flash-decoding over the KV cache: scores, online softmax, value mix, split over positions
//   k_matres    x += W . v              (attention output projection wo; FFN down projection w2, MoE-weighted)
//   k_ffn_up    RMSNorm -> [router] -> silu/gelu(w1 . xn) * (w3 . xn)
// and once per token: k_embed (embedding row + sink re-rotation) and k_output (final norm + classifier
// [+ greedy argmax]).  Every weight byte is read exactly once per token with 16-byte loads.
#pragma once

#include "common.cuh"

#include <cooperative_groups.h>

#define CALM_MAX_ACTIVE 8 // experts evaluated per token (Mixtral: 2)

struct MoeSel { // router decision of the current layer, written by k_ffn_up, read by k_matres
	int expert[CALM_MAX_ACTIVE];
	float weight[CALM_MAX_ACTIVE];
};

// ------------------------------------------------------------------------------------------------
// Warp-level matvec core: R rows (any pointers) against the staged activation vector.
// Each lane owns every 32nd 16-byte vector of a row; U vectors per row are requested before the
// first is consumed, so a warp keeps R*U*512 bytes in flight.

template <int DBITS, int R, int U, bool CHECK = true>
__device__ __forceinline__ void rows_consume(const uint4 (&w)[U][R], int v0, int nvec, const float4* __restrict__ xs4, float (&acc)[R]) {
	constexpr int Q = WFmt<DBITS>::VW / 4;
	const int lane = threadIdx.x & 31;
#pragma unroll
	for (int u = 0; u < U; ++u) {
		int v = v0 + 32 * u;
		if (!CHECK || v < nvec) {
			float4 xv[Q];
			const float4* xp = xs4 + (size_t)(v >> 5) * Q * 32;
#pragma unroll
			for (int q = 0; q < Q; ++q) xv[q] = xp[q * 32 + (lane ^ xs_swz<DBITS>(q))];
			float4 g3 = make_float4(0.f, 0.f, 0.f, 0.f);
			if (DBITS == 4) g3 = xs4[(xs_floats<DBITS>(nvec * WFmt<DBITS>::VW) >> 2) + v]; // the vector's group sums (common.cuh xs_aux_floats)
#pragma unroll
			for (int r = 0; r < R; ++r) acc[r] = dot_vec<DBITS>(w[u][r], xv, g3, acc[r]);
		}
	}
}

template <int DBITS, int R, int U = 4>
__device__ __forceinline__ void warp_dot_rows(const uint4* const (&rp)[R], int nvec, const float4* __restrict__ xs4, float (&out)[R]) {
	const int lane = threadIdx.x & 31;

	float acc[R];
#pragma unroll
	for (int r = 0; r < R; ++r) acc[r] = 0.f;

	if (nvec % (32 * U) == 0) { // whole batches (every production shape): no bounds predicates in the hot loop
		for (int v0 = lane; v0 < nvec; v0 += 32 * U) {
			uint4 w[U][R];
#pragma unroll
			for (int u = 0; u < U; ++u)
#pragma unroll
				for (int r = 0; r < R; ++r) w[u][r] = ldg_stream(rp[r] + v0 + 32 * u);
			rows_consume<DBITS, R, U, false>(w, v0, nvec, xs4, acc);
		}
	} else {
		for (int v0 = lane; v0 < nvec; v0 += 32 * U) {
			uint4 w[U][R];
#pragma unroll
			for (int u = 0; u < U; ++u) {
				int v = v0 + 32 * u;
#pragma unroll
				for (int r = 0; r < R; ++r) w[u][r] = v < nvec ? ldg_stream(rp[r] + v) : make_uint4(0, 0, 0, 0);
			}
			rows_consume<DBITS, R, U>(w, v0, nvec, xs4, acc);
		}
	}
#pragma unroll
	for (int r = 0; r < R; ++r) out[r] = warp_sum(acc[r]);
}

// (batched body of stage_vector below: every thread owns up to SV_MAX 16-byte pieces)
// RMSNorm is applied the way the reference CUDA backend applies it (infer.cu:296-330, 453): x * weight goes to shared
// memory at once and the matvec RESULT is multiplied by 1/sqrt(mean(x^2) + eps), so the only thing between the loads of
// x and the first weight load is ONE barrier (which also publishes the per-warp sums of squares).  LayerNorm needs
// the mean first and keeps the two-pass form of the CPU reference (infer.c:183-207).  Returns that output factor.
template <int DBITS, int SV_MAX>
__device__ __forceinline__ float stage_vector_batched(float* xs, float* red, const float* __restrict__ x, int n, const float* __restrict__ normw, float eps, bool ln,
                                                      float* xb_out) {
	const int tid = threadIdx.x, nthr = blockDim.x;
	const int n4 = n >> 2;
	const int total4 = xs_floats<DBITS>(n) >> 2;
	const float4* x4 = reinterpret_cast<const float4*>(x);
	float4 v[SV_MAX];
#pragma unroll
	for (int k = 0; k < SV_MAX; ++k) {
		int i = tid + k * nthr;
		v[k] = i < n4 ? __ldcg(x4 + i) : make_float4(0.f, 0.f, 0.f, 0.f);
	}
	float post = 1.f;
	bool rms = false;
	if (normw) {
		float4 w[SV_MAX];
#pragma unroll
		for (int k = 0; k < SV_MAX; ++k) {
			int i = tid + k * nthr;
			w[k] = i < n4 ? __ldg(reinterpret_cast<const float4*>(normw) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
		}
		if (ln) {
			float s = 0.f;
#pragma unroll
			for (int k = 0; k < SV_MAX; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
			const float mean = block_sum(s, red) / n;
			float ss = 0.f;
#pragma unroll
			for (int k = 0; k < SV_MAX; ++k) {
				if (tid + k * nthr < n4) {
					float dx = v[k].x - mean, dy = v[k].y - mean, dz = v[k].z - mean, dw = v[k].w - mean;
					ss = fmaf(dx, dx, ss), ss = fmaf(dy, dy, ss), ss = fmaf(dz, dz, ss), ss = fmaf(dw, dw, ss);
				}
			}
			ss = block_sum(ss, red);
			const float scale = 1.0f / sqrtf(ss / n + eps);
#pragma unroll
			for (int k = 0; k < SV_MAX; ++k) {
				v[k].x = (v[k].x - mean) * scale * w[k].x, v[k].y = (v[k].y - mean) * scale * w[k].y;
				v[k].z = (v[k].z - mean) * scale * w[k].z, v[k].w = (v[k].w - mean) * scale * w[k].w;
			}
		} else {
			rms = true;
			float ss = 0.f;
#pragma unroll
			for (int k = 0; k < SV_MAX; ++k) {
				ss = fmaf(v[k].x, v[k].x, ss), ss = fmaf(v[k].y, v[k].y, ss), ss = fmaf(v[k].z, v[k].z, ss), ss = fmaf(v[k].w, v[k].w, ss);
				v[k].x *= w[k].x, v[k].y *= w[k].y, v[k].z *= w[k].z, v[k].w *= w[k].w;
			}
			ss = warp_sum(ss);
			if ((tid & 31) == 0) red[tid >> 5] = ss;
		}
	}
#pragma unroll
	for (int k = 0; k < SV_MAX; ++k) {
		int i = tid + k * nthr;
		if (i < n4) {
			if (xb_out && !rms) reinterpret_cast<float4*>(xb_out)[i] = v[k];
			*reinterpret_cast<float4*>(xs + xs_index<DBITS>(4 * i)) = v[k]; // 4 consecutive elements stay consecutive
		}
		if (DBITS == 4) { // gf4: 3 * (sum of the group of 8) behind the vector; threads i, i ^ 1 hold the two halves of a group (nthr is even)
			const float h = i < n4 ? (v[k].x + v[k].y) + (v[k].z + v[k].w) : 0.f;
			const float o = __shfl_xor_sync(0xffffffffu, h, 1);
			if (!(i & 1) && i < n4) xs[total4 * 4 + (i >> 1)] = 3.f * (h + o);
		}
	}
	for (int i = n4 + tid; i < total4; i += nthr) *reinterpret_cast<float4*>(xs + xs_index<DBITS>(4 * i)) = make_float4(0.f, 0.f, 0.f, 0.f);
	if (DBITS == 4)
		for (int gi = (n4 >> 1) + tid; gi < (total4 >> 1); gi += nthr) xs[total4 * 4 + gi] = 0.f;
	__syncthreads();
	if (rms) {
		const int lane = tid & 31, nwarps = (nthr + 31) >> 5;
		const float ss = warp_sum(lane < nwarps ? red[lane] : 0.f);
		post = 1.0f / sqrtf(ss / n + eps);
		if (xb_out) { // the normalised vector itself (norm_par: the FFN reuses it)
#pragma unroll
			for (int k = 0; k < SV_MAX; ++k) {
				int i = tid + k * nthr;
				if (i < n4) reinterpret_cast<float4*>(xb_out)[i] = make_float4(v[k].x * post, v[k].y * post, v[k].z * post, v[k].w * post);
			}
		}
	}
	return post;
}

// Stage an activation vector into shared memory in the permuted layout of common.cuh, optionally
// applying RMSNorm / LayerNorm-without-bias (reference infer.c:183-207: mean only when ln, variance around the
// mean, eps inside the sqrt, then * weight).  Ends with a __syncthreads().  Returns the factor the caller must
// multiply its dot products by (1 unless the RMS scale was left for the epilogue, see stage_vector_batched).
// Every thread requests all of its elements (16-byte loads, up to SV_MAX per thread) before it touches the
// first one, so staging costs one L2 round trip instead of one per element.
template <int DBITS, int SV_MAX = 8>
__device__ __forceinline__ float stage_vector(float* xs, float* red, const float* __restrict__ x, int n, const float* __restrict__ normw, float eps, bool ln,
                                              float* xb_out) {
	const int tid = threadIdx.x, nthr = blockDim.x;
	const int n4 = n >> 2; // n is a multiple of 32
	if (SV_MAX > 4 && n4 <= nthr * 4) // the common case (dim 4096, 256 threads): half the registers
		return stage_vector_batched<DBITS, 4>(xs, red, x, n, normw, eps, ln, xb_out);
	if (n4 <= nthr * SV_MAX) return stage_vector_batched<DBITS, SV_MAX>(xs, red, x, n, normw, eps, ln, xb_out);
	// long vectors: same thing, element by element (two reads of x when normalising)
	float mean = 0.f, scale = 1.f;
	if (normw) {
		if (ln) {
			float s = 0.f;
			for (int j = tid; j < n; j += nthr) s += __ldcg(x + j);
			mean = block_sum(s, red) / n;
		}
		float ss = 0.f;
		for (int j = tid; j < n; j += nthr) {
			float d = __ldcg(x + j) - mean;
			ss = fmaf(d, d, ss);
		}
		ss = block_sum(ss, red);
		scale = 1.0f / sqrtf(ss / n + eps);
	}
	const int total = xs_floats<DBITS>(n);
	for (int j = tid; j < total; j += nthr) {
		float v = 0.f;
		if (j < n) {
			v = __ldcg(x + j);
			if (normw) v = (v - mean) * scale * normw[j];
			if (xb_out) xb_out[j] = v;
		}
		xs[xs_index<DBITS>(j)] = v;
	}
	__syncthreads();
	if (DBITS == 4) { // group sums, same association as the batched path
		for (int gi = tid; gi < (total >> 3); gi += nthr) {
			float e[8];
#pragma unroll
			for (int k = 0; k < 8; ++k) e[k] = xs[xs_index<DBITS>(8 * gi + k)];
			xs[total + gi] = 3.f * (((e[0] + e[1]) + (e[2] + e[3])) + ((e[4] + e[5]) + (e[6] + e[7])));
		}
		__syncthreads();
	}
	return 1.f;
}

__device__ __forceinline__ float act_silu(float x) { // reference infer.c:273-275
	return x / (1.0f + expf(-x));
}
__device__ __forceinline__ float act_gelu(float x) { // reference infer.c:269-271
	return 0.5f * x * (1.0f + tanhf(0.797885f * (x + 0.044715f * x * x * x)));
}

// ------------------------------------------------------------------------------------------------
// k_embed: x = decode(E[token]) (reference infer.c:335-347, infer.cu:142-148), and -- in the extra
// blocks -- the attention-sink re-rotation by one RoPE step for every layer once the cache has rolled
// over (reference infer.c:384-394, infer.cu:150-180).

template <typename KVT>
struct EmbedArgs {
	float* x;
	const void* table;
	const TokenParams* tp;
	int dim;
	int embed_blocks;
	float2* rope_cs;           // [head_dim / 2]: (cos, sin)(pos * freq) of this token, written here for every layer's k_qkv
	unsigned long long* stamp; // perf_cuda: {min start, max end} of this launch, or NULL
	unsigned long long* stamp_reset; // perf_cuda: all slots of the token, re-armed here
	int n_stamps;
	// sinks
	KVT* key_cache;
	const float* rope_freq;
	int n_layers, n_kv_heads, head_dim, seq_len;
};

template <int DBITS, typename KVT>
__global__ void k_embed(const EmbedArgs<KVT> a) {
	pdl_enter();
	if (a.stamp_reset) { // grid-stride: (start, end) = (max, 0); every later kernel of the token waits for this grid
		for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.n_stamps; j += gridDim.x * blockDim.x) a.stamp_reset[2 * j] = ~0ull, a.stamp_reset[2 * j + 1] = 0ull;
	}
	if ((int)blockIdx.x < a.embed_blocks) {
		int i = blockIdx.x * blockDim.x + threadIdx.x;
		if (i < a.dim) a.x[i] = weight_at<DBITS>(a.table, (size_t)a.tp->token * a.dim + i);
		if (blockIdx.x == 0 && (int)threadIdx.x < a.head_dim / 2) { // RoPE angles (reference infer.c:223-236), once per token instead of once per row pair
			float fcr, fci;
			sincosf((float)a.tp->pos * a.rope_freq[threadIdx.x], &fci, &fcr);
			a.rope_cs[threadIdx.x] = make_float2(fcr, fci);
		}
		return;
	}
	const int kv_sink = a.tp->kv_sink;
	if (kv_sink == 0) return;
	const int kv_dim = a.n_kv_heads * a.head_dim;
	const int pairs = a.n_layers * kv_sink * (kv_dim / 2);
	for (int i = (blockIdx.x - a.embed_blocks) * blockDim.x + threadIdx.x; i < pairs; i += (gridDim.x - a.embed_blocks) * blockDim.x) {
		int k = (i % (kv_dim / 2)) * 2;
		int r = (i / (kv_dim / 2)) % kv_sink;
		int l = i / (kv_dim / 2) / kv_sink;
		int h = k / a.head_dim, d = k % a.head_dim;
		KVT* p = a.key_cache + (((size_t)l * a.n_kv_heads + h) * a.seq_len + r) * a.head_dim + d;
		float fcr, fci;
		sincosf(a.rope_freq[d >> 1], &fci, &fcr); // one position step
		float v0 = kv_load(p), v1 = kv_load(p + 1);
		kv_store(p, v0 * fcr - v1 * fci);
		kv_store(p + 1, v0 * fci + v1 * fcr);
	}
}

// ------------------------------------------------------------------------------------------------
// k_qkv

template <typename KVT>
struct QkvArgs {
	const float* x;
	const float* normw;
	const void* wq;
	const void* wk;
	const void* wv;
	const float* bias;
	float* q_out;
	KVT* kc; // this layer: [n_kv_heads][seq_len][head_dim]
	KVT* vc;
	const float2* rope_cs;  // [head_dim/2]: (cos, sin) of pos * theta^(-j/rotary_dim) (angle 0 beyond rotary_dim), from k_embed
	float* xb_out;          // normalised x for the FFN when norm_par, else NULL
	const TokenParams* tp;
	int dim, q_dim, kv_dim, head_dim, seq_len;
	float eps, clip;
	int ln;
	unsigned long long* stamp;
};

// Before waiting for the previous kernel a warp asks the L2 for its first row pair (cp.async.bulk.prefetch.L2: no registers;
// weights are immutable, so this is always legal).  (Issuing the first loads into registers instead keeps 32 more registers
// live across the staging, which costs a CTA per SM.)
#define QKV_THREADS 256
// One warp per row pair (the whole 2 x rowbytes pair is requested in one batch), 3 CTAs per SM.  (A one-CTA-per-SM form with
// equal contiguous shares, meant to leave half the register file to an early attention CTA, makes most warps wait for a
// second DRAM round trip.)
template <int DBITS, typename KVT>
__global__ void __launch_bounds__(QKV_THREADS, 3) k_qkv(const QkvArgs<KVT> a) {
	pdl_launch_next();
	extern __shared__ __align__(16) float smem[];
	float* red = smem;
	float* xs = smem + 32;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const int nvec = a.dim / WFmt<DBITS>::VW;
	const size_t rowvecs = (size_t)nvec; // 16-byte vectors per row
	const int npairs = (a.q_dim + 2 * a.kv_dim) / 2;
	auto rows_of = [&](int p, const uint4* (&rp)[2], int& j, int& k) {
		j = 2 * p; // row in the concatenated [wq; wk; wv]
		const void* w;
		if (j < a.q_dim) {
			w = a.wq, k = j;
		} else if (j < a.q_dim + a.kv_dim) {
			w = a.wk, k = j - a.q_dim;
		} else {
			w = a.wv, k = j - a.q_dim - a.kv_dim;
		}
		rp[0] = reinterpret_cast<const uint4*>(w) + (size_t)k * rowvecs, rp[1] = rp[0] + rowvecs;
	};
	// weights first: they do not depend on the previous kernel, so their latency hides its tail and the staging of x
	const int p0 = blockIdx.x * nwarps + warp;
	if (p0 < npairs && lane == 0) {
		const uint4* rp[2];
		int j, k;
		rows_of(p0, rp, j, k);
		l2_prefetch_row(rp[0], nvec * 16), l2_prefetch_row(rp[1], nvec * 16);
	}
	pdl_wait_prev();
	stamp_begin(a.stamp);
	const float post = stage_vector<DBITS>(xs, red, a.x, a.dim, a.normw, a.eps, a.ln != 0, blockIdx.x == 0 ? a.xb_out : nullptr);
	const int kv_pos = a.tp->kv_pos;

	for (int p = p0; p < npairs; p += gridDim.x * nwarps) {
		const uint4* rp[2];
		int j, k;
		rows_of(p, rp, j, k);
		float v[2];
		warp_dot_rows<DBITS, 2, 4>(rp, nvec, reinterpret_cast<const float4*>(xs), v);

		if (lane == 0) {
			float v0 = v[0] * post, v1 = v[1] * post;
			if (a.bias) v0 += a.bias[j], v1 += a.bias[j + 1];
			v0 = fminf(fmaxf(v0, -a.clip), a.clip);
			v1 = fminf(fmaxf(v1, -a.clip), a.clip);
			if (j < a.q_dim + a.kv_dim) { // rotate q and k (reference infer.c:223-236); angles from k_embed's table
				const float2 cs = a.rope_cs[(j % a.head_dim) >> 1];
				float r0 = v0 * cs.x - v1 * cs.y, r1 = v0 * cs.y + v1 * cs.x;
				v0 = r0, v1 = r1;
			}
			if (j < a.q_dim) {
				a.q_out[k] = v0, a.q_out[k + 1] = v1;
			} else {
				KVT* c = (j < a.q_dim + a.kv_dim) ? a.kc : a.vc;
				int h = k / a.head_dim, d = k % a.head_dim;
				KVT* dst = c + ((size_t)h * a.seq_len + kv_pos) * a.head_dim + d;
				kv_store(dst, v0);
				kv_store(dst + 1, v1);
			}
		}
	}
	stamp_end(a.stamp);
}

// ------------------------------------------------------------------------------------------------
// Attention (flash-decoding).  Work item = (unit, slice): a unit is one kv head together with a group of
// HG query heads that share it (so K and V are read once for all of them), a slice is a contiguous range
// of cached positions.  A group of LPP lanes owns one position at a time (8 head dims per lane: one
// 16-byte load of K and one of V); P positions per group are in flight and the next P are requested
// before the current ones are consumed.  Scores are scaled by 1/sqrt(head_dim) after the dot (reference
// infer.c:246), the softmax is the max-shifted one of infer.c:252-258 evaluated online, and 1/sum is
// applied once at the end.  Slices are merged through global partials (m, l, acc[head_dim]) by the last
// CTA of the unit to arrive, in two passes whose loads are all independent.

struct AttnArgs {
	const float* q;   // [n_heads*head_dim] rotated queries
	const void* kc;   // this layer
	const void* vc;
	float* partial;   // [units][nsplit][HG][head_dim + 2]
	unsigned* counter; // [units], zero between launches
	float* out;       // [n_heads*head_dim]
	const TokenParams* tp;
	int head_dim, seq_len, nsplit, lpp; // lpp: lanes per position (power of two >= head_dim/8)
	int kv_mul, qgroups;                // query heads per kv head; qgroups = kv_mul / HG
	float inv_sqrt_hd;
	int nbmax;                          // k_attn2: 16-position blocks per CTA = ceil(ceil(seq_len / 16) / nsplit)
	unsigned long long* cells;          // k_attn2: [units][nsplit][HG][head_dim + 2] {value, epoch} cells of the slice fold
	unsigned epoch_stride, epoch_idx;   // epoch = tp_seq * stride + idx (unique per token and layer, never 0)
	int* err;                           // mapped host word for the fold's watchdog
	unsigned long long* dbg;            // perf: 16 timestamps of CTA 0 / extremes over CTAs (first layer only), or NULL
	unsigned long long* stamp;
};

template <typename KVT>
struct KvRaw;
template <>
struct KvRaw<__half> {
	typedef uint4 type; // 8 halves
	static __device__ __forceinline__ uint4 load(const __half* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
	static __device__ __forceinline__ uint4 zero() { return make_uint4(0, 0, 0, 0); }
	static __device__ __forceinline__ void unpack(const uint4& r, float (&o)[8]) {
		float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
		float2 c = __half22float2(*reinterpret_cast<const __half2*>(&r.z)), d = __half22float2(*reinterpret_cast<const __half2*>(&r.w));
		o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y, o[4] = c.x, o[5] = c.y, o[6] = d.x, o[7] = d.y;
	}
};
template <>
struct KvRaw<uint8_t> {
	typedef uint2 type; // 8 e5m2 bytes
	static __device__ __forceinline__ uint2 load(const uint8_t* p) { return __ldcg(reinterpret_cast<const uint2*>(p)); }
	static __device__ __forceinline__ uint2 zero() { return make_uint2(0, 0); }
	static __device__ __forceinline__ void unpack(const uint2& r, float (&o)[8]) {
		float2 a = e5m2x2_lo(r.x), b = e5m2x2_hi(r.x), c = e5m2x2_lo(r.y), d = e5m2x2_hi(r.y);
		o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y, o[4] = c.x, o[5] = c.y, o[6] = d.x, o[7] = d.y;
	}
};

// After the position loop of a work item: merge the lane groups of a warp and the warps of the CTA (shared memory) into ONE
// record (m, l, acc) per head, written to `dst` [HG][head_dim + 2] (the slice's global partial, or shared memory).
// m / l / acc: per-lane state of this warp's HH heads (8 head dims per lane, li = lane % lpp).
template <int HH>
__device__ __forceinline__ void attn_cta_merge(const AttnArgs& a, int HG, int h0, int nh, int warp, int nwarps, float (&m)[HH], float (&l)[HH], float (&acc)[HH][8],
                                               float* scratch, float* dst) {
	const int lane = threadIdx.x & 31;
	const int hd = a.head_dim, lpp = a.lpp;
	const int grp = lane / lpp, li = lane % lpp;
	const bool dact = li * 8 < hd;
	// merge the position groups of a warp
	for (int o = lpp; o < 32; o <<= 1) {
#pragma unroll
		for (int h = 0; h < HH; ++h) {
			float mo = __shfl_xor_sync(0xffffffffu, m[h], o), lo = __shfl_xor_sync(0xffffffffu, l[h], o);
			float mn = fmaxf(m[h], mo);
			float ca = expf(m[h] - mn), cb = expf(mo - mn);
			l[h] = l[h] * ca + lo * cb;
#pragma unroll
			for (int e = 0; e < 8; ++e) {
				float ao = __shfl_xor_sync(0xffffffffu, acc[h][e], o);
				acc[h][e] = acc[h][e] * ca + ao * cb;
			}
			m[h] = mn;
		}
	}

	// merge warps through shared memory: rec[warp][h][hd+2]
	const int rec = hd + 2;
	__syncthreads(); // scratch may still be in use by a previous item
	if (grp == 0) {
#pragma unroll
		for (int h = 0; h < HH; ++h) {
			if (h < nh) { // the warp sets write disjoint heads
				float* r = scratch + ((size_t)warp * HG + h0 + h) * rec;
				if (dact) {
#pragma unroll
					for (int e = 0; e < 8; ++e) r[li * 8 + e] = acc[h][e];
				}
				if (li == 0) r[hd] = m[h], r[hd + 1] = l[h];
			}
		}
	}
	__syncthreads();
	// per (warp, head) rescaling coefficients once (nwarps * HG exponentials instead of nwarps per element)
	__shared__ float s_coef[16][8], s_mn[8];
	if ((int)threadIdx.x < nwarps * HG) {
		const int w = threadIdx.x / HG, h = threadIdx.x % HG;
		float mn = -FLT_MAX;
		for (int w2 = 0; w2 < nwarps; ++w2) mn = fmaxf(mn, scratch[((size_t)w2 * HG + h) * rec + hd]);
		s_coef[w][h] = expf(scratch[((size_t)w * HG + h) * rec + hd] - mn);
		if (w == 0) s_mn[h] = mn;
	}
	__syncthreads();
	for (int idx = threadIdx.x; idx < HG * rec; idx += blockDim.x) {
		int h = idx / rec, e = idx % rec;
		float v;
		if (e == hd) {
			v = s_mn[h];
		} else {
			v = 0.f;
			for (int w = 0; w < nwarps; ++w) v = fmaf(scratch[((size_t)w * HG + h) * rec + e], s_coef[w][h], v); // e == hd+1 merges the sums the same way
		}
		dst[idx] = v;
	}
}

// attn_cta_merge into the slice's global partial, then the last slice of the unit to arrive folds all slices into the
// normalised output (two passes, all loads independent; deterministic).
template <int HH>
__device__ __forceinline__ void attn_tail(const AttnArgs& a, int HG, int unit, int split, int hbase, int h0, int nh, int warp, int nwarps, float (&m)[HH], float (&l)[HH],
                                          float (&acc)[HH][8], float* scratch, int* flag) {
	const int hd = a.head_dim, rec = hd + 2;
	attn_cta_merge<HH>(a, HG, h0, nh, warp, nwarps, m, l, acc, scratch, a.partial + ((size_t)unit * a.nsplit + split) * HG * rec);

	// the last slice of this unit to finish folds all slices and writes the normalised output
	__threadfence();
	__syncthreads();
	if (threadIdx.x == 0) {
		unsigned old = atomicAdd(a.counter + unit, 1u);
		*flag = (old == (unsigned)a.nsplit - 1);
	}
	__syncthreads();
	if (!*flag) return;
	__threadfence();
	const int ns = a.nsplit;
	const float* pk = a.partial + (size_t)unit * ns * HG * rec;
	float* coef = scratch;                  // [ns][HG]: l_s, then exp(m_s - M)
	float* msv = scratch + (size_t)ns * HG; // [ns][HG]: m_s; msv[ns*HG + h]: 1 / L_h
	for (int i = threadIdx.x; i < ns * HG; i += blockDim.x) {
		const float* r = pk + (size_t)i * rec; // i = s * HG + h
		coef[i] = __ldcg(r + hd + 1);
		msv[i] = __ldcg(r + hd);
	}
	__syncthreads();
	if ((int)threadIdx.x < HG) {
		const int h = threadIdx.x;
		float M = -FLT_MAX;
		for (int s_ = 0; s_ < ns; ++s_) M = fmaxf(M, msv[s_ * HG + h]);
		float L = 0.f;
		for (int s_ = 0; s_ < ns; ++s_) {
			float c = expf(msv[s_ * HG + h] - M);
			L = fmaf(coef[s_ * HG + h], c, L);
			coef[s_ * HG + h] = c;
		}
		msv[h] = 1.0f / L; // msv[0..HG) is dead by now (each thread only read its own column... see sync below)
	}
	__syncthreads();
	for (int idx = threadIdx.x; idx < HG * hd; idx += blockDim.x) {
		int h = idx / hd, e = idx % hd;
		float n0 = 0.f, n1 = 0.f, n2 = 0.f, n3 = 0.f;
		int s_ = 0;
		for (; s_ + 4 <= ns; s_ += 4) {
			float p0 = __ldcg(pk + ((size_t)(s_ + 0) * HG + h) * rec + e), p1 = __ldcg(pk + ((size_t)(s_ + 1) * HG + h) * rec + e);
			float p2 = __ldcg(pk + ((size_t)(s_ + 2) * HG + h) * rec + e), p3 = __ldcg(pk + ((size_t)(s_ + 3) * HG + h) * rec + e);
			n0 = fmaf(p0, coef[(s_ + 0) * HG + h], n0), n1 = fmaf(p1, coef[(s_ + 1) * HG + h], n1);
			n2 = fmaf(p2, coef[(s_ + 2) * HG + h], n2), n3 = fmaf(p3, coef[(s_ + 3) * HG + h], n3);
		}
		for (; s_ < ns; ++s_) n0 = fmaf(__ldcg(pk + ((size_t)s_ * HG + h) * rec + e), coef[s_ * HG + h], n0);
		__stcg(a.out + (size_t)(hbase + h) * hd + e, ((n0 + n1) + (n2 + n3)) * msv[h]);
	}
	if (threadIdx.x == 0) a.counter[unit] = 0;
}

// One work item, executed by all warps of the calling CTA.  Every warp walks its share of the slice's positions
// for HH of the unit's HG query heads.  P positions per lane group are in flight, and the next P are requested
// before the current ones are consumed.
// LPPC > 0 (compile-time lanes per position, with HH * P == LPPC) selects the transposing score path: the
// HH * P partial dot products of a step are reduced across the lane group so that every lane ends up with
// ONE complete score (15 shuffles instead of 64 for 16 lanes), evaluates its two exponentials once, and
// the probabilities are broadcast back for the value accumulation.
// scratch: shared, >= max(nwarps * HG * (hd + 2), 2 * nsplit * HG) floats.  flag: shared int.
template <typename KVT, int HH, int P, int LPPC = 0>
__device__ __forceinline__ void attn_item(const AttnArgs& a, int HG, int unit, int split, int kv_len, float* scratch, int* flag) {
	typedef typename KvRaw<KVT>::type raw_t;
	const int kvh = unit / a.qgroups;
	const int hbase = kvh * a.kv_mul + (unit % a.qgroups) * HG; // first query head of this unit
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const int nh = min(HH, HG); // heads this warp really has
	const int hd = a.head_dim, lpp = a.lpp;
	const int G = 32 / lpp; // position groups per warp
	const int grp = lane / lpp, li = lane % lpp;
	const bool dact = li * 8 < hd; // lane holds real head dims

	const int chunk = (kv_len + a.nsplit - 1) / a.nsplit;
	const int t0 = split * chunk, t1 = min(kv_len, t0 + chunk);

	const KVT* kbase = reinterpret_cast<const KVT*>(a.kc) + (size_t)kvh * a.seq_len * hd + li * 8;
	const KVT* vbase = reinterpret_cast<const KVT*>(a.vc) + (size_t)kvh * a.seq_len * hd + li * 8;

	float qr[HH][8], acc[HH][8], m[HH], l[HH];
#pragma unroll
	for (int h = 0; h < HH; ++h) {
		m[h] = -FLT_MAX, l[h] = 0.f;
#pragma unroll
		for (int d = 0; d < 8; ++d) {
			acc[h][d] = 0.f;
			qr[h][d] = (dact && h < nh) ? __ldcg(a.q + (size_t)(hbase + h) * hd + li * 8 + d) : 0.f;
		}
	}

	const int stride = nwarps * G; // positions per step over all groups of the CTA
	auto fetch = [&](int tw, raw_t (&kr)[P], raw_t (&vr)[P]) {
#pragma unroll
		for (int i = 0; i < P; ++i) {
			int t = tw + grp + i * stride;
			bool ok = t < t1 && dact;
			kr[i] = ok ? KvRaw<KVT>::load(kbase + (size_t)t * hd) : KvRaw<KVT>::zero();
			vr[i] = ok ? KvRaw<KVT>::load(vbase + (size_t)t * hd) : KvRaw<KVT>::zero();
		}
	};
	float mh = -FLT_MAX, lh = 0.f; // transposing path: running max / sum of THIS lane's head (li / P)
	auto update = [&](int tw, const raw_t (&kr)[P], const raw_t (&vr)[P]) {
		float kf[P][8], vf[P][8];
		bool ok[P];
#pragma unroll
		for (int i = 0; i < P; ++i) {
			ok[i] = tw + grp + i * stride < t1;
			KvRaw<KVT>::unpack(kr[i], kf[i]);
			KvRaw<KVT>::unpack(vr[i], vf[i]);
		}
		if constexpr (LPPC > 0) {
			constexpr int NC = HH * P; // scores per step; lane li ends up owning combo li % NC
			static_assert(LPPC == 0 || (NC <= LPPC && LPPC % NC == 0), "combos must divide the lane group");
			float part[NC]; // combo c = h * P + i
#pragma unroll
			for (int h = 0; h < HH; ++h)
#pragma unroll
				for (int i = 0; i < P; ++i) {
					float d = 0.f;
#pragma unroll
					for (int e = 0; e < 8; ++e) d = fmaf(qr[h][e], kf[i][e], d);
					part[h * P + i] = d;
				}
			// more lanes than combos: plain butterfly first
#pragma unroll
			for (int s_ = LPPC / 2; s_ >= NC; s_ >>= 1) {
#pragma unroll
				for (int k = 0; k < NC; ++k) part[k] += __shfl_xor_sync(0xffffffffu, part[k], s_);
			}
			// transposing reduction: after the step with stride s a lane keeps the half of its values selected by bit s
#pragma unroll
			for (int s_ = NC / 2; s_ >= 1; s_ >>= 1) {
				const bool up = li & s_;
#pragma unroll
				for (int k = 0; k < s_; ++k) {
					float send = up ? part[k] : part[k + s_];
					float recv = __shfl_xor_sync(0xffffffffu, send, s_);
					part[k] = (up ? part[k + s_] : part[k]) + recv;
				}
			}
			// lane li now owns combo c = li % NC: head c / P, position c % P
			const bool valid = tw + grp + (li % P) * stride < t1;
			const float sc = valid ? part[0] * a.inv_sqrt_hd : -FLT_MAX;
			float gmax = sc;
#pragma unroll
			for (int o = 1; o < P; o <<= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o));
			const float mnew = fmaxf(mh, gmax);
			const float corr = __expf(mh - mnew);
			const float pr = valid ? __expf(sc - mnew) : 0.f;
			float ps = pr;
#pragma unroll
			for (int o = 1; o < P; o <<= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o);
			lh = fmaf(lh, corr, ps);
			mh = mnew;
			const int gbase = grp * LPPC;
#pragma unroll
			for (int h = 0; h < HH; ++h) {
				const float ch = __shfl_sync(0xffffffffu, corr, gbase + h * P);
				float pw[P];
#pragma unroll
				for (int i = 0; i < P; ++i) pw[i] = __shfl_sync(0xffffffffu, pr, gbase + h * P + i);
#pragma unroll
				for (int e = 0; e < 8; ++e) {
					float v = acc[h][e] * ch;
#pragma unroll
					for (int i = 0; i < P; ++i) v = fmaf(pw[i], vf[i][e], v);
					acc[h][e] = v;
				}
			}
			(void)ok;
			return;
		}
#pragma unroll
		for (int h = 0; h < HH; ++h) {
			float sc[P], smax = m[h];
#pragma unroll
			for (int i = 0; i < P; ++i) {
				float d = 0.f;
#pragma unroll
				for (int e = 0; e < 8; ++e) d = fmaf(qr[h][e], kf[i][e], d);
				for (int o = 1; o < lpp; o <<= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
				sc[i] = ok[i] ? d * a.inv_sqrt_hd : -FLT_MAX;
				smax = fmaxf(smax, sc[i]);
			}
			float corr = expf(m[h] - smax);
			m[h] = smax;
			float pw[P], ps = 0.f;
#pragma unroll
			for (int i = 0; i < P; ++i) {
				pw[i] = ok[i] ? expf(sc[i] - smax) : 0.f;
				ps += pw[i];
			}
			l[h] = fmaf(l[h], corr, ps);
#pragma unroll
			for (int e = 0; e < 8; ++e) {
				float v = acc[h][e] * corr;
#pragma unroll
				for (int i = 0; i < P; ++i) v = fmaf(pw[i], vf[i][e], v);
				acc[h][e] = v;
			}
		}
	};

	// software pipeline over steps of stride * P positions (warp-uniform trip count: the shuffles above are full-warp)
	raw_t ka[P], va[P], kb[P], vb[P];
	const int step = stride * P;
	int tw = t0 + warp * G;
	if (tw < t1) fetch(tw, ka, va);
	while (tw < t1) {
		if (tw + step < t1) fetch(tw + step, kb, vb);
		update(tw, ka, va);
		tw += step;
		if (tw >= t1) break;
		if (tw + step < t1) fetch(tw + step, ka, va);
		update(tw, kb, vb);
		tw += step;
	}

	if constexpr (LPPC > 0) { // running max / sum live in the lanes that own the head: hand them to every lane of the group
#pragma unroll
		for (int h = 0; h < HH; ++h) {
			m[h] = __shfl_sync(0xffffffffu, mh, grp * LPPC + h * P);
			l[h] = __shfl_sync(0xffffffffu, lh, grp * LPPC + h * P);
		}
	}

	attn_tail<HH>(a, HG, unit, split, hbase, 0, nh, warp, nwarps, m, l, acc, scratch, flag);
}

#define ATTN_THREADS 256
template <typename KVT, int HG>
__global__ void __launch_bounds__(ATTN_THREADS) k_attn(__grid_constant__ const AttnArgs a) {
	pdl_enter();
	stamp_begin(a.stamp);
	extern __shared__ __align__(16) float smem[];
	__shared__ int flag;
	const int unit = blockIdx.x / a.nsplit, split = blockIdx.x % a.nsplit, kv_len = a.tp->kv_len;
	// transposing score path when the lanes of a position are a small multiple of the heads (head_dim 128 / 64)
	bool done = false;
	if constexpr (HG == 2 || HG == 4 || HG == 8) {
		if (a.lpp == 16 && HG >= 4) {
			attn_item<KVT, HG, 16 / HG, 16>(a, HG, unit, split, kv_len, smem, &flag);
			done = true;
		} else if (a.lpp == 8) {
			attn_item<KVT, HG, 8 / HG, 8>(a, HG, unit, split, kv_len, smem, &flag);
			done = true;
		}
	}
	if (!done) attn_item<KVT, HG, (HG > 4 ? 2 : 4)>(a, HG, unit, split, kv_len, smem, &flag);
	stamp_end(a.stamp);
}

// ------------------------------------------------------------------------------------------------
// Tensor parallelism: matvec -> all-reduce in ONE kernel over NVLink peer memory (one-shot push, flag-in-data).
// Every rank owns an exchange area that all peers map (cudaIpc): cell[slot][src rank][row] = {partial, epoch}, 8 bytes.
// CTA b of rank r computes the partial of its rows and stores {value, epoch} cells into slot (epoch & 1) of every
// PEER's area -- one 128-byte line per 16 rows, each cell a single 8-byte store, so a reader that sees the epoch
// sees the value: no fence, no separate flag, one NVLink one-way latency.  It then polls its own area for the cells
// CTA b of every peer pushes (same rows: the grids are equal) and adds the partials in rank order, so all ranks end
// up with bit-identical residual vectors.  A CTA pushes before it polls and the grid is co-resident, so ranks cannot
// deadlock; two slots suffice because a rank reaches epoch e+2 only after it has consumed every peer's cells of
// e+1, i.e. after every peer has finished its whole epoch-e kernel.  Replaces an NCCL kernel + an add kernel.

#define TP_MAX_WORLD 8
#define TP_MAX_ITERS 16

struct TpExchange {
	int world, rank;
	unsigned idx, stride;      // epoch = tp_seq * stride + idx  (> 0; the areas start zeroed)
	const TokenParams* tp;
	uint2* cell[TP_MAX_WORLD]; // rank p's area  [2][world][d]
	int* err;                  // mapped host word: watchdog code
};

// part[it * 16 + k]: row 2 * ((it * gridDim.x + blockIdx.x) * 8) + k of this rank's partial.  All 256 threads call.
__device__ __forceinline__ void tp_exchange_add(const TpExchange& t, const float* part, int niter, float* y, int d) {
	const unsigned epoch = (unsigned)t.tp->tp_seq * t.stride + t.idx;
	const int slot = epoch & 1;
	const int W = t.world;
	__syncthreads(); // part[] complete
	const int cells = niter * 16;
	for (int i = threadIdx.x; i < cells * (W - 1); i += blockDim.x) {
		int peer = i / cells;
		const int j = i - peer * cells;
		peer += peer >= t.rank; // skip self
		const int row = 2 * (((j >> 4) * gridDim.x + blockIdx.x) * 8) + (j & 15);
		if (row < d) {
			uint2* dst = t.cell[peer] + ((size_t)slot * W + t.rank) * d + row;
			// ONE 64-bit store: a reader that sees the epoch word sees the value word (a .v2 access is two scalar accesses to the memory model)
			const unsigned long long cell = ((unsigned long long)epoch << 32) | __float_as_uint(part[j]);
			asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(dst), "l"(cell) : "memory");
		}
	}
	for (int j = threadIdx.x; j < cells; j += blockDim.x) {
		const int row = 2 * (((j >> 4) * gridDim.x + blockIdx.x) * 8) + (j & 15);
		if (row >= d) continue;
		const uint2* base = t.cell[t.rank] + (size_t)slot * W * d + row;
		float sum = 0.f;
		for (int p = 0; p < W; ++p) { // rank order: identical on every rank
			if (p == t.rank) {
				sum += part[j];
				continue;
			}
			unsigned vx, spins = 0;
			unsigned long long t0 = 0;
			for (;;) {
				unsigned long long cell;
				asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(cell) : "l"(base + (size_t)p * d) : "memory");
				vx = (unsigned)cell;
				if ((unsigned)(cell >> 32) == epoch) break;
				if ((++spins & 1023) == 0) {
					unsigned long long now;
					asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
					if (!t0) t0 = now;
					if (now - t0 > 20000000000ull) { // 20 s: a peer died or the ranks diverged -- fail loudly, never hang the GPU
						if (t.err) *reinterpret_cast<volatile int*>(t.err) = 9000 + p;
						__threadfence_system();
						__trap();
					}
				}
			}
			sum += __uint_as_float(vx);
		}
		y[row] += sum;
	}
}

// The same exchange for a CTA that owns the CONTIGUOUS rows [row0, row0 + nrows) (ring-fed kernels): part[j] = this rank's partial
// of row row0 + j.  Cells are indexed by row, so the two forms interoperate with any row-to-CTA mapping as long as every rank
// pushes every row once.  All threads of the CTA call; the grid must be co-resident (it is: at most one or two CTAs per SM).
__device__ __forceinline__ void tp_exchange_rows(const TpExchange& t, const float* part, int row0, int nrows, float* y, int d) {
	const unsigned epoch = (unsigned)t.tp->tp_seq * t.stride + t.idx;
	const int slot = epoch & 1, W = t.world;
	__syncthreads(); // part[] complete
	for (int i = threadIdx.x; i < nrows * (W - 1); i += blockDim.x) {
		int peer = i / nrows;
		const int j = i - peer * nrows;
		peer += peer >= t.rank; // skip self
		const unsigned long long cell = ((unsigned long long)epoch << 32) | __float_as_uint(part[j]);
		asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(t.cell[peer] + ((size_t)slot * W + t.rank) * d + row0 + j), "l"(cell) : "memory");
	}
	for (int j = threadIdx.x; j < nrows; j += blockDim.x) {
		const uint2* base = t.cell[t.rank] + (size_t)slot * W * d + row0 + j;
		float sum = 0.f;
		for (int p = 0; p < W; ++p) { // rank order: identical on every rank
			if (p == t.rank) {
				sum += part[j];
				continue;
			}
			unsigned spins = 0;
			unsigned long long t0 = 0, cell;
			for (;;) {
				asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(cell) : "l"(base + (size_t)p * d) : "memory");
				if ((unsigned)(cell >> 32) == epoch) break;
				if ((++spins & 1023) == 0) {
					unsigned long long now;
					asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
					if (!t0) t0 = now;
					if (now - t0 > 20000000000ull) {
						if (t.err) *reinterpret_cast<volatile int*>(t.err) = 9000 + p;
						__threadfence_system();
						__trap();
					}
				}
			}
			sum += __uint_as_float((unsigned)cell);
		}
		y[row0 + j] += sum;
	}
}

// ------------------------------------------------------------------------------------------------
// k_matres: y[row] (+)= sum_e weight_e * (W_e[row] . xin_e)   -- wo (+ residual, infer.c:410-415) and
// w2 (* router weight, + residual, infer.c:452-456).  Experts are visited in selection order by the
// same lane, so the sum is deterministic (the reference CUDA path uses atomicAdd, infer.cu:618).

struct MatResArgs {
	const float* xin; // [nact][n]
	const void* w;    // [n_experts?][d][n]
	float* y;         // [d]
	const MoeSel* sel; // NULL: one pass with expert 0, weight 1
	int n, d, nact;
	int accumulate;   // 1: y += ..., 0: y = ...
	TpExchange tpx;   // world > 1: the partial is summed over the tensor-parallel ranks inside this kernel
	unsigned long long* stamp;
	int S;            // k_matres_ring: chunks per task, i.e. per K-slice of a row pair (k_matres reads whole rows)
};

template <int DBITS>
__global__ void __launch_bounds__(256, 2) k_matres(const MatResArgs a) {
	pdl_launch_next();
	extern __shared__ __align__(16) float smem[];
	__shared__ __align__(16) float tp_part[TP_MAX_ITERS * 16];
	float* red = smem;
	float* xs = smem + 32;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const int nvec = a.n / WFmt<DBITS>::VW;
	const size_t esize = (size_t)a.d * nvec; // 16-byte vectors per expert
	const bool long_rows = nvec >= 32 * 8 && DBITS != 4; // a warp has ONE pair and is latency-bound: 8 KB in flight per warp (wo: the whole pair at once)
	// dense models: request the first row pair before waiting for the previous kernel (the expert of a MoE layer is its result)
	const int p0 = blockIdx.x * nwarps + warp;
	const bool early = a.sel == nullptr && p0 < a.d / 2;
	if (early && lane == 0) {
		const uint4* r0 = reinterpret_cast<const uint4*>(a.w) + (size_t)(2 * p0) * nvec;
		l2_prefetch_row(r0, nvec * 16), l2_prefetch_row(r0 + nvec, nvec * 16);
	}
	pdl_wait_prev();
	stamp_begin(a.stamp);

	for (int e = 0; e < a.nact; ++e) {
		if (e > 0) __syncthreads();
		stage_vector<DBITS, 16>(xs, red, a.xin + (size_t)e * a.n, a.n, nullptr, 0.f, false, nullptr);
		const int ex = a.sel ? a.sel->expert[e] : 0;
		const float ew = a.sel ? a.sel->weight[e] : 1.f;
		const uint4* wb = reinterpret_cast<const uint4*>(a.w) + (size_t)ex * esize;
		int it = 0;
		for (int p = blockIdx.x * nwarps + warp; p < a.d / 2; p += gridDim.x * nwarps, ++it) {
			const uint4* rp[2] = {wb + (size_t)(2 * p) * nvec, wb + (size_t)(2 * p + 1) * nvec};
			float v[2];
			const float4* xs4 = reinterpret_cast<const float4*>(xs);
			if (long_rows)
				warp_dot_rows<DBITS, 2, 8>(rp, nvec, xs4, v);
			else
				warp_dot_rows<DBITS, 2, 4>(rp, nvec, xs4, v);
			if (lane == 0) {
				if (a.tpx.world > 1) { // this rank's partial (router-weighted over the active experts, in selection order): summed over the ranks below
					float* tpp = tp_part + it * 16 + warp * 2;
					tpp[0] = (e ? tpp[0] : 0.f) + v[0] * ew, tpp[1] = (e ? tpp[1] : 0.f) + v[1] * ew;
					continue;
				}
				float2* dst = reinterpret_cast<float2*>(a.y + 2 * p);
				float2 cur = (a.accumulate || e > 0) ? *dst : make_float2(0.f, 0.f);
				cur.x += v[0] * ew;
				cur.y += v[1] * ew;
				*dst = cur;
			}
		}
	}
	if (a.tpx.world > 1) { // blockDim.x == 256, i.e. 16 rows per CTA and iteration
		const int per = gridDim.x * 8;
		tp_exchange_add(a.tpx, tp_part, (a.d / 2 - blockIdx.x * 8 + per - 1) / per, a.y, a.d);
	}
	stamp_end(a.stamp);
}

// ------------------------------------------------------------------------------------------------
// k_ffn_up: hb[e][i] = act(w1_e[i] . xn) * (w3_e[i] . xn) (reference infer.c:437-450), with the
// router evaluated first by every CTA for MoE models (logits = gate . xn, top-k by repeated arg-max
// with strict '>' so the lowest index wins ties, weights = softmax over the selected; infer.c:277-305).

struct FfnUpArgs {
	unsigned long long* stamp;
	const float* x;
	const float* normw; // NULL: stage `x` as is (norm_par: x = saved attention-norm output)
	const void* gate;   // router (n_experts, dim) or NULL
	const void* w1;
	const void* w3;
	float* hb;          // [nact][hidden]
	MoeSel* sel;        // written by CTA 0
	int dim, hidden, n_experts, nact;
	float eps;
	int ln, gelu;
	size_t expert_stride; // 16-byte vectors between experts in w1 / w3 (tensor parallelism: a rank's rows are a slice of every expert)
};

template <int DBITS>
__global__ void __launch_bounds__(256, 3) k_ffn_up(__grid_constant__ const FfnUpArgs a) {
	pdl_launch_next();
	extern __shared__ __align__(16) float smem[];
	__shared__ float glog[64];
	__shared__ MoeSel ssel;
	float* red = smem;
	float* xs = smem + 32;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const int nvec = a.dim / WFmt<DBITS>::VW;
	const float4* xs4 = reinterpret_cast<const float4*>(xs);
	// dense models: the first (w1, w3) row pair is requested before the previous kernel has finished and x is staged
	const int p0 = blockIdx.x * nwarps + warp;
	const bool early = a.n_experts == 0 && p0 < a.hidden;
	if (early && lane == 0) {
		l2_prefetch_row(reinterpret_cast<const uint4*>(a.w1) + (size_t)p0 * nvec, nvec * 16);
		l2_prefetch_row(reinterpret_cast<const uint4*>(a.w3) + (size_t)p0 * nvec, nvec * 16);
	}
	pdl_wait_prev();
	stamp_begin(a.stamp);
	const float post = stage_vector<DBITS>(xs, red, a.x, a.dim, a.normw, a.eps, a.ln != 0, nullptr);

	if (a.n_experts) {
		for (int e = warp; e < a.n_experts; e += nwarps) {
			const uint4* rp[1] = {reinterpret_cast<const uint4*>(a.gate) + (size_t)e * nvec};
			float v[1];
			warp_dot_rows<DBITS, 1>(rp, nvec, xs4, v);
			if (lane == 0) glog[e] = v[0] * post;
		}
		__syncthreads();
		if (threadIdx.x == 0) {
			float mx = -FLT_MAX;
			for (int j = 0; j < a.n_experts; ++j) mx = fmaxf(mx, glog[j]);
			unsigned long long mask = 0;
			float wsum = 0.f;
			for (int k = 0; k < a.nact; ++k) {
				int best = -1;
				for (int j = 0; j < a.n_experts; ++j)
					if (!((mask >> j) & 1ull) && (best < 0 || glog[j] > glog[best])) best = j;
				ssel.expert[k] = best;
				ssel.weight[k] = expf(glog[best] - mx);
				wsum += ssel.weight[k];
				mask |= 1ull << best;
			}
			for (int k = 0; k < a.nact; ++k) ssel.weight[k] /= wsum;
			if (blockIdx.x == 0) *a.sel = ssel;
		}
		__syncthreads();
	}

	const size_t esize = a.expert_stride ? a.expert_stride : (size_t)a.hidden * nvec;
	const int total = a.nact * a.hidden;
	for (int p = blockIdx.x * nwarps + warp; p < total; p += gridDim.x * nwarps) {
		int e = p / a.hidden, i = p % a.hidden;
		size_t off = (a.n_experts ? (size_t)ssel.expert[e] * esize : 0) + (size_t)i * nvec;
		const uint4* rp[2] = {reinterpret_cast<const uint4*>(a.w1) + off, reinterpret_cast<const uint4*>(a.w3) + off};
		float v[2];
		warp_dot_rows<DBITS, 2, 4>(rp, nvec, xs4, v);
		if (lane == 0) {
			const float u1 = v[0] * post, u3 = v[1] * post;
			a.hb[p] = (a.gelu ? act_gelu(u1) : act_silu(u1)) * u3;
		}
	}
	stamp_end(a.stamp);
}

// ------------------------------------------------------------------------------------------------
// k_output: logits = Wcls . norm(x) (reference infer.c:466-469, infer.cu:628-649) written in 128-byte
// pieces (the destination may be pinned host memory), plus per-CTA greedy candidates
// (first maximum wins, reference sampler.c:34-42).

struct OutputArgs {
	const float* x;
	const float* normw;
	const void* wcls;
	float* logits;
	float* cand_val; // [gridDim.x]
	int* cand_idx;
	int dim, vocab;
	float eps;
	int ln;
	unsigned long long* stamp;
	// tensor parallelism (SURVEY.md s.8e: "lm_head: rows split by vocab"): this rank owns classifier rows [row0, row1) and
	// stores its logits and per-CTA greedy candidates straight into EVERY rank's gather area over NVLink (peer[rank] is
	// its own); k_tp_gather then waits for all slices.  world <= 1: rows [0, vocab) into `logits` / `cand_*`.
	int row0, row1, world, rank;
	float* peer_logits[TP_MAX_WORLD];
	float* peer_cand_val[TP_MAX_WORLD]; // [world][gridDim.x]
	int* peer_cand_idx[TP_MAX_WORLD];
};

template <int DBITS>
__global__ void __launch_bounds__(256) k_output(const OutputArgs a) {
	pdl_enter();
	stamp_begin(a.stamp);
	constexpr int R = 4;
	extern __shared__ __align__(16) float smem[];
	__shared__ float outbuf[32]; // nwarps * R
	__shared__ float bval[8];
	__shared__ int bidx[8];
	float* red = smem;
	float* xs = smem + 32;
	const float post = stage_vector<DBITS>(xs, red, a.x, a.dim, a.normw, a.eps, a.ln != 0, nullptr);

	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5; // nwarps == 8
	const int nvec = a.dim / WFmt<DBITS>::VW;
	const int rows_per_iter = nwarps * R;
	float best = -FLT_MAX;
	int besti = 0x7fffffff;

	const int row_end = a.world > 1 ? a.row1 : a.vocab;
	for (int base = (a.world > 1 ? a.row0 : 0) + blockIdx.x * rows_per_iter; base < row_end; base += gridDim.x * rows_per_iter) {
		int r0 = base + warp * R;
		const uint4* rp[R];
#pragma unroll
		for (int r = 0; r < R; ++r) rp[r] = reinterpret_cast<const uint4*>(a.wcls) + (size_t)min(r0 + r, row_end - 1) * nvec;
		float v[R];
		warp_dot_rows<DBITS, R>(rp, nvec, reinterpret_cast<const float4*>(xs), v);
		if (lane == 0) {
#pragma unroll
			for (int r = 0; r < R; ++r) {
				v[r] *= post;
				outbuf[warp * R + r] = v[r];
				if (r0 + r < row_end && v[r] > best) best = v[r], besti = r0 + r;
			}
		}
		__syncthreads();
		if (threadIdx.x < rows_per_iter && base + (int)threadIdx.x < row_end) {
			if (a.world > 1) {
				for (int p = 0; p < a.world; ++p) a.peer_logits[p][base + threadIdx.x] = outbuf[threadIdx.x];
			} else {
				a.logits[base + threadIdx.x] = outbuf[threadIdx.x];
			}
		}
		__syncthreads();
	}

	if (a.cand_val || a.world > 1) {
		if (lane == 0) bval[warp] = best, bidx[warp] = besti;
		__syncthreads();
		if (threadIdx.x == 0) {
			for (int w = 1; w < nwarps; ++w)
				if (bval[w] > best || (bval[w] == best && bidx[w] < besti)) best = bval[w], besti = bidx[w];
			if (a.world > 1) {
				for (int p = 0; p < a.world; ++p) a.peer_cand_val[p][a.rank * gridDim.x + blockIdx.x] = best, a.peer_cand_idx[p][a.rank * gridDim.x + blockIdx.x] = besti;
			} else {
				a.cand_val[blockIdx.x] = best;
				a.cand_idx[blockIdx.x] = besti;
			}
		}
	}
	if (a.world > 1) __threadfence_system(); // the slices must be visible to the peers before k_tp_gather raises this rank's flag
	stamp_end(a.stamp);
}

// Tensor parallelism, after k_output: tell every peer that this rank's logits slice has landed, wait for theirs, then
// copy the complete vector from the gather area to where the caller wants it (mapped host memory or the device copy).
// flag cell [src rank] in every rank's area holds the token sequence number of the last complete slice from that rank.
// A rank cannot overwrite a peer's gather area before the peer has copied it out: its next classifier launch lies behind a
// full token of per-layer exchanges with that peer.
struct TpGatherArgs {
	int world, rank;
	const TokenParams* tp;
	unsigned* flags[TP_MAX_WORLD]; // rank p's flag cells [world]
	const float* src;
	float* dst; // NULL: no copy
	int n;
	int* err;
};

__global__ void __launch_bounds__(256) k_tp_gather(const TpGatherArgs a) {
	pdl_enter();
	const unsigned epoch = (unsigned)a.tp->tp_seq;
	if (blockIdx.x == 0 && (int)threadIdx.x < a.world && (int)threadIdx.x != a.rank) {
		__threadfence_system();
		asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(a.flags[threadIdx.x] + a.rank), "r"(epoch) : "memory");
	}
	if ((int)threadIdx.x < a.world && (int)threadIdx.x != a.rank) {
		unsigned v, spins = 0;
		unsigned long long t0 = 0;
		for (;;) {
			asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(a.flags[a.rank] + threadIdx.x) : "memory");
			if (v == epoch) break;
			if ((++spins & 1023) == 0) {
				const unsigned long long now = globaltimer_ns();
				if (!t0) t0 = now;
				if (now - t0 > 20000000000ull) { // 20 s: a peer died or the ranks diverged -- fail loudly, never hang the GPU
					if (a.err) *reinterpret_cast<volatile int*>(a.err) = 9100 + threadIdx.x;
					__threadfence_system();
					__trap();
				}
			}
		}
	}
	__syncthreads();
	if (a.dst) {
		const float4* s4 = reinterpret_cast<const float4*>(a.src);
		float4* d4 = reinterpret_cast<float4*>(a.dst);
		const int n4 = a.n >> 2;
		for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += gridDim.x * blockDim.x) d4[i] = __ldcg(s4 + i);
		for (int i = (n4 << 2) + blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += gridDim.x * blockDim.x) a.dst[i] = __ldcg(a.src + i);
	}
}

// Fold the per-CTA candidates, publish the greedy token, and advance the token parameters so the
// next replay of the graph consumes it (device-resident decode loop).
__global__ void k_advance(const float* cand_val, const int* cand_idx, int ncand, TokenParams* tp, int* out_tokens, int* last_token, int advance, int vocab) {
	pdl_enter();
	__shared__ float sv[256];
	__shared__ int si[256];
	float best = -FLT_MAX;
	int besti = 0x7fffffff;
	for (int i = threadIdx.x; i < ncand; i += blockDim.x) {
		float v = cand_val[i];
		int ix = cand_idx[i];
		if (v > best || (v == best && ix < besti)) best = v, besti = ix;
	}
	sv[threadIdx.x] = best, si[threadIdx.x] = besti;
	__syncthreads();
	for (int s = blockDim.x / 2; s > 0; s >>= 1) {
		if ((int)threadIdx.x < s) {
			float v = sv[threadIdx.x + s];
			int ix = si[threadIdx.x + s];
			if (v > sv[threadIdx.x] || (v == sv[threadIdx.x] && ix < si[threadIdx.x])) sv[threadIdx.x] = v, si[threadIdx.x] = ix;
		}
		__syncthreads();
	}
	if (threadIdx.x == 0) {
		int tok = si[0];
		if (tok < 0 || tok >= vocab) tok = 0; // only reachable when every logit is NaN
		*last_token = tok;
		if (advance) {
			out_tokens[tp->step] = tok;
			int pos = tp->pos + 1, seq_len = tp->seq_len;
			int sink = pos >= seq_len ? 2 : 0; // KV_SINKS
			tp->token = tok;
			tp->tp_seq += 1;
			tp->pos = pos;
			tp->kv_sink = sink;
			tp->kv_pos = sink + (pos - sink) % (seq_len - sink);
			tp->kv_len = pos >= seq_len ? seq_len : pos + 1;
			tp->step = tp->step + 1;
		}
	}
}

__global__ void k_set_params(TokenParams* tp, int token, int pos, int seq_len, int step) {
	int sink = pos >= seq_len ? 2 : 0; // reference infer.c:330-332
	tp->token = token;
	tp->pos = pos;
	tp->kv_sink = sink;
	tp->kv_pos = sink + (pos - sink) % (seq_len - sink);
	tp->kv_len = pos >= seq_len ? seq_len : pos + 1;
	tp->step = step;
	tp->seq_len = seq_len;
	tp->tp_seq += 1;
}

// ------------------------------------------------------------------------------------------------
// Device-side min-p sampling (reference sampler.c:44-90): cutoff = max + log(minp) * T; survivors get
// p_i = exp((l_i - max) / T); r = coin * sum(p); the first index whose running sum exceeds r wins, the last survivor
// when rounding leaves none.  The reference adds the survivors one by one in index order; k_sample_scan keeps that
// order (per-chunk lists compacted in index order) and k_sample_pick walks them sequentially with one thread, so the
// additions are the reference's additions as long as there are at most SAMPLE_EXACT survivors; beyond that (flat
// distributions) per-chunk sums are added chunk by chunk, which can move a bin edge by an ulp.
// The coin comes from the reference's xorshift* generator (sampler.c:7-17), advanced on the device.

#define SAMPLE_CHUNK 1024
#define SAMPLE_EXACT 2048

struct SampleState {
	unsigned long long rng;
	float temperature;
	float cut_delta; // log(minp) * temperature, formed on the host with the host libm like the reference does
};

struct SampleArgs {
	const float* logits;
	const float* cand_val; // per-CTA maxima of k_output
	int ncand, vocab, nchunks;
	const SampleState* st;
	int* count;      // [nchunks]
	float* csum;     // [nchunks] sequential sum of the chunk's survivors
	int* sidx;       // [nchunks][SAMPLE_CHUNK]
	float* sprob;
};

// one chunk of the vocabulary: its survivors, in index order, and their sequential sum.  MASK: a logit of -inf (a token
// its row's automaton does not allow) never survives, also where the cut is -inf (minp 0)
template <bool MASK = false>
__device__ __forceinline__ void sample_scan(const SampleArgs& a, const unsigned chunk) {
	__shared__ float red[8];
	__shared__ int wcount[8];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	float mx = -FLT_MAX;
	for (int i = tid; i < a.ncand; i += 256) mx = fmaxf(mx, a.cand_val[i]);
	for (int m = 16; m > 0; m >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));
	if (lane == 0) red[warp] = mx;
	__syncthreads();
	mx = red[0];
	for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
	const float temp = a.st->temperature, cutoff = mx + a.st->cut_delta;

	// 4 consecutive entries per thread, so that thread order is index order
	const int base = chunk * SAMPLE_CHUNK + tid * 4;
	float p[4];
	int keep = 0;
#pragma unroll
	for (int k = 0; k < 4; ++k) {
		float l = base + k < a.vocab ? a.logits[base + k] : -FLT_MAX;
		bool s = base + k < a.vocab && l >= cutoff;
		if constexpr (MASK) s = s && l != -INFINITY;
		p[k] = s ? expf((l - mx) / temp) : -1.f;
		keep += s;
	}
	int incl = keep;
	for (int m = 1; m < 32; m <<= 1) {
		int o = __shfl_up_sync(0xffffffffu, incl, m);
		if (lane >= m) incl += o;
	}
	if (lane == 31) wcount[warp] = incl;
	__syncthreads();
	int off = incl - keep;
	for (int w = 0; w < warp; ++w) off += wcount[w];
	int* li = a.sidx + (size_t)chunk * SAMPLE_CHUNK;
	float* lp = a.sprob + (size_t)chunk * SAMPLE_CHUNK;
#pragma unroll
	for (int k = 0; k < 4; ++k)
		if (p[k] >= 0.f) li[off] = base + k, lp[off] = p[k], ++off;
	__syncthreads();
	if (tid == 0) {
		int n = 0;
		for (int w = 0; w < 8; ++w) n += wcount[w];
		float sum = 0.f;
		for (int j = 0; j < n; ++j) sum += lp[j];
		a.count[chunk] = n, a.csum[chunk] = sum;
	}
}

__global__ void __launch_bounds__(256) k_sample_scan(const SampleArgs a) {
	pdl_enter();
	sample_scan(a, blockIdx.x);
}

__device__ __forceinline__ unsigned xorshift_u32(unsigned long long& s) { // reference sampler.c:7-13
	s ^= s >> 12;
	s ^= s << 25;
	s ^= s >> 27;
	return (unsigned)((s * 0x2545F4914F6CDD1Dull) >> 32);
}

// The reference's two sequential passes (sum, then walk to the coin), then the bookkeeping of k_advance.  One CTA: up to
// SAMPLE_EXACT survivors are first gathered -- in index order, coalesced -- into shared memory by all threads, and thread 0
// then performs exactly the reference's left-to-right float additions on them (4 cycles each instead of a global-memory
// round trip); with more survivors the per-chunk sums of k_sample_scan are walked and only the chunk holding the coin is
// expanded.
__device__ __forceinline__ void sample_pick(const SampleArgs a, SampleState* st, TokenParams* tp, int* out_tokens, int* last_token, int advance) {
	__shared__ float sp[SAMPLE_EXACT];
	__shared__ int si[SAMPLE_EXACT];
	__shared__ int coff[256]; // exclusive prefix of the chunk counts (nchunks <= 256: vocabularies up to 262144)
	__shared__ int stotal;
	const int tid = threadIdx.x;
	const bool small_tab = a.nchunks <= 256;
	if (tid == 0) {
		int total = 0;
		for (int c = 0; c < a.nchunks; ++c) {
			if (small_tab) coff[c] = total;
			total += a.count[c];
		}
		stotal = total;
	}
	__syncthreads();
	const int total = stotal;
	const bool exact = total <= SAMPLE_EXACT && small_tab;
	if (exact) {
		for (int c = 0; c < a.nchunks; ++c) {
			const int n = a.count[c], o = coff[c];
			for (int j = tid; j < n; j += blockDim.x) sp[o + j] = a.sprob[(size_t)c * SAMPLE_CHUNK + j], si[o + j] = a.sidx[(size_t)c * SAMPLE_CHUNK + j];
		}
	}
	__syncthreads();
	if (tid != 0) return;
	unsigned long long rng = st->rng;
	const float coin = (float)(xorshift_u32(rng) >> 8) / 16777216.0f; // sampler.c:15-17
	st->rng = rng;
	int tok = -1, fallback = 0;
	if (exact) {
		float cum = 0.f;
		for (int j = 0; j < total; ++j) cum += sp[j];
		if (total) fallback = si[total - 1];
		const float r = coin * cum;
		float cdf = 0.f;
		for (int j = 0; j < total; ++j) {
			cdf += sp[j];
			if (r < cdf) {
				tok = si[j];
				break;
			}
		}
	} else {
		float cum = 0.f;
		for (int c = 0; c < a.nchunks; ++c) {
			cum += a.csum[c];
			if (a.count[c]) fallback = a.sidx[(size_t)c * SAMPLE_CHUNK + a.count[c] - 1];
		}
		const float r = coin * cum;
		float cdf = 0.f;
		for (int c = 0; c < a.nchunks && tok < 0; ++c) {
			if (r < cdf + a.csum[c]) {
				const float* lp = a.sprob + (size_t)c * SAMPLE_CHUNK;
				for (int j = 0; j < a.count[c]; ++j) {
					cdf += lp[j];
					if (r < cdf) {
						tok = a.sidx[(size_t)c * SAMPLE_CHUNK + j];
						break;
					}
				}
				if (tok < 0) continue; // rounding: the edge belongs to a later chunk
			} else {
				cdf += a.csum[c];
			}
		}
	}
	if (tok < 0) tok = fallback;
	*last_token = tok;
	if (advance) {
		out_tokens[tp->step] = tok;
		int pos = tp->pos + 1, seq_len = tp->seq_len;
		int sink = pos >= seq_len ? 2 : 0; // KV_SINKS
		tp->token = tok;
		tp->tp_seq += 1;
		tp->pos = pos;
		tp->kv_sink = sink;
		tp->kv_pos = sink + (pos - sink) % (seq_len - sink);
		tp->kv_len = pos >= seq_len ? seq_len : pos + 1;
		tp->step += 1;
	}
}

__global__ void __launch_bounds__(256) k_sample_pick(const SampleArgs a, SampleState* st, TokenParams* tp, int* out_tokens, int* last_token, int advance) {
	pdl_enter();
	sample_pick(a, st, tp, out_tokens, last_token, advance);
}

// n rows sampled side by side (calm_b200_verify_sample): row r is `a` with every array advanced by r rows -- logits by
// `vocab`, cand_val by `ncand`, the state by one, the counts and sums by `nchunks` and the lists by nchunks * SAMPLE_CHUNK
// -- and its token goes to tokens[r].  k_sample_scan_rows runs chunk blockIdx.x of row blockIdx.y, k_sample_pick_rows row
// blockIdx.x; each row is exactly k_sample_scan + k_sample_pick on that row.
__device__ __forceinline__ SampleArgs sample_row(const SampleArgs& a, int r) {
	SampleArgs b = a;
	b.logits += (size_t)r * a.vocab, b.cand_val += (size_t)r * a.ncand, b.st += r;
	b.count += (size_t)r * a.nchunks, b.csum += (size_t)r * a.nchunks;
	b.sidx += (size_t)r * a.nchunks * SAMPLE_CHUNK, b.sprob += (size_t)r * a.nchunks * SAMPLE_CHUNK;
	return b;
}

__global__ void __launch_bounds__(256) k_sample_scan_rows(const SampleArgs a) {
	pdl_enter();
	sample_scan(sample_row(a, blockIdx.y), blockIdx.x);
}

// k_sample_scan_rows where masked tokens (-inf) never survive (calm_b200_decode_sample_queue_constrained)
__global__ void __launch_bounds__(256) k_sample_scan_rows_masked(const SampleArgs a) {
	pdl_enter();
	sample_scan<true>(sample_row(a, blockIdx.y), blockIdx.x);
}

__global__ void __launch_bounds__(256) k_sample_pick_rows(const SampleArgs a, SampleState* st, int* tokens) {
	pdl_enter();
	const int r = blockIdx.x;
	sample_pick(sample_row(a, r), st + r, nullptr, nullptr, tokens + r, 0);
}

// ------------------------------------------------------------------------------------------------
// Top-k / top-p truncation of sampled rows (calm_b200_decode_sample_queue_truncated; the rule is include/calm_b200.h's).
// One cluster of TRUNC_CTAS CTAs per row: CTA c stages ids [c S, (c + 1) S), S = ceil(vocab / TRUNC_CTAS), into shared
// memory with one bulk copy, then radix-selects over the order-preserving key of each allowed logit, 8 bits a round.  A
// round's histograms (a count and a 2^40-scaled mass per bucket) are built per warp, summed per CTA, and every CTA sums
// all TRUNC_CTAS of them through distributed shared memory, so every CTA takes the same decision with integer sums.
// Finally each CTA writes -inf over its dropped entries of the row, in place: what the masked scan then leaves out.

#define TRUNC_CTAS 8
#define TRUNC_VOCAB_MAX (TRUNC_CTAS * 32768) // 128 KB of staged logits per CTA (the sampler's exact-table limit too)

// a step's truncated sampled rows: row[i] with its request's top_k[i] (0: off) and top_p[i] (1: off), by value
struct TruncRows {
	int row[16];
	int top_k[16];
	float top_p[16];
};

__device__ __forceinline__ uint32_t trunc_key(float l) { // larger logit, larger key
	const uint32_t u = __float_as_uint(l);
	return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}
__device__ __forceinline__ float trunc_logit(uint32_t k) {
	return __uint_as_float((k & 0x80000000u) ? k & 0x7fffffffu : ~k);
}
// m(v) = floor(expf((l - M) / T) * 2^40): the sampler's survivor weight, exactly scaled to an integer
__device__ __forceinline__ unsigned long long trunc_mass(float l, float mx, float temp) {
	return (unsigned long long)(expf((l - mx) / temp) * 1099511627776.0f);
}
// ceil(z * p) for 0 < p <= 1 taken exactly, p = mant 2^e
__device__ __forceinline__ unsigned long long trunc_target(unsigned long long z, float p) {
	const uint32_t u = __float_as_uint(p);
	const int be = (u >> 23) & 0xff;
	const unsigned long long mant = be ? (u & 0x7fffffu) | 0x800000u : u & 0x7fffffu;
	const int sh = (be ? be : 1) - 150; // p = mant 2^sh, sh <= -23
	const unsigned __int128 prod = (unsigned __int128)z * mant;
	if (-sh >= 128) return prod ? 1 : 0;
	const unsigned __int128 q = prod >> -sh;
	return (unsigned long long)q + ((q << -sh) != prod ? 1 : 0);
}

struct TruncHist {
	unsigned cnt[256];
	unsigned long long mass[256];
};

__global__ void __cluster_dims__(TRUNC_CTAS, 1, 1) __launch_bounds__(256) k_sample_trunc_rows(const SampleArgs a0, const TruncRows t) {
	namespace cg = cooperative_groups;
	extern __shared__ __align__(16) float seg_raw[]; // [S + 8]: the segment from seg_raw[4 - h] on
	__shared__ TruncHist wh[8];                      // per warp
	__shared__ TruncHist ch[2];                      // the CTA's, ping-pong between rounds (read by the whole cluster)
	__shared__ unsigned long long cz[2];             // the CTA's part of a cluster sum
	__shared__ unsigned ctie[2];
	__shared__ __align__(8) uint64_t bar;
	__shared__ uint32_t sel_key;
	__shared__ unsigned sel_rem;
	__shared__ unsigned long long sel_above;
	__shared__ unsigned sel_group;
	__shared__ unsigned wscan[8];
	pdl_enter();
	cg::cluster_group cluster = cg::this_cluster();
	const int c = (int)cluster.block_rank(), tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int row = t.row[blockIdx.y], K = t.top_k[blockIdx.y];
	const float P = t.top_p[blockIdx.y];
	const SampleArgs a = sample_row(a0, row);
	float* logits = const_cast<float*>(a.logits); // the step's own row of pf.vlogits, truncated in place
	const int S = (a.vocab + TRUNC_CTAS - 1) / TRUNC_CTAS, lo = c * S, n = max(0, min(S, a.vocab - lo));

	// the segment, aligned part by one bulk copy, the <= 3 entries on each side of it by plain loads
	const float* gp = logits + lo;
	const int h = n ? (int)(((16 - ((uintptr_t)gp & 15)) & 15) >> 2) : 0, hb = min(h, n);
	const int nb = n > hb ? ((n - hb) >> 2) << 2 : 0;
	float* seg = seg_raw + 4 - h;
	if (tid == 0) {
		mbar_init(&bar, 1);
		mbar_init_fence();
	}
	__syncthreads();
	if (tid == 0) {
		mbar_expect_tx(&bar, nb * 4u);
		if (nb) tma_load_1d(seg + hb, gp + hb, nb * 4u, &bar);
	}
	if (tid < hb) seg[tid] = gp[tid];
	if (tid < n - hb - nb) seg[hb + nb + tid] = gp[hb + nb + tid];

	float mx = -FLT_MAX; // M and T as sample_scan forms them
	for (int i = tid; i < a.ncand; i += 256) mx = fmaxf(mx, a.cand_val[i]);
	mx = warp_max(mx);
	if (lane == 0) wscan[warp] = __float_as_uint(mx);
	mbar_wait(&bar, 0);
	__syncthreads();
	mx = __uint_as_float(wscan[0]);
	for (int i = 1; i < 8; ++i) mx = fmaxf(mx, __uint_as_float(wscan[i]));
	const float temp = a.st->temperature;

	// sums x over the cluster (every CTA gets the total); slot `s` alternates between consecutive calls
	int zs = 0;
	auto cluster_sum = [&](unsigned long long x) {
		for (int m = 16; m > 0; m >>= 1) x += __shfl_xor_sync(0xffffffffu, x, m);
		if (lane == 0) wh[warp].mass[0] = x;
		__syncthreads();
		if (tid == 0) {
			unsigned long long s = 0;
			for (int w = 0; w < 8; ++w) s += wh[w].mass[0];
			cz[zs] = s;
		}
		cluster.sync();
		unsigned long long tot = 0;
		for (int r = 0; r < TRUNC_CTAS; ++r) tot += *cluster.map_shared_rank(&cz[zs], r);
		zs ^= 1;
		return tot;
	};

	// One radix round over the allowed entries whose key agrees with `pre` above bit `shift + 8` and that `in` admits:
	// the cluster's count and mass histograms of their next digit, then the walk from the top bucket that stops where
	// the running count (BY_MASS: mass) reaches `need`.  The mass of the excluded top-k tie group (key kx, rx of its
	// tokens in the set) is added back by every CTA alike.  Leaves the chosen digit in sel_key, the remainder in
	// sel_rem / sel_above (what lies above the chosen bucket) and the bucket's count in sel_group.
	int hs = 0;
	auto radix_round = [&](uint32_t pre, int shift, auto in, bool by_mass, unsigned long long need, uint32_t kx, unsigned rx, unsigned long long mxk) {
		TruncHist& w = wh[warp];
		for (int b = lane; b < 256; b += 32) w.cnt[b] = 0, w.mass[b] = 0;
		__syncwarp();
		const uint32_t hmask = shift == 24 ? 0u : ~0u << (shift + 8);
		for (int i = tid; i < n; i += 256) {
			const float l = seg[i];
			const uint32_t k = trunc_key(l);
			if (l == -INFINITY || (k & hmask) != (pre & hmask) || !in(k)) continue;
			const int b = (k >> shift) & 255;
			atomicAdd(&w.cnt[b], 1u);
			if (by_mass) atomicAdd(&w.mass[b], trunc_mass(l, mx, temp));
		}
		__syncthreads();
		TruncHist& o = ch[hs];
		{
			unsigned cn = 0;
			unsigned long long ms = 0;
			for (int v = 0; v < 8; ++v) cn += wh[v].cnt[tid], ms += wh[v].mass[tid];
			o.cnt[tid] = cn, o.mass[tid] = ms;
		}
		cluster.sync();
		unsigned cn = 0;
		unsigned long long ms = 0;
		for (int r = 0; r < TRUNC_CTAS; ++r) {
			const TruncHist* rh = cluster.map_shared_rank(&o, r);
			cn += rh->cnt[tid], ms += rh->mass[tid];
		}
		if (rx && (kx & hmask) == (pre & hmask) && (int)((kx >> shift) & 255) == tid) cn += rx, ms += rx * mxk;
		wh[0].cnt[tid] = cn, wh[0].mass[tid] = ms; // (every warp is past reading wh: the cluster barrier)
		hs ^= 1;
		__syncthreads();
		if (tid == 0) {
			unsigned long long acc = 0;
			int b = 255;
			for (; b > 0; --b) {
				const unsigned long long x = by_mass ? wh[0].mass[b] : wh[0].cnt[b];
				if (acc + x >= need) break;
				acc += x;
			}
			sel_key = (pre & hmask) | ((uint32_t)b << shift);
			sel_above = acc, sel_group = wh[0].cnt[b];
		}
		__syncthreads();
	};

	// top-k: (vk, rk), the K-th rank's key and how many of its tied tokens the set keeps; off (vk 0) when K >= allowed
	uint32_t vk = 0, sel = 0;
	unsigned rk = 0;
	const unsigned long long allowed = cluster_sum([&] {
		unsigned x = 0;
		for (int i = tid; i < n; i += 256) x += seg[i] != -INFINITY;
		return (unsigned long long)x;
	}());
	auto all = [](uint32_t) { return true; };
	if (K > 0 && (unsigned long long)K < allowed) {
		unsigned long long need = K;
		for (int shift = 24; shift >= 0; shift -= 8) {
			radix_round(sel, shift, all, false, need, 0, 0, 0);
			sel = sel_key, need -= sel_above;
		}
		vk = sel, rk = (unsigned)need;
	}
	uint32_t v = vk; // the kept set: keys above v, and the first r tokens of key v
	unsigned r = rk;
	if (P < 1.0f) {
		const unsigned long long mk = vk ? trunc_mass(trunc_logit(vk), mx, temp) : 0;
		unsigned long long z = 0;
		for (int i = tid; i < n; i += 256) {
			const float l = seg[i];
			if (l != -INFINITY && trunc_key(l) > vk) z += trunc_mass(l, mx, temp);
		}
		z = cluster_sum(z) + rk * mk;
		unsigned long long need = trunc_target(z, P);
		auto above_k = [vk](uint32_t k) { return k > vk; };
		sel = 0;
		for (int shift = 24; shift >= 0; shift -= 8) {
			radix_round(sel, shift, above_k, true, need, vk, rk, mk);
			sel = sel_key, need -= sel_above;
		}
		const unsigned long long mp = trunc_mass(trunc_logit(sel), mx, temp); // > 0: the walk stops at a bucket with mass
		v = sel, r = (unsigned)min((unsigned long long)sel_group, (need + mp - 1) / mp);
	}
	if (v) {
		// this CTA's tied tokens before those of the CTAs below it
		unsigned ties = 0;
		for (int i = tid; i < n; i += 256) ties += trunc_key(seg[i]) == v && seg[i] != -INFINITY;
		for (int m = 16; m > 0; m >>= 1) ties += __shfl_xor_sync(0xffffffffu, ties, m);
		if (lane == 0) wscan[warp] = ties;
		__syncthreads();
		if (tid == 0) {
			unsigned s = 0;
			for (int w = 0; w < 8; ++w) s += wscan[w];
			ctie[zs] = s;
		}
		cluster.sync();
		unsigned before = 0;
		for (int q = 0; q < c; ++q) before += *cluster.map_shared_rank(&ctie[zs], q);
		const int keep = (int)min(max((long long)r - before, 0ll), (long long)ctie[zs]);
		// in id order: 4 consecutive entries per thread, 1024 a pass, the tied ones ranked by a block scan
		int seen = 0;
		for (int base = 0; base < n; base += 1024) {
			const int i0 = base + tid * 4;
			bool tie[4], drop[4];
			int nt = 0;
#pragma unroll
			for (int j = 0; j < 4; ++j) {
				const float l = i0 + j < n ? seg[i0 + j] : -INFINITY;
				const uint32_t k = trunc_key(l);
				tie[j] = l != -INFINITY && k == v;
				drop[j] = l != -INFINITY && k < v;
				nt += tie[j];
			}
			int incl = nt;
			for (int m = 1; m < 32; m <<= 1) {
				const int x = __shfl_up_sync(0xffffffffu, incl, m);
				if (lane >= m) incl += x;
			}
			__syncthreads(); // (the previous pass is done with wscan)
			if (lane == 31) wscan[warp] = incl;
			__syncthreads();
			int rank = seen + incl - nt;
			for (int w = 0; w < warp; ++w) rank += wscan[w];
			for (int w = 0; w < 8; ++w) seen += wscan[w];
#pragma unroll
			for (int j = 0; j < 4; ++j) {
				if (tie[j]) drop[j] = rank++ >= keep;
				if (drop[j]) logits[lo + i0 + j] = -INFINITY;
			}
		}
	}
	cluster.sync(); // no CTA leaves while another may still read its shared memory
}

// per-chunk maxima of a logits vector (stand-alone sampler entry point: what k_output's candidates are in a token)
__global__ void __launch_bounds__(256) k_chunk_max(const float* logits, int vocab, float* out) {
	__shared__ float red[8];
	float mx = -FLT_MAX;
	for (int i = blockIdx.x * SAMPLE_CHUNK + threadIdx.x; i < min(vocab, (int)(blockIdx.x + 1) * SAMPLE_CHUNK); i += blockDim.x) mx = fmaxf(mx, logits[i]);
	mx = warp_max(mx);
	if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
		out[blockIdx.x] = mx;
	}
}

// x += p (tensor-parallel: the all-reduced partial of wo / w2 joins the residual stream)
__global__ void k_addvec(float* x, const float* p, int n) {
	pdl_enter();
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) x[i] += p[i];
}

// plain matvec (unit tests, per-kernel roofline bench): y = W . x
struct MatvecArgs {
	const float* x;
	const void* w;
	float* y;
	int n, d;
};

template <int DBITS>
__global__ void __launch_bounds__(256) k_matvec(const MatvecArgs a) {
	extern __shared__ __align__(16) float smem[];
	float* red = smem;
	float* xs = smem + 32;
	stage_vector<DBITS>(xs, red, a.x, a.n, nullptr, 0.f, false, nullptr);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
	const int nvec = a.n / WFmt<DBITS>::VW;
	for (int p = blockIdx.x * nwarps + warp; p < (a.d + 1) / 2; p += gridDim.x * nwarps) {
		int r1 = min(2 * p + 1, a.d - 1);
		const uint4* rp[2] = {reinterpret_cast<const uint4*>(a.w) + (size_t)(2 * p) * nvec, reinterpret_cast<const uint4*>(a.w) + (size_t)r1 * nvec};
		float v[2];
		warp_dot_rows<DBITS, 2>(rp, nvec, reinterpret_cast<const float4*>(xs), v);
		if (lane == 0) {
			a.y[2 * p] = v[0];
			if (2 * p + 1 < a.d) a.y[2 * p + 1] = v[1];
		}
	}
}

// deterministic pseudo-random cache fill (bench: decode at a late position without the prefix)
template <typename KVT>
__global__ void k_fill_kv(KVT* kc, KVT* vc, size_t n_layers_heads, int seq_len, int head_dim, int n_pos, unsigned long long seed) {
	size_t total = n_layers_heads * (size_t)n_pos * head_dim;
	for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
		size_t lh = i / ((size_t)n_pos * head_dim), rem = i % ((size_t)n_pos * head_dim);
		size_t idx = lh * seq_len * head_dim + rem;
		unsigned long long z = (i + 1) * 0x9E3779B97F4A7C15ull + seed;
		z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
		z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
		z ^= z >> 31;
		float a = ((z & 0xffffff) / 16777216.f - 0.5f) * 2.f;         // U(-1,1)
		float b = (((z >> 24) & 0xffffff) / 16777216.f - 0.5f) * 2.f;
		kv_store(kc + idx, a);
		kv_store(vc + idx, b);
	}
}
