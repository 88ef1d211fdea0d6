// prefill.cuh -- batched prompt pass (SURVEY.md s.8f row 1; reference behaviour replaced: run.c:206-209 feeds the prompt one
// token at a time through forward(), README.md:80).  T prompt tokens go through every layer together, so each weight
// matrix is read once per 128-token tile instead of once per token and the projections become real GEMMs on the
// Hopper tensor cores:
//
//   k_pf_gemm   D[128 tokens][128 weight rows] (+)= X_tile . W_tile^T with wgmma.mma_async (m64n128k16, f16 in, fp32
//               accumulators in registers).  B = the weight tile, dequantised ON THE FLY by one warpgroup from the model's
//               own format (fp16 / e5m2 / gf4: all exact in f16) into the 128-byte-swizzled K-major shared-memory layout
//               the MMA reads; A = the activations as TWO f16 matrices hi + lo (x = hi + lo to 22 bits, so the result
//               carries fp32-grade inputs: two MMAs per k-step into the same accumulator), brought in by 2-D TMA
//               (cp.async.bulk.tensor, SWIZZLE_128B).  Two consumer warpgroups own 64 tokens each; stages are handed
//               over through mbarriers, and the epilogue works on the accumulator registers directly: bias / clip /
//               RoPE / KV-cache append (QKV), residual add (wo, w2), act(w1 x) * (w3 x) with both accumulators held by
//               the same thread (FFN up).  A thread holds adjacent weight rows (features 2c, 2c + 1) of a token, so a
//               RoPE pair never leaves the thread and every store is a contiguous pair.
//   k_pf_attn   causal attention of the block against the cache (fp32 math on the cached fp16 / e5m2 entries, online
//               softmax; reference infer.c:238-267), one warp per query token, K/V tiles staged in shared memory.
//   k_pf_norm   RMSNorm / LayerNorm per token (reference infer.c:183-207) -> hi / lo f16 rows.
//
// Scoring (calm_b200_score, the reference's study(): run.c:291-308) adds the classifier over all rows of the block without
// ever writing the [T][vocab] logits: the final norm (k_pf_norm), k_pf_gemm in PF_CLS mode, whose epilogue reduces each
// token's 128 logits of the tile to one (max, sum exp(logit - max)) record and keeps the target's logit, and k_pf_logprob,
// which merges a token's records in a fixed order into ln softmax(logits)[target].  The packed scoring calls (score_batch,
// score_context) put several sequences into one block: per-row RoPE positions (k_pf_rope_rows) and attention that starts
// each sequence's key tiles at its own first row (k_pf_attn<.., SEG>); everything else works per row.  A packed block
// may also hold contexts, once each, and sequences that continue them: a sequence's rows attend
// to its context's rows and then its own as one key sequence (k_pf_attn<.., SEG, CTX>).  The greedy scoring calls run
// PF_CLS_GREEDY and k_pf_logprob<true>, which also give each row's argmax, with the same log-probability bits.  The top-k
// scoring calls run PF_CLS_TOPK and k_pf_logprob<false, true>: each tile's k largest logits, merged into each row's k largest.
// The short-block GEMM of calm_b200_verify_greedy (k_vf_gemm, verify.cuh) dequantises through this file's weight
// conversions (e5m2_word_h2, gf4_word_h2) and ends in its epilogue (pf_epilogue_pair for UP, WO and DOWN).
//
// Parity contract (tests/test_prefill_gpu.py): after forward_prefill_cuda(tokens, n, pos0) the KV cache and the logits of
// the following token equal those of n serial forward(FF_UPDATE_KV_ONLY) calls within the stated tolerances.
#pragma once

#include <cuda.h>

#include "stages.cuh"

#define PF_BM 128 // weight rows per tile  (the N of the MMA)
#define PF_BN 128 // tokens per tile       (two consumer warpgroups of 64: the M of the MMA)
#define PF_BK 64  // k per stage: 64 f16 = 128 bytes = one swizzle atom
#define PF_THREADS 384 // warpgroup 0: dequantising producers (thread 0 also issues the TMA); warpgroups 1, 2: MMA + epilogue
enum { PF_QKV = 0, PF_WO = 1, PF_UP = 2, PF_DOWN = 3, PF_CLS = 4, PF_CLS_GREEDY = 5, PF_CLS_TOPK = 6, PF_CLS_SAMPLE = 7, PF_QKV_SLOTS = 8 }; // PF_CLS_GREEDY: PF_CLS + each tile's argmax; PF_CLS_SAMPLE (k_vf_gemm only): PF_CLS_GREEDY + the logit rows
// PF_QKV_SLOTS (k_vf_gemm only): PF_QKV, but row t's keys and values go to cache slot VfArgs::slot[t] instead of pos0 + t
#define PF_TOPK_MAX 20 // PF_CLS_TOPK: PF_CLS + each tile's k <= PF_TOPK_MAX largest logits (CALM_B200_TOPK_MAX)

// ---------------------------------------------------------------- wgmma / TMA wrappers
__device__ __forceinline__ void wgmma_fence() { // accumulator registers written by ordinary instructions -> visible to wgmma
	asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
	asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() { // at most N committed groups of this warpgroup still in flight
	asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses to accumulator registers across wgmma_wait
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
	for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] += A[64 x 16] . B[128 x 16]^T, f16 x f16 -> f32, A and B K-major in shared memory; issued by the whole warpgroup
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t desc_a, uint64_t desc_b) {
	asm volatile(
	    "{\n\t"
	    "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
	    "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
	    "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
	    "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
	    "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
	    "%64, %65, 1, 1, 1, 0, 0;\n\t"
	    "}"
	    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
	      "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
	      "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
	      "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
	      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
	      "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
	      "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
	    : "l"(desc_a), "l"(desc_b)
	    : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)), "l"(map),
	             "r"(c0), "r"(c1), "r"(smem_u32(bar))
	             : "memory");
}
// bounded wait (about 2 s): a broken pipeline traps with a message instead of hanging the GPU
__device__ __forceinline__ void mbar_wait_guard(uint64_t* bar, uint32_t parity) {
	unsigned spins = 0;
	while (!mbar_try_wait(bar, parity)) {
		if (++spins > (1u << 26)) {
			printf("calm_b200: k_pf_gemm pipeline stalled (block %d,%d thread %d)\n", blockIdx.x, blockIdx.y, threadIdx.x);
			__trap();
		}
	}
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { // generic-proxy writes to shared memory -> visible to the async proxy (tensor core reads)
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// wgmma shared-memory matrix descriptor: K-major tile, rows of 128 bytes (64 f16), 128-byte swizzle (layout type 1),
// 8-row groups 1024 bytes apart (stride byte offset); the leading byte offset is unused by swizzled K-major layouts
__device__ __forceinline__ uint64_t wgmma_desc_sw128(const void* tile) {
	const uint64_t addr = (uint64_t)(smem_u32(tile) & 0x3FFFF) >> 4;
	return addr | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// ---------------------------------------------------------------- small kernels

// X[t][:] = decode(E[tokens[t]])  (reference infer.c:335-347)
template <int DBITS>
__global__ void k_pf_embed(float* X, const void* table, const int* tokens, int n, int dim) {
	pdl_enter();
	const int t = blockIdx.x;
	if (t >= n) return;
	const size_t base = (size_t)tokens[t] * dim;
	for (int i = threadIdx.x; i < dim; i += blockDim.x) X[(size_t)t * dim + i] = weight_at<DBITS>(table, base + i);
}

// rope[t][j] = (cos, sin)((pos0 + t) * freq[j])
__global__ void k_pf_rope(float2* rope, const float* freq, int n, int half_hd, int pos0) {
	pdl_enter();
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n * half_hd) return;
	float s, c;
	sincosf((float)(pos0 + i / half_hd) * freq[i % half_hd], &s, &c);
	rope[i] = make_float2(c, s);
}

// rope[t][j] = (cos, sin)(rowpos[t] * freq[j]): the table of a packed block, whose positions restart with each context
// and sequence it holds; for rowpos[t] = pos0 + t the same float arguments as k_pf_rope, so the same bits
__global__ void k_pf_rope_rows(float2* rope, const float* freq, const int* rowpos, int n, int half_hd) {
	pdl_enter();
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n * half_hd) return;
	float s, c;
	sincosf((float)rowpos[i / half_hd] * freq[i % half_hd], &s, &c);
	rope[i] = make_float2(c, s);
}

// one CTA per token: norm (infer.c:183-207) then hi / lo split; rows beyond n (tile padding) are not written and hold whatever
// an earlier, longer pass left: a GEMM's output column depends on its own token's row only, and every epilogue drops t >= n
__global__ void __launch_bounds__(256) k_pf_norm(const float* X, const float* normw, __half* hi, __half* lo, int n, int dim, float eps, int ln) {
	pdl_enter();
	__shared__ float red[32];
	const int t = blockIdx.x;
	if (t >= n) return;
	const float* x = X + (size_t)t * dim;
	float mean = 0.f;
	if (ln) {
		float s = 0.f;
		for (int i = threadIdx.x; i < dim; i += blockDim.x) s += x[i];
		mean = block_sum(s, red) / dim;
	}
	float ss = 0.f;
	for (int i = threadIdx.x; i < dim; i += blockDim.x) {
		const float d = x[i] - mean;
		ss = fmaf(d, d, ss);
	}
	ss = block_sum(ss, red);
	const float scale = 1.0f / sqrtf(ss / dim + eps);
	for (int i = threadIdx.x; i < dim; i += blockDim.x) {
		const float v = (x[i] - mean) * scale * normw[i];
		__half h, l;
		split_hl(v, h, l);
		hi[(size_t)t * dim + i] = h, lo[(size_t)t * dim + i] = l;
	}
}

// ---------------------------------------------------------------- the GEMM

struct PfGemmArgs {
	const void* w[3]; // QKV: wq, wk, wv   UP: w1, w3   WO / DOWN: w
	int K, n_tokens;
	// QKV epilogue
	float* Q;         // [T][q_dim]
	int q_dim, kv_dim, head_dim, seq_len, pos0;
	const float* bias;
	float clip;
	const float2* rope; // [T][head_dim / 2]
	void* kc;           // this layer: [n_kv_heads][seq_len][head_dim]
	void* vc;
	// WO / DOWN epilogue
	float* X; // [T][dim] residual stream
	int dim;
	// UP epilogue
	__half* Hhi;
	__half* Hlo;
	int hidden, gelu;
	// CLS epilogue: w[0] = the classifier [vocab][K], one CTA column per 128 vocabulary rows
	const int* targets; // [T] the token whose log-probability is wanted after each row
	float2* part;       // [T][gridDim.x] (max, sum exp(logit - max)) of the token's logits in each vocabulary tile
	float* tgt;         // [T] logit of the target
	int vocab;
	int* gidx; // (PF_CLS_GREEDY) [T][gridDim.x] the lowest vocabulary index of the token's maximum logit in each tile
	// (PF_CLS_TOPK) [T][gridDim.x][topk] the token's topk largest logits in each tile and their vocabulary indices, by logit
	// descending and, on equal logits, index ascending; a tile with fewer than topk rows pads with (-INFINITY, INT_MAX)
	float* topv;
	int* topi;
	int topk;
};

// 64 weights of one row (one k-stage) -> 8 swizzled 16-byte chunks of f16 in the weight tile
template <int DBITS>
__device__ __forceinline__ void pf_load_raw(const unsigned char* row, int kb, uint4 (&raw)[DBITS / 2]) {
	const uint4* p = reinterpret_cast<const uint4*>(row + (size_t)kb * (PF_BK * DBITS / 8));
#pragma unroll
	for (int i = 0; i < DBITS / 2; ++i) raw[i] = ldg_stream(p + i);
}
// The weight formats -> f16, exactly (the prompt pass and k_vf_gemm dequantise through these two)
// four e5m2 weights -> two f16 pairs in weight order: an e5m2 byte is the high byte of the f16 (reference infer.c:28-35)
__device__ __forceinline__ uint2 e5m2_word_h2(uint32_t w) {
	return make_uint2(__byte_perm(w, 0, 0x1404), __byte_perm(w, 0, 0x3424));
}
// a gf4 word (scale byte + eight 3-bit codes) -> four f16 pairs in weight order: (q - 4) * s / -4 (reference
// infer.c:37-40); at most 6 significant bits: exact in f16
__device__ __forceinline__ uint4 gf4_word_h2(uint32_t w) {
	const float sf = e5m2_to_float((uint8_t)(w & 0xff)) * -0.25f;
	uint32_t h[4];
#pragma unroll
	for (int k = 0; k < 4; ++k) {
		const float a0 = (float)((int)((w >> (8 + 6 * k)) & 7) - 4) * sf, a1 = (float)((int)((w >> (11 + 6 * k)) & 7) - 4) * sf;
		h[k] = pack_h2(__float2half_rn(a0), __float2half_rn(a1));
	}
	return make_uint4(h[0], h[1], h[2], h[3]);
}

template <int DBITS>
__device__ __forceinline__ void pf_store_a(unsigned char* tile, int r, const uint4 (&raw)[DBITS / 2]) {
	unsigned char* rowp = tile + r * 128;
	auto put = [&](int c, uint4 v) { *reinterpret_cast<uint4*>(rowp + ((c ^ (r & 7)) << 4)) = v; };
	if constexpr (DBITS == 16) {
#pragma unroll
		for (int c = 0; c < 8; ++c) put(c, raw[c]);
	} else if constexpr (DBITS == 8) {
#pragma unroll
		for (int i = 0; i < 4; ++i) {
			const uint2 h0 = e5m2_word_h2(raw[i].x), h1 = e5m2_word_h2(raw[i].y), h2 = e5m2_word_h2(raw[i].z), h3 = e5m2_word_h2(raw[i].w);
			put(2 * i, make_uint4(h0.x, h0.y, h1.x, h1.y));
			put(2 * i + 1, make_uint4(h2.x, h2.y, h3.x, h3.y));
		}
	} else {
#pragma unroll
		for (int i = 0; i < 2; ++i) {
			const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
			for (int j = 0; j < 4; ++j) put(4 * i + j, gf4_word_h2(w[j]));
		}
	}
}

template <int MODE>
__host__ __device__ constexpr int pf_stages() {
	return MODE == PF_UP ? 3 : 4;
}
template <int MODE>
__host__ __device__ constexpr size_t pf_stage_bytes() {
	return (size_t)(MODE == PF_UP ? 2 : 1) * PF_BM * 128 + 2 * PF_BN * 128; // A tile(s) + B hi + B lo
}
template <int MODE>
__host__ __device__ constexpr size_t pf_smem_bytes() {
	return pf_stages<MODE>() * pf_stage_bytes<MODE>() + 1024; // + alignment slack
}

// The epilogue of UP, WO and DOWN for token t and the output rows (gr, gr + 1) (gr even) whose finished sums are x0, x1
// (UP: of w1, with g0, g1 those of w3).  UP: act(w1 x) * (w3 x) as hi + lo; WO / DOWN: residual add.  (QKV's epilogue is
// written out in each kernel: as a function it compiles to different instructions in k_pf_gemm.)
template <int MODE>
__device__ __forceinline__ void pf_epilogue_pair(const PfGemmArgs& a, int gr, int t, float x0, float x1, float g0, float g1) {
	if constexpr (MODE == PF_UP) {
		const float h0 = (a.gelu ? act_gelu(x0) : act_silu(x0)) * g0, h1 = (a.gelu ? act_gelu(x1) : act_silu(x1)) * g1;
		__half hh0, hl0, hh1, hl1;
		split_hl(h0, hh0, hl0), split_hl(h1, hh1, hl1);
		*reinterpret_cast<uint32_t*>(a.Hhi + (size_t)t * a.hidden + gr) = pack_h2(hh0, hh1);
		*reinterpret_cast<uint32_t*>(a.Hlo + (size_t)t * a.hidden + gr) = pack_h2(hl0, hl1);
	} else {
		float2* dst = reinterpret_cast<float2*>(a.X + (size_t)t * a.dim + gr);
		const float2 o = *dst;
		*dst = make_float2(o.x + x0, o.y + x1);
	}
}

template <int MODE, int DBITS, typename KVT>
__global__ void __launch_bounds__(PF_THREADS, 1) k_pf_gemm(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo, const PfGemmArgs a) {
	constexpr int STAGES = pf_stages<MODE>(), NA = MODE == PF_UP ? 2 : 1;
	extern __shared__ unsigned char smem_dyn[];
	__shared__ __align__(8) uint64_t full[STAGES], empty[STAGES];
	unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)smem_dyn + 1023) & ~(uintptr_t)1023);
	const int tid = threadIdx.x, wg = tid >> 7, warp = tid >> 5, lane = tid & 31;
	const int row0 = blockIdx.x * PF_BM, tok0 = blockIdx.y * PF_BN;
	const int nkb = a.K / PF_BK;
	auto w_tile = [&](int s, int i) { return smem + (size_t)s * pf_stage_bytes<MODE>() + (size_t)i * PF_BM * 128; };
	auto x_tile = [&](int s, int i) { return smem + (size_t)s * pf_stage_bytes<MODE>() + (size_t)NA * PF_BM * 128 + (size_t)i * PF_BN * 128; };

	pdl_launch_next();
	if (tid == 0) {
		// full: the TMA thread's expect_tx arrival + one arrival per producer warp; empty: one arrival per consumer warp
		for (int s = 0; s < STAGES; ++s) mbar_init(&full[s], 1 + 4), mbar_init(&empty[s], 8);
		mbar_init_fence();
	}
	__syncthreads();
	pdl_wait_prev(); // activations (and, for the KV rows, the cache) come from the previous kernels of the layer

	if (wg == 0) {
		// ===== producers: one weight-tile row per thread, dequantised into the swizzled layout; thread 0 also brings in the
		// two activation tiles of every k-stage with TMA
		const int r = tid; // 0..127
		const unsigned char* rowp[NA];
		{
			const size_t rowbytes = (size_t)a.K * DBITS / 8;
			const int gr = row0 + r;
			if constexpr (MODE == PF_QKV) {
				const void* w = gr < a.q_dim ? a.w[0] : (gr < a.q_dim + a.kv_dim ? a.w[1] : a.w[2]);
				const int k = gr < a.q_dim ? gr : (gr < a.q_dim + a.kv_dim ? gr - a.q_dim : gr - a.q_dim - a.kv_dim);
				rowp[0] = reinterpret_cast<const unsigned char*>(w) + (size_t)k * rowbytes;
			} else if constexpr (MODE == PF_UP) {
				rowp[0] = reinterpret_cast<const unsigned char*>(a.w[0]) + (size_t)gr * rowbytes;
				rowp[1] = reinterpret_cast<const unsigned char*>(a.w[1]) + (size_t)gr * rowbytes;
			} else if constexpr (MODE == PF_CLS || MODE == PF_CLS_GREEDY || MODE == PF_CLS_TOPK) { // the last vocabulary tile may be partial: its spare rows repeat the last row
				rowp[0] = reinterpret_cast<const unsigned char*>(a.w[0]) + (size_t)min(gr, a.vocab - 1) * rowbytes;
			} else {
				rowp[0] = reinterpret_cast<const unsigned char*>(a.w[0]) + (size_t)gr * rowbytes;
			}
		}
		uint4 raw[NA][DBITS / 2];
#pragma unroll
		for (int i = 0; i < NA; ++i) pf_load_raw<DBITS>(rowp[i], 0, raw[i]);
		for (int kb = 0; kb < nkb; ++kb) {
			const int s = kb % STAGES;
			mbar_wait_guard(&empty[s], ((kb / STAGES) & 1) ^ 1);
			if (tid == 0) {
				mbar_expect_tx(&full[s], 2 * PF_BN * 128);
				tma_load_2d(x_tile(s, 0), &tm_hi, kb * PF_BK, tok0, &full[s]);
				tma_load_2d(x_tile(s, 1), &tm_lo, kb * PF_BK, tok0, &full[s]);
			}
#pragma unroll
			for (int i = 0; i < NA; ++i) pf_store_a<DBITS>(w_tile(s, i), r, raw[i]);
			if (kb + 1 < nkb) { // the next stage's bytes travel while this one is being multiplied
#pragma unroll
				for (int i = 0; i < NA; ++i) pf_load_raw<DBITS>(rowp[i], kb + 1, raw[i]);
			}
			fence_async_smem();
			__syncwarp();
			if (lane == 0) mbar_arrive(&full[s]);
		}
	} else {
		// ===== consumers: warpgroup c = wg - 1 multiplies tokens 64 c .. 64 c + 63 of the tile against all 128 weight rows
		const int c = wg - 1;
		float acc[NA][64];
#pragma unroll
		for (int i = 0; i < NA; ++i)
#pragma unroll
			for (int j = 0; j < 64; ++j) acc[i][j] = 0.f;
		for (int kb = 0; kb < nkb; ++kb) {
			const int s = kb % STAGES;
			mbar_wait_guard(&full[s], (kb / STAGES) & 1);
			wgmma_fence();
#pragma unroll
			for (int k = 0; k < PF_BK / 16; ++k) { // 16 f16 = 32 bytes along K inside the swizzle atom: +2 in the 16-byte address field
				const uint64_t dx_hi = wgmma_desc_sw128(x_tile(s, 0) + c * 64 * 128) + 2 * k, dx_lo = wgmma_desc_sw128(x_tile(s, 1) + c * 64 * 128) + 2 * k;
#pragma unroll
				for (int i = 0; i < NA; ++i) {
					const uint64_t dw = wgmma_desc_sw128(w_tile(s, i)) + 2 * k;
					wgmma_m64n128k16(acc[i], dx_hi, dw);
					wgmma_m64n128k16(acc[i], dx_lo, dw);
				}
			}
			wgmma_commit();
			wgmma_wait<1>(); // the MMAs of the previous stage have finished reading it
#pragma unroll
			for (int i = 0; i < NA; ++i) acc_fence(acc[i]);
			if (kb > 0 && lane == 0) mbar_arrive(&empty[(kb - 1) % STAGES]);
		}
		wgmma_wait<0>();
#pragma unroll
		for (int i = 0; i < NA; ++i) acc_fence(acc[i]);

		// accumulator fragment of m64nN: register 4 j + 2 h + e holds token 16 w + lane / 4 + 8 h, weight row 8 j + 2 (lane % 4) + e
		const int w4 = warp & 3;
		const int tb = tok0 + c * 64 + w4 * 16 + (lane >> 2);
		if constexpr (MODE == PF_CLS || MODE == PF_CLS_GREEDY || MODE == PF_CLS_TOPK) {
			// the quad of lanes 4 (lane / 4) .. + 3 holds all 128 logits of tokens tb and tb + 8: 32 per lane, then two shuffles.
			// Every lane runs the shuffles; only the stores are masked to the block's tokens.
			// PF_CLS_GREEDY also tracks gi, the vocabulary index of the first maximum: a lane's indices ascend with (j, e), so a
			// strict > keeps the lowest, and the shuffles give a tie to the lower index.  m and s take the same operations in
			// the same order as in PF_CLS, so the records are the same bits.
			// PF_CLS_TOPK computes m and s exactly as PF_CLS and then selects the tile's topk largest logits, one per round: each
			// lane offers its largest logit not yet taken (a strict > over ascending indices keeps the lowest index of equal
			// values), the quad's shuffles keep the larger value or, on equal values, the lower index, and the lane that owns
			// the winner marks it taken.
			const int q = lane & 3;
#pragma unroll
			for (int h = 0; h < 2; ++h) {
				const int t = tb + 8 * h;
				float m = -FLT_MAX;
				int gi = 0x7fffffff;
#pragma unroll
				for (int j = 0; j < PF_BM / 8; ++j)
#pragma unroll
					for (int e = 0; e < 2; ++e)
						if (row0 + 8 * j + 2 * q + e < a.vocab) {
							const float v = acc[0][4 * j + 2 * h + e];
							if constexpr (MODE == PF_CLS_GREEDY) gi = v > m ? row0 + 8 * j + 2 * q + e : gi;
							m = fmaxf(m, v);
						}
				if constexpr (MODE == PF_CLS_GREEDY) {
#pragma unroll
					for (int o = 1; o <= 2; o <<= 1) {
						const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
						const int i2 = __shfl_xor_sync(0xffffffffu, gi, o);
						if (m2 > m || (m2 == m && i2 < gi)) gi = i2;
						m = fmaxf(m, m2);
					}
				} else {
					m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
					m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
				}
				float s = 0.f;
#pragma unroll
				for (int j = 0; j < PF_BM / 8; ++j)
#pragma unroll
					for (int e = 0; e < 2; ++e)
						if (row0 + 8 * j + 2 * q + e < a.vocab) s += expf(acc[0][4 * j + 2 * h + e] - m);
				s += __shfl_xor_sync(0xffffffffu, s, 1);
				s += __shfl_xor_sync(0xffffffffu, s, 2);
				if (t < a.n_tokens) {
					const int tr = a.targets[t] - row0; // the target's row in this tile, if it lies here
#pragma unroll
					for (int j = 0; j < PF_BM / 8; ++j)
#pragma unroll
						for (int e = 0; e < 2; ++e)
							if (8 * j + 2 * q + e == tr) a.tgt[t] = acc[0][4 * j + 2 * h + e];
					if (q == 0) a.part[(size_t)t * gridDim.x + blockIdx.x] = make_float2(m, s);
					if constexpr (MODE == PF_CLS_GREEDY)
						if (q == 0) a.gidx[(size_t)t * gridDim.x + blockIdx.x] = gi;
				}
				if constexpr (MODE == PF_CLS_TOPK) {
					const size_t rec = ((size_t)t * gridDim.x + blockIdx.x) * a.topk;
					uint32_t taken = 0; // bit 2 j + e: this lane's logit of row 8 j + 2 q + e
					for (int r = 0; r < a.topk; ++r) {
						float bv = -INFINITY;
						int bi = INT_MAX, bp = 0;
#pragma unroll
						for (int j = 0; j < PF_BM / 8; ++j)
#pragma unroll
							for (int e = 0; e < 2; ++e) {
								const float v = acc[0][4 * j + 2 * h + e];
								if (row0 + 8 * j + 2 * q + e < a.vocab && !((taken >> (2 * j + e)) & 1u) && v > bv) bv = v, bi = row0 + 8 * j + 2 * q + e, bp = 2 * j + e;
							}
						const int mine = bi;
#pragma unroll
						for (int o = 1; o <= 2; o <<= 1) {
							const float v2 = __shfl_xor_sync(0xffffffffu, bv, o);
							const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
							if (v2 > bv || (v2 == bv && i2 < bi)) bv = v2, bi = i2;
						}
						if (bi == mine) taken |= 1u << bp; // (a lane with nothing left re-marks a taken or invalid bit)
						if (q == 0 && t < a.n_tokens) a.topv[rec + r] = bv, a.topi[rec + r] = bi;
					}
				}
			}
			return;
		}
#pragma unroll
		for (int j = 0; j < PF_BM / 8; ++j) {
			const int gr = row0 + 8 * j + 2 * (lane & 3); // even: (gr, gr + 1) is a RoPE pair
#pragma unroll
			for (int h = 0; h < 2; ++h) {
				const int t = tb + 8 * h;
				if (t >= a.n_tokens) continue;
				if constexpr (MODE == PF_QKV) {
					float x0 = acc[0][4 * j + 2 * h], x1 = acc[0][4 * j + 2 * h + 1];
					const bool is_q = gr < a.q_dim, is_k = !is_q && gr < a.q_dim + a.kv_dim;
					const int k = is_q ? gr : (is_k ? gr - a.q_dim : gr - a.q_dim - a.kv_dim);
					const int d = k % a.head_dim, hh = k / a.head_dim;
					if (a.bias) x0 += a.bias[gr], x1 += a.bias[gr + 1];
					x0 = fminf(fmaxf(x0, -a.clip), a.clip), x1 = fminf(fmaxf(x1, -a.clip), a.clip);
					if (is_q || is_k) {
						const float2 cs = a.rope[(size_t)t * (a.head_dim / 2) + (d >> 1)];
						const float r0 = fmaf(-x1, cs.y, x0 * cs.x), r1 = fmaf(x0, cs.y, x1 * cs.x);
						x0 = r0, x1 = r1;
					}
					if (is_q) {
						*reinterpret_cast<float2*>(a.Q + (size_t)t * a.q_dim + k) = make_float2(x0, x1);
					} else {
						KVT* dst = reinterpret_cast<KVT*>(is_k ? a.kc : a.vc) + ((size_t)hh * a.seq_len + a.pos0 + t) * a.head_dim + d;
						kv_store(dst, x0), kv_store(dst + 1, x1);
					}
				} else {
					pf_epilogue_pair<MODE>(a, gr, t, acc[0][4 * j + 2 * h], acc[0][4 * j + 2 * h + 1], acc[NA - 1][4 * j + 2 * h], acc[NA - 1][4 * j + 2 * h + 1]);
				}
			}
		}
	}
}

// ---------------------------------------------------------------- scoring: log-probability of each row's target
// One warp per token: merge the nvt (max, sum) records of the PF_CLS tiles, lane-strided and then by a butterfly, in an
// order fixed by nvt alone (no atomics), so that repeated calls give the same bits.  logprob = tgt - M - ln S with
// M = max m_v and S = sum s_v exp(m_v - M).
// GREEDY (after PF_CLS_GREEDY) also merges the tiles' argmax records gidx into greedy[t], the lowest vocabulary index of
// the maximum logit: lane-strided over ascending tiles a strict > keeps the first maximum, and in the butterfly an equal
// value takes the lower index, so the result does not depend on the merge order.  The (M, S) merge is unchanged.
// TOPK (after PF_CLS_TOPK) also merges the tiles' sorted top-k lists topv / topi [n][nvt][k] into the row's k largest
// logits: lane l owns tiles l, l + 32, .., with a head per tile in shared memory (how many of its entries are taken) and
// its best head in registers; each round a butterfly picks the largest value, the lower index on equal values, and the
// winning lane advances that tile and looks over its tiles again.  Indices are distinct, so the order of the merge does not
// matter.  top_ids[t][r] is the index and top_logprobs[t][r] = logit - M - ln S, the expression of logprob[t].
__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
	const float mn = fmaxf(m, m2);
	s = s * expf(m - mn) + s2 * expf(m2 - mn);
	m = mn;
}
template <bool GREEDY, bool TOPK = false>
__global__ void __launch_bounds__(256) k_pf_logprob(const float2* part, const float* tgt, float* logprob, int n, int nvt, const int* gidx, int* greedy,
                                                    const float* topv, const int* topi, int k, int* top_ids, float* top_logprobs) {
	pdl_enter();
	const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
	if (t >= n) return;
	const float2* p = part + (size_t)t * nvt;
	float m = -FLT_MAX, s = 0.f;
	int gi = 0x7fffffff;
	for (int v = lane; v < nvt; v += 32) {
		const float2 r = p[v];
		if constexpr (GREEDY)
			if (r.x > m) gi = gidx[(size_t)t * nvt + v];
		lse_merge(m, s, r.x, r.y);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) { // lane 0's result: a fixed tree over the lanes
		const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
		if constexpr (GREEDY) {
			const int i2 = __shfl_xor_sync(0xffffffffu, gi, o);
			if (m2 > m || (m2 == m && i2 < gi)) gi = i2;
		}
		lse_merge(m, s, m2, s2);
	}
	if (lane == 0) {
		logprob[t] = tgt[t] - m - logf(s);
		if constexpr (GREEDY) greedy[t] = gi;
	}
	if constexpr (TOPK) {
		extern __shared__ unsigned char pf_heads[]; // [8 warps][nvt]
		unsigned char* head = pf_heads + (threadIdx.x >> 5) * nvt;
		const float* tv = topv + (size_t)t * nvt * k;
		const int* ti = topi + (size_t)t * nvt * k;
		for (int v = lane; v < nvt; v += 32) head[v] = 0;
		float bv;
		int bi, bt;
		auto best_head = [&]() {
			bv = -INFINITY, bi = INT_MAX, bt = -1;
			for (int v = lane; v < nvt; v += 32) {
				const int h = head[v];
				if (h < k) {
					const float x = tv[(size_t)v * k + h];
					const int i = ti[(size_t)v * k + h];
					if (x > bv || (x == bv && i < bi)) bv = x, bi = i, bt = v;
				}
			}
		};
		best_head();
		for (int r = 0; r < k; ++r) {
			float wv = bv;
			int wi = bi;
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) {
				const float v2 = __shfl_xor_sync(0xffffffffu, wv, o);
				const int i2 = __shfl_xor_sync(0xffffffffu, wi, o);
				if (v2 > wv || (v2 == wv && i2 < wi)) wv = v2, wi = i2;
			}
			if (lane == 0) top_ids[(size_t)t * k + r] = wi, top_logprobs[(size_t)t * k + r] = wv - m - logf(s);
			if (wi == bi && bt >= 0) {
				++head[bt];
				best_head();
			}
		}
	}
}

// ---------------------------------------------------------------- causal attention of the block against the cache
#define PFA_WARPS 8
#define PFA_TILE 32 // keys per shared-memory tile: one per lane

struct PfAttnArgs {
	const float* Q; // [T][q_dim]
	const void* kc; // this layer
	const void* vc;
	__half* Ohi;    // [T][q_dim]
	__half* Olo;
	int n_tokens, pos0, seq_len, q_dim, kv_mul;
	float inv_sqrt_hd;
	const int* seg; // [T] (SEG variant) the first row of the row's sequence; read by no other variant
	const int2* ctx; // [T] (CTX variant) the row's context: its first row and its length (0: none); read by no other variant
};

// DPL (2 or 4) consecutive cache elements -> floats with a single shared-memory load
template <int DPL>
__device__ __forceinline__ void pf_load_dims(const __half* p, float (&o)[DPL]) {
	if constexpr (DPL == 4) {
		const uint2 r = *reinterpret_cast<const uint2*>(p);
		const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&r.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&r.y));
		o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y;
	} else {
		const float2 a = __half22float2(*reinterpret_cast<const __half2*>(p));
		o[0] = a.x, o[1] = a.y;
	}
}
template <int DPL>
__device__ __forceinline__ void pf_load_dims(const uint8_t* p, float (&o)[DPL]) {
	if constexpr (DPL == 4) {
		const uint32_t r = *reinterpret_cast<const uint32_t*>(p);
		const float2 a = e5m2x2_lo(r), b = e5m2x2_hi(r);
		o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y;
	} else {
		const uint32_t r = *reinterpret_cast<const unsigned short*>(p);
		const float2 a = e5m2x2_lo(r);
		o[0] = a.x, o[1] = a.y;
	}
}

// CTA = (kv head, 8 consecutive query tokens); warp = one token with all kv_mul query heads of the kv head (KM of them per pass).
// SEG: a packed block, row t in cache slot pos0 + t: the scoring calls' (score_batch, score_context; pos0 = 0), or one of
// decode_sample_batch's prompt blocks (pos0 = the block's first slot of the packed prompt region).  seg[] holds absolute
// cache slots.  The host starts every sequence at a multiple of 8 slots, so the CTA's rows share one segment starting at
// slot s = seg[first row], and the key tiles run from s: tile j of a sequence holds the same keys in the same order as tile
// j of the sequence run alone from position 0, and each warp's online softmax sees exactly the values of that lone pass.
// A sequence that straddles a block edge continues in the next block from the same s, whose slots the earlier block wrote.
// CTX (with SEG): a packed block that also holds contexts its sequences continue.  A CTA's rows start at
// row s and continue the nc-row context at rows c0 .. c0 + nc - 1 (ctx[first row]).  The keys run over one virtual index v:
// v < nc is row c0 + v, v >= nc is row s + v - nc; row t sees v <= nc + t - s.  A tile may straddle the two ranges, so each
// tile row finds its own address.  Tile j then holds the keys of tile j of ctx ++ sequence scored alone from position 0,
// with the same zero fill, visibility and value-loop bound, so every floating-point operation is that lone pass's.
template <typename KVT, int HD, int KM, bool SEG = false, bool CTX = false>
__global__ void __launch_bounds__(PFA_WARPS * 32) k_pf_attn(const PfAttnArgs a) {
	static_assert(SEG || !CTX, "the context walk starts from a segmented block");
	pdl_enter();
	constexpr int DPL = HD / 32;               // head dims owned by a lane in the value pass
	constexpr int KSTR = HD * sizeof(KVT) + 16; // padded key row: 16-byte reads of one row per lane are conflict-free per quarter warp
	__shared__ __align__(16) unsigned char ks[PFA_TILE * KSTR];
	__shared__ __align__(16) unsigned char vs[PFA_TILE * HD * sizeof(KVT)];
	__shared__ __align__(16) float qs[PFA_WARPS][KM * HD];
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
	const int kvh = blockIdx.y, t = blockIdx.x * PFA_WARPS + warp;
	const bool live = t < a.n_tokens;
	int last = a.pos0 + min(a.n_tokens - 1, (int)blockIdx.x * PFA_WARPS + PFA_WARPS - 1); // last key position any warp of the CTA needs
	int mypos = a.pos0 + t;
	int kfirst = 0; // first key slot of the CTA's rows
	if constexpr (SEG) {
		kfirst = a.seg[blockIdx.x * PFA_WARPS];
		// a CTA straddling two sequences would attend across them: stop instead (no message: a format string would move the
		// global-constant offsets every other kernel of the module is built with)
		if (live && a.seg[t] != kfirst) __trap();
		if constexpr (CTX) { // from here on, key positions are virtual indices
			const int nc = a.ctx[blockIdx.x * PFA_WARPS].y;
			last += nc - kfirst, mypos += nc - kfirst, kfirst = 0;
		}
	}
	const KVT* kbase = reinterpret_cast<const KVT*>(a.kc) + (size_t)kvh * a.seq_len * HD;
	const KVT* vbase = reinterpret_cast<const KVT*>(a.vc) + (size_t)kvh * a.seq_len * HD;
	for (int hg = 0; hg < a.kv_mul; hg += KM) { // KM query heads per pass over the keys
		const int h0 = kvh * a.kv_mul + hg;
		for (int i = lane; i < KM * HD; i += 32) qs[warp][i] = live ? a.Q[(size_t)t * a.q_dim + (size_t)h0 * HD + i] : 0.f;
		float m[KM], l[KM], acc[KM][DPL];
#pragma unroll
		for (int h = 0; h < KM; ++h) {
			m[h] = -FLT_MAX, l[h] = 0.f;
#pragma unroll
			for (int d = 0; d < DPL; ++d) acc[h][d] = 0.f;
		}
		for (int k0 = kfirst; k0 <= last; k0 += PFA_TILE) {
			__syncthreads(); // the previous tile is no longer being read
			for (int i = threadIdx.x; i < PFA_TILE * HD * (int)sizeof(KVT) / 16; i += blockDim.x) {
				const int row = i / (HD * (int)sizeof(KVT) / 16), c = i % (HD * (int)sizeof(KVT) / 16);
				const bool in = k0 + row <= last;
				int slot = k0 + row;
				if constexpr (CTX) { // (read per tile: held in registers through the score pass, they add spills)
					const int2 cx = __ldg(a.ctx + blockIdx.x * PFA_WARPS);
					slot = slot < cx.y ? cx.x + slot : __ldg(a.seg + blockIdx.x * PFA_WARPS) + slot - cx.y;
				}
				const uint4 z = make_uint4(0, 0, 0, 0);
				*reinterpret_cast<uint4*>(ks + row * KSTR + c * 16) = in ? __ldcg(reinterpret_cast<const uint4*>(kbase + (size_t)slot * HD) + c) : z;
				*reinterpret_cast<uint4*>(vs + row * HD * sizeof(KVT) + c * 16) = in ? __ldcg(reinterpret_cast<const uint4*>(vbase + (size_t)slot * HD) + c) : z;
			}
			__syncthreads();
			if (!live || k0 > mypos) continue; // (warp-uniform) causal: nothing of this tile is visible to this token
			const bool vis = k0 + lane <= mypos;
			// scores of key (k0 + lane) against the KM heads
			float sc[KM];
#pragma unroll
			for (int h = 0; h < KM; ++h) sc[h] = 0.f;
			const unsigned char* krow = ks + lane * KSTR;
#pragma unroll 4
			for (int c = 0; c < HD / 8; ++c) {
				float kf[8];
				kv_load8(reinterpret_cast<const KVT*>(krow) + c * 8, kf);
#pragma unroll
				for (int h = 0; h < KM; ++h) {
					const float4 q0 = *reinterpret_cast<const float4*>(&qs[warp][h * HD + c * 8]), q1 = *reinterpret_cast<const float4*>(&qs[warp][h * HD + c * 8 + 4]);
					float s = sc[h];
					s = fmaf(q0.x, kf[0], s), s = fmaf(q0.y, kf[1], s), s = fmaf(q0.z, kf[2], s), s = fmaf(q0.w, kf[3], s);
					s = fmaf(q1.x, kf[4], s), s = fmaf(q1.y, kf[5], s), s = fmaf(q1.z, kf[6], s), s = fmaf(q1.w, kf[7], s);
					sc[h] = s;
				}
			}
			float p[KM];
#pragma unroll
			for (int h = 0; h < KM; ++h) {
				const float s = vis ? sc[h] * a.inv_sqrt_hd : -FLT_MAX;
				const float mn = fmaxf(m[h], warp_max(s));
				const float corr = expf(m[h] - mn);
				p[h] = vis ? expf(s - mn) : 0.f;
				l[h] = fmaf(l[h], corr, warp_sum(p[h]));
				m[h] = mn;
#pragma unroll
				for (int d = 0; d < DPL; ++d) acc[h][d] *= corr;
			}
			// values: lane owns head dims [lane * DPL, lane * DPL + DPL)
			const int nk = min(PFA_TILE, mypos - k0 + 1);
			for (int j = 0; j < nk; ++j) {
				float vf[DPL];
				pf_load_dims<DPL>(reinterpret_cast<const KVT*>(vs) + (size_t)j * HD + lane * DPL, vf); // one 8- / 4- / 2-byte load
#pragma unroll
				for (int h = 0; h < KM; ++h) {
					const float pj = __shfl_sync(0xffffffffu, p[h], j);
#pragma unroll
					for (int d = 0; d < DPL; ++d) acc[h][d] = fmaf(pj, vf[d], acc[h][d]);
				}
			}
		}
		if (live) {
#pragma unroll
			for (int h = 0; h < KM; ++h) {
				const float inv = 1.0f / l[h];
#pragma unroll
				for (int d = 0; d < DPL; ++d) {
					__half hh, hl;
					split_hl(acc[h][d] * inv, hh, hl);
					const size_t o = (size_t)t * a.q_dim + (size_t)(h0 + h) * HD + lane * DPL + d;
					a.Ohi[o] = hh, a.Olo[o] = hl;
				}
			}
		}
		__syncwarp();
	}
}
