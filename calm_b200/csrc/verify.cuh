// verify.cuh -- the short-block GEMM of calm_b200_verify_greedy / _sample: the five projections of a layer and the classifier for a
// block of at most 16 tokens (a decode token and its drafts), streaming the weights over every SM as the decode does.
//
//   k_vf_gemm   out[rows][16 tokens] = W . X^T with mma.sync m16n8k16 (f16 in, fp32 accumulators): the weight rows are
//               the M side, 16 per warp fragment, dequantised in registers by the prompt pass's own fp16 / e5m2 /
//               gf4 -> f16 conversions (e5m2_word_h2, gf4_word_h2, as pf_store_a); the tokens are the N side, two n8 tiles, and the activations enter
//               as the pass's f16 hi + lo pair, two MMAs into one accumulator.  Inside a 64-wide k chunk, lane (g, t)
//               owns k = 16 t .. 16 t + 15 of its rows g and g + 8 (one contiguous load per row) and the MMA's k slots
//               are mapped onto those k in the same way for A and B, so every product still meets its own activation.
//               A task is (128 weight rows, one K-slice of VF_KS): the 16 rows of the block's activations for that
//               slice sit in shared memory, and a CTA keeps its slice while it walks its row blocks.  Each task writes
//               its fp32 partial sums; the CTA that completes a row block's last slice (an arrival counter, reset by
//               that CTA) adds the slices in ascending order and runs the epilogue of k_pf_gemm on the completed sums:
//               QKV bias / clip / RoPE / Q rows and KV append as k_pf_gemm writes it out, k_pf_gemm's pf_epilogue_pair
//               for the residual add (WO, DOWN) and act(w1 x) * (w3 x) split into hi + lo (UP), and for the classifier each 128-row vocabulary tile's (max, sum) and argmax records in the
//               layout PF_CLS_GREEDY writes, which the unchanged k_pf_logprob<true, false> merges.  Nothing is added
//               with atomics and the fold order is fixed, so repeated calls give the same bits.
//               PF_CLS_SAMPLE (calm_b200_verify_sample) is PF_CLS_GREEDY that also stores the fold's logits of every
//               token row, and each tile's maximum, which k_sample_scan_rows / k_sample_pick_rows (stages.cuh) sample,
//               all rows side by side: the same accumulator values the argmax records come from.
//               PF_QKV_SLOTS (calm_b200_decode_sample_queue) is PF_QKV with each row's keys and values at its own slot.
//               TOPK (with PF_CLS_GREEDY or PF_CLS_SAMPLE; calm_b200_decode_sample_queue_logprobs) computes every record
//               above with the same operations and then each tile's a.topk largest logits of every token row, in
//               PF_CLS_TOPK's layout and by its rule, which the unchanged k_pf_logprob<.., true> merges.
//               PEN (with TOPK, whose lists are empty at a.topk == 0; calm_b200_decode_sample_queue_penalties) replaces
//               each logit of a row whose v.lane[t] is non-negative by the request's processed logit (sq_pen_logit)
//               before any record is formed, so the argmax records, logit rows, tile maxima, (max, sum) records and top-k
//               lists all see the processed values.  Other rows are not touched.
//               MASK (with TOPK and PEN; calm_b200_decode_sample_queue_constrained) then sets to -inf each logit of a row
//               whose v.mstate[t] is non-negative at every token its automaton state does not allow (v.allow), in the
//               same pass, so every record sees the masked values.  A tile with no allowed entry gives (m = -FLT_MAX,
//               sum = 0, gi = INT_MAX), its top-k lists (-inf, INT_MAX).
#pragma once

#include "prefill.cuh"

#define VF_TOK 16     // tokens of a block: two n8 tiles (CALM_B200_VERIFY_MAX)
#define VF_ROWS 128   // weight rows per row block: 8 warps of 16; for the classifier one vocabulary tile (PF_BM)
#define VF_THREADS 256
#define VF_KS 512     // k per slice: 16 tokens x 512 x (hi + lo) f16 = 32 KB of shared memory
#define VF_XSTR (VF_KS + 8) // padded activation row (halves): a quarter warp's 16-byte reads hit distinct banks
#define VF_CLS_UNITS 256    // vocabulary tiles per classifier launch (bounds the partial-sum buffer)

struct VfArgs {
	const __half* xhi; // [>= 16][K] the block's activations, row t = token t
	const __half* xlo;
	float* acc;        // [nsl][rows][16] partial sums of each K-slice
	unsigned* cnt;     // [units] arrivals per row block; zero between launches (the folding CTA resets its own)
	int nsl;           // K-slices
	int units;         // row blocks; UP: hidden / 128, whose w1 and w3 rows are tasks of their own
	int rows;          // rows of the partial-sum layout (UP: 2 * hidden)
	int tile0, nvt;    // CLS: the first vocabulary tile of this launch, and the tiles of the vocabulary
	float* logits;     // PF_CLS_SAMPLE: [n_tokens][vocab] the logit rows
	float* tmax;       // PF_CLS_SAMPLE: [n_tokens][nvt] each tile's maximum logit (the sampler's cand_val)
	const int* slot;   // PF_QKV_SLOTS: [n_tokens] the cache slot of each row's keys and values
	// PEN: the lanes' state (sq_pen_logit), and row t's lane, or -1 for a row left as it is
	const int* lane;    // [VF_TOK] (k_sq_lanes)
	const int* pcnt;    // [16][vocab] count of the token among the request's generated tokens, | SQ_PEN_SEEN if in ctx ++ prompt
	const float* pbias; // [16][vocab] b(v): the request's logit bias, 0 off its list
	const float4* ppar; // [16] (presence, frequency, repetition, 0)
	// MASK: row t's automaton state, or -1 for a row left as it is, and the states' bitmasks
	const int* mstate;       // [VF_TOK] (k_sq_lanes)
	const uint32_t* allow;   // [n_states][ceil(vocab / 32)] bit v % 32 of word v / 32: token v is allowed
};

#define SQ_PEN_SEEN (1 << 30) // a count row's mark of a token in the request's ctx ++ prompt; the count is the bits below

// One logit of a non-neutral request through its processing (include/calm_b200.h), each operation one IEEE fp32
// operation rounded to nearest: w is the token's count word, b its bias, par (presence, frequency, repetition, 0).
__device__ __forceinline__ float sq_pen_logit(float l, int w, float b, float4 par) {
	const int c = w & (SQ_PEN_SEEN - 1);
	const float l1 = w != 0 && par.z != 1.0f ? (l > 0.0f ? __fdiv_rn(l, par.z) : __fmul_rn(l, par.z)) : l; // seen: in ctx ++ prompt, or c > 0
	const float a = __fsub_rn(__fsub_rn(b, __fmul_rn(par.y, (float)c)), c > 0 ? par.x : 0.0f);
	return a == 0.0f ? l1 : __fadd_rn(l1, a);
}

template <int DBITS>
struct VfFmt {
	static constexpr int WORDS = DBITS / 2; // 32-bit words of one lane's 16 weights of a row
	static constexpr int U = 16 / WORDS; // 64-wide k chunks per batch of loads: 2 rows x 16 words in flight per lane
};

__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
	asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
	             : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
	             : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// one lane's 16 consecutive weights of a row (k = k0 .. k0 + 15), raw
template <int DBITS>
__device__ __forceinline__ void vf_load(const unsigned char* row, int k0, uint32_t (&w)[VfFmt<DBITS>::WORDS]) {
	const unsigned char* p = row + (size_t)k0 * DBITS / 8;
	if constexpr (DBITS == 4) {
		const uint2 v = ldg_stream8(reinterpret_cast<const uint2*>(p));
		w[0] = v.x, w[1] = v.y;
	} else {
#pragma unroll
		for (int i = 0; i < DBITS / 8; ++i) {
			const uint4 v = ldg_stream(reinterpret_cast<const uint4*>(p) + i);
			w[4 * i] = v.x, w[4 * i + 1] = v.y, w[4 * i + 2] = v.z, w[4 * i + 3] = v.w;
		}
	}
}

// the same 16 weights as 8 f16 pairs in k order, through pf_store_a's conversions
template <int DBITS>
__device__ __forceinline__ void vf_dequant(const uint32_t (&w)[VfFmt<DBITS>::WORDS], uint32_t (&h)[8]) {
	if constexpr (DBITS == 16) {
#pragma unroll
		for (int i = 0; i < 8; ++i) h[i] = w[i];
	} else if constexpr (DBITS == 8) {
#pragma unroll
		for (int i = 0; i < 4; ++i) {
			const uint2 p = e5m2_word_h2(w[i]);
			h[2 * i] = p.x, h[2 * i + 1] = p.y;
		}
	} else {
#pragma unroll
		for (int j = 0; j < 2; ++j) {
			const uint4 p = gf4_word_h2(w[j]);
			h[4 * j] = p.x, h[4 * j + 1] = p.y, h[4 * j + 2] = p.z, h[4 * j + 3] = p.w;
		}
	}
}

template <int MODE, int DBITS, typename KVT, bool TOPK = false, bool PEN = false, bool MASK = false>
__global__ void __launch_bounds__(VF_THREADS, 2) k_vf_gemm(const PfGemmArgs a, const VfArgs v) {
	constexpr int W = VfFmt<DBITS>::WORDS, U = VfFmt<DBITS>::U;
	constexpr bool CLS = MODE == PF_CLS_GREEDY || MODE == PF_CLS_SAMPLE;
	static_assert(CLS || !TOPK, "the top-k lists are a classifier epilogue");
	static_assert(TOPK || !PEN, "the processed logits come with the top-k epilogue (a.topk may be 0)");
	static_assert(PEN || !MASK, "the mask comes with the processed logits (every lane may be -1)");
	__shared__ __align__(16) __half xs[2][VF_TOK][VF_XSTR];
	__shared__ unsigned last_s;
	const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
	const int s = blockIdx.y, k_lo = s * VF_KS, klen = min(VF_KS, a.K - k_lo), nch = klen / 64;
	const size_t rowbytes = (size_t)a.K * DBITS / 8;
	const int arrivals = MODE == PF_UP ? 2 * v.nsl : v.nsl;
	const int nunits = MODE == PF_UP ? 2 * v.units : v.units;

	// the weight row of partial-sum row r (this launch's numbering)
	auto row_ptr = [&](int r) -> const unsigned char* {
		if constexpr (MODE == PF_QKV || MODE == PF_QKV_SLOTS) {
			const void* w = r < a.q_dim ? a.w[0] : (r < a.q_dim + a.kv_dim ? a.w[1] : a.w[2]);
			const int k = r < a.q_dim ? r : (r < a.q_dim + a.kv_dim ? r - a.q_dim : r - a.q_dim - a.kv_dim);
			return reinterpret_cast<const unsigned char*>(w) + (size_t)k * rowbytes;
		} else if constexpr (MODE == PF_UP) {
			return reinterpret_cast<const unsigned char*>(r < a.hidden ? a.w[0] : a.w[1]) + (size_t)(r < a.hidden ? r : r - a.hidden) * rowbytes;
		} else if constexpr (CLS) { // the last vocabulary tile may be partial: its spare rows repeat the last row
			return reinterpret_cast<const unsigned char*>(a.w[0]) + (size_t)min(v.tile0 * VF_ROWS + r, a.vocab - 1) * rowbytes;
		} else {
			return reinterpret_cast<const unsigned char*>(a.w[0]) + (size_t)r * rowbytes;
		}
	};

	uint32_t raw[U][2][W];
	const unsigned char* rp[2];
	auto load_batch = [&](int c0) {
#pragma unroll
		for (int u = 0; u < U; ++u)
			if (c0 + u < nch)
#pragma unroll
				for (int i = 0; i < 2; ++i) vf_load<DBITS>(rp[i], k_lo + 64 * (c0 + u) + 16 * t4, raw[u][i]);
	};
	auto set_rows = [&](int unit) {
		const int r = unit * VF_ROWS + warp * 16 + g;
		rp[0] = row_ptr(r), rp[1] = row_ptr(r + 8);
	};

	// the first weights travel while the previous kernel drains and while the activations are staged
	pdl_launch_next();
	int unit = blockIdx.x;
	if (unit < nunits) set_rows(unit), load_batch(0);
	pdl_wait_prev();
	for (int i = tid; i < 2 * VF_TOK * (VF_KS / 8); i += VF_THREADS) {
		const int hl = i / (VF_TOK * (VF_KS / 8)), tok = i / (VF_KS / 8) % VF_TOK, c = i % (VF_KS / 8);
		uint4 x = make_uint4(0, 0, 0, 0);
		if (tok < a.n_tokens && 8 * c < klen) x = *reinterpret_cast<const uint4*>((hl ? v.xlo : v.xhi) + (size_t)tok * a.K + k_lo + 8 * c);
		*reinterpret_cast<uint4*>(&xs[hl][tok][8 * c]) = x;
	}
	__syncthreads();

	for (; unit < nunits; unit += gridDim.x) {
		float acc[2][4] = {};
		for (int c0 = 0; c0 < nch; c0 += U) {
			uint32_t cur[U][2][W];
#pragma unroll
			for (int u = 0; u < U; ++u)
#pragma unroll
				for (int i = 0; i < 2; ++i)
#pragma unroll
					for (int j = 0; j < W; ++j) cur[u][i][j] = raw[u][i][j];
			if (c0 + U < nch) load_batch(c0 + U);
#pragma unroll
			for (int u = 0; u < U; ++u) {
				if (c0 + u >= nch) break;
				const int kc = 64 * (c0 + u) + 16 * t4;
				uint32_t h0[8], h1[8];
				vf_dequant<DBITS>(cur[u][0], h0), vf_dequant<DBITS>(cur[u][1], h1);
				uint4 bx[2][2][2]; // [hi / lo][n tile][16-byte half]
#pragma unroll
				for (int hl = 0; hl < 2; ++hl)
#pragma unroll
					for (int nt = 0; nt < 2; ++nt) {
						const uint4* p = reinterpret_cast<const uint4*>(&xs[hl][8 * nt + g][kc]);
						bx[hl][nt][0] = p[0], bx[hl][nt][1] = p[1];
					}
#pragma unroll
				for (int st = 0; st < 4; ++st) { // MMA k slots (2 t4, 2 t4 + 1 | + 8, + 9) = k (4 st, 4 st + 1 | + 2, + 3) of the lane's 16
#pragma unroll
					for (int nt = 0; nt < 2; ++nt)
#pragma unroll
						for (int hl = 0; hl < 2; ++hl) {
							const uint4 q = bx[hl][nt][st >> 1];
							const uint32_t b0 = (st & 1) ? q.z : q.x, b1 = (st & 1) ? q.w : q.y;
							mma_m16n8k16(acc[nt], h0[2 * st], h1[2 * st], h0[2 * st + 1], h1[2 * st + 1], b0, b1);
						}
				}
			}
		}
		// partial sums: acc[nt][2 e + j] = row (g + 8 e), token 8 nt + 2 t4 + j
		{
			const int r = unit * VF_ROWS + warp * 16 + g;
#pragma unroll
			for (int nt = 0; nt < 2; ++nt)
#pragma unroll
				for (int e = 0; e < 2; ++e)
					__stcg(reinterpret_cast<float2*>(v.acc + ((size_t)s * v.rows + r + 8 * e) * VF_TOK + 8 * nt + 2 * t4), make_float2(acc[nt][2 * e], acc[nt][2 * e + 1]));
		}
		const int fu = MODE == PF_UP ? unit % v.units : unit; // the row block this task completes a slice of
		const int next = unit + gridDim.x;
		if (next < nunits) set_rows(next), load_batch(0); // the next task's first weights travel during the arrival and the fold
		__threadfence();
		__syncthreads();
		if (tid == 0) last_s = atomicAdd(v.cnt + fu, 1u) == (unsigned)arrivals - 1;
		__syncthreads();
		if (!last_s) continue;
		__threadfence();

		// ===== the fold: this CTA completed the row block's last slice.  Thread = row pair (2 rp, 2 rp + 1) x tokens 4 tq ..
		const int rp = tid & 63, tq = tid >> 6;
		const int r0 = fu * VF_ROWS + 2 * rp;
		float x[2][4] = {}, gt[2][4] = {};
		for (int sl = 0; sl < v.nsl; ++sl) {
#pragma unroll
			for (int e = 0; e < 2; ++e) {
				const float4 p = __ldcg(reinterpret_cast<const float4*>(v.acc + ((size_t)sl * v.rows + r0 + e) * VF_TOK + 4 * tq));
				x[e][0] += p.x, x[e][1] += p.y, x[e][2] += p.z, x[e][3] += p.w;
				if constexpr (MODE == PF_UP) {
					const float4 q = __ldcg(reinterpret_cast<const float4*>(v.acc + ((size_t)sl * v.rows + a.hidden + r0 + e) * VF_TOK + 4 * tq));
					gt[e][0] += q.x, gt[e][1] += q.y, gt[e][2] += q.z, gt[e][3] += q.w;
				}
			}
		}
		if (tid == 0) v.cnt[fu] = 0;
		if constexpr (CLS) {
			__shared__ float lg[VF_TOK][VF_ROWS];
#pragma unroll
			for (int j = 0; j < 4; ++j) lg[4 * tq + j][2 * rp] = x[0][j], lg[4 * tq + j][2 * rp + 1] = x[1][j];
			__syncthreads();
			if constexpr (PEN) { // consecutive threads on consecutive vocabulary entries of a row, so the lane rows load coalesced
				const int pbase = (v.tile0 + fu) * VF_ROWS;
				for (int e = tid; e < VF_TOK * VF_ROWS; e += VF_THREADS) {
					const int t = e / VF_ROWS, r = e % VF_ROWS, ln = v.lane[t];
					if (t < a.n_tokens && ln >= 0 && pbase + r < a.vocab) {
						const size_t o = (size_t)ln * a.vocab + pbase + r;
						lg[t][r] = sq_pen_logit(lg[t][r], v.pcnt[o], v.pbias[o], v.ppar[ln]);
					}
				}
				if constexpr (MASK) { // each entry by the thread that processed it; pbase is a multiple of 128, so a row's tile is 4 words
					const int words = (a.vocab + 31) >> 5;
					for (int e = tid; e < VF_TOK * VF_ROWS; e += VF_THREADS) {
						const int t = e / VF_ROWS, r = e % VF_ROWS, s = v.mstate[t];
						if (t < a.n_tokens && s >= 0 && pbase + r < a.vocab && !((v.allow[(size_t)s * words + ((pbase + r) >> 5)] >> (r & 31)) & 1u))
							lg[t][r] = -INFINITY;
					}
				}
				__syncthreads();
			}
			// warp w: tokens 2 w, 2 w + 1.  Lane: rows lane + 32 i, ascending, so a strict > keeps the lowest index of the
			// maximum; the butterfly gives a tie to the lower index.  Then sum exp(logit - max) over the tile's rows.
			const int tile = v.tile0 + fu, rbase = tile * VF_ROWS;
#pragma unroll
			for (int h = 0; h < 2; ++h) {
				const int t = 2 * warp + h;
				float m = -FLT_MAX;
				int gi = 0x7fffffff;
#pragma unroll
				for (int i = 0; i < 4; ++i) {
					const int r = lane + 32 * i;
					if (rbase + r < a.vocab && lg[t][r] > m) m = lg[t][r], gi = rbase + r;
				}
#pragma unroll
				for (int o = 1; o < 32; o <<= 1) {
					const float m2 = __shfl_xor_sync(0xffffffffu, m, o);
					const int i2 = __shfl_xor_sync(0xffffffffu, gi, o);
					if (m2 > m || (m2 == m && i2 < gi)) gi = i2;
					m = fmaxf(m, m2);
				}
				float sum = 0.f;
#pragma unroll
				for (int i = 0; i < 4; ++i) {
					const int r = lane + 32 * i;
					if (rbase + r < a.vocab) sum += expf(lg[t][r] - m);
				}
				sum = warp_sum(sum);
				if (lane == 0 && t < a.n_tokens) {
					a.part[(size_t)t * v.nvt + tile] = make_float2(m, sum);
					a.gidx[(size_t)t * v.nvt + tile] = gi;
					if (tile == 0) a.tgt[t] = lg[t][0]; // (the target is token 0: k_pf_logprob needs one, the caller reads only the argmax)
				}
				if constexpr (MODE == PF_CLS_SAMPLE) { // the same values out: the tile's logits, coalesced, and its maximum
					if (t < a.n_tokens) {
#pragma unroll
						for (int i = 0; i < 4; ++i) {
							const int r = lane + 32 * i;
							if (rbase + r < a.vocab) v.logits[(size_t)t * a.vocab + rbase + r] = lg[t][r];
						}
						if (lane == 0) v.tmax[(size_t)t * v.nvt + tile] = m;
					}
				}
			}
			if constexpr (TOPK) { // PF_CLS_TOPK's selection over the same logits, one per round: each lane offers its largest
				// logit not yet taken (a strict > over its ascending rows keeps the lowest index of equal values), the butterfly
				// keeps the larger value or, on equal values, the lower index, and the owner marks it taken.  The warp's two
				// tokens go through the rounds together, so that their independent butterflies overlap.
				const int tw = 2 * warp;
				if (tw < a.n_tokens) {
					uint32_t taken[2] = {0, 0}; // bit i: this lane's row lane + 32 i
					for (int r = 0; r < a.topk; ++r) {
						float bv[2];
						int bi[2], bp[2], mine[2];
#pragma unroll
						for (int h = 0; h < 2; ++h) {
							bv[h] = -INFINITY, bi[h] = INT_MAX, bp[h] = 0;
#pragma unroll
							for (int i = 0; i < 4; ++i) {
								const int rr = lane + 32 * i;
								const float x = lg[tw + h][rr];
								if (rbase + rr < a.vocab && !((taken[h] >> i) & 1u) && x > bv[h]) bv[h] = x, bi[h] = rbase + rr, bp[h] = i;
							}
							mine[h] = bi[h];
						}
#pragma unroll
						for (int o = 1; o < 32; o <<= 1)
#pragma unroll
							for (int h = 0; h < 2; ++h) {
								const float v2 = __shfl_xor_sync(0xffffffffu, bv[h], o);
								const int i2 = __shfl_xor_sync(0xffffffffu, bi[h], o);
								if (v2 > bv[h] || (v2 == bv[h] && i2 < bi[h])) bv[h] = v2, bi[h] = i2;
							}
#pragma unroll
						for (int h = 0; h < 2; ++h) {
							if (bi[h] == mine[h]) taken[h] |= 1u << bp[h]; // (a lane with nothing left re-marks a taken or invalid bit)
							const size_t rec = ((size_t)(tw + h) * v.nvt + tile) * a.topk;
							if (lane == 0 && tw + h < a.n_tokens) a.topv[rec + r] = bv[h], a.topi[rec + r] = bi[h];
						}
					}
				}
			}
			__syncthreads(); // lg is rewritten by this CTA's next fold only after this
		} else {
			const int gr = r0; // even: (gr, gr + 1) is a RoPE pair
#pragma unroll
			for (int j = 0; j < 4; ++j) {
				const int t = 4 * tq + j;
				if (t >= a.n_tokens) continue;
				if constexpr (MODE == PF_QKV || MODE == PF_QKV_SLOTS) {
					float x0 = x[0][j], x1 = x[1][j];
					const bool is_q = gr < a.q_dim, is_k = !is_q && gr < a.q_dim + a.kv_dim;
					const int k = is_q ? gr : (is_k ? gr - a.q_dim : gr - a.q_dim - a.kv_dim);
					const int d = k % a.head_dim, hh = k / a.head_dim;
					if (a.bias) x0 += a.bias[gr], x1 += a.bias[gr + 1];
					x0 = fminf(fmaxf(x0, -a.clip), a.clip), x1 = fminf(fmaxf(x1, -a.clip), a.clip);
					if (is_q || is_k) {
						const float2 cs = a.rope[(size_t)t * (a.head_dim / 2) + (d >> 1)];
						const float q0 = fmaf(-x1, cs.y, x0 * cs.x), q1 = fmaf(x0, cs.y, x1 * cs.x);
						x0 = q0, x1 = q1;
					}
					if (is_q) {
						*reinterpret_cast<float2*>(a.Q + (size_t)t * a.q_dim + k) = make_float2(x0, x1);
					} else {
						if constexpr (MODE == PF_QKV_SLOTS) { // (a statement of its own: PF_QKV's address arithmetic stays as it was)
							KVT* dst = reinterpret_cast<KVT*>(is_k ? a.kc : a.vc) + ((size_t)hh * a.seq_len + v.slot[t]) * a.head_dim + d;
							kv_store(dst, x0), kv_store(dst + 1, x1);
						} else {
							KVT* dst = reinterpret_cast<KVT*>(is_k ? a.kc : a.vc) + ((size_t)hh * a.seq_len + a.pos0 + t) * a.head_dim + d;
							kv_store(dst, x0), kv_store(dst + 1, x1);
						}
					}
				} else {
					pf_epilogue_pair<MODE>(a, gr, t, x[0][j], x[1][j], gt[0][j], gt[1][j]);
				}
			}
		}
	}
}
