// attn.cuh -- k_attn2: flash-decoding with the KV slice brought into shared memory by bulk TMA copies that are issued
// BEFORE the dependency wait, and the score and value passes run on the tensor cores.
//
// Why: the cache prefix of a layer is immutable while k_qkv of the same layer runs (k_qkv only writes slot kv_pos), so the
// attention kernel -- resident early thanks to programmatic dependent launch -- can request its whole K/V slice while the
// q/k/v matvec is still streaming weights.  When the dependency wait returns, the 16.8 MB a Llama-3-8B layer reads at
// position 4095 are already on chip, and what remains on the critical path is q -> scores -> softmax -> values out of
// shared memory (no DRAM round trips) plus the fold of the unit's slices.
//
// Work split: unit = kv head x group of HG query heads (as k_attn); the positions of a unit are cut into blocks of
// ATTN2_BP = 16 positions and dealt round-robin to the unit's `nsplit` CTAs (block b belongs to CTA b % nsplit), so the
// split is balanced for every kv_len and does NOT depend on kv_len -- which the pre-wait code only knows as a hint
// (TokenParams may still be about to be rewritten by the previous token's tail; the hint decides what to request early,
// never what is computed).  One mbarrier per block; a 16-position K block and V block are one bulk copy each
// ([position][head_dim] is contiguous per (layer, kv head)).  Once a block has landed, the positions its copy does not hold
// correctly are patched in shared memory (attn2_fix_block), so the passes below have no per-position cases.
//
// Arithmetic: mma.sync m16n8k16, f16 operands, f32 accumulators.  The M rows are the unit's query heads twice: row h holds
// the f16 hi part of head h, row HG + h its lo part (q = hi + lo to about 22 bits; a per-head power-of-two scale keeps hi
// in f16 range and is undone exactly on the score), and the two rows are added after each product.
//   scores  S = Q K^T: warps take blocks round-robin; N = 8 positions, K = 16 head dims per MMA, each lane reads 8
//           consecutive dims of its position with one load and feeds two MMAs (the dims of an MMA's K are a fixed
//           permutation of the head dims, the same for q and k).  Scaled scores go to shared memory.
//   softmax one warp per head: CTA-wide max, p = exp(s - max), sum; p is stored as f16 hi + lo rows again.
//   values  O = P V: warp w owns head dims [16 w, 16 w + 16) over all of the CTA's positions (N = 8 dims, K = one block);
//           V is transposed in registers (two rows -> one k-packed pair per dim).
// So the CTA's (m, l, acc) record comes out directly, without a merge of per-warp partials.  Reference arithmetic:
// infer.c:238-267.
#pragma once

#include "stages.cuh"

#define ATTN2_BP 16   // positions per block (one bulk copy of K, one of V)
#define ATTN2_MAXB 32 // blocks per CTA

// shared memory: K blocks | V blocks | scores [HG][np] f32 | probabilities hi / lo [2 HG][np + 8] f16 | this CTA's record
// [HG][head_dim + 2] f32, with np = nbmax * ATTN2_BP (the probability rows are padded so the 8 rows of an A fragment load
// fall in different banks)
template <typename KVT>
__host__ __device__ inline size_t attn2_smem_bytes(int hg, int head_dim, int nbmax) {
	const size_t np = (size_t)nbmax * ATTN2_BP;
	return 2 * np * head_dim * sizeof(KVT) + hg * np * sizeof(float) + 2 * hg * (np + 8) * sizeof(__half) + (size_t)hg * (head_dim + 2) * sizeof(float);
}

// The slices of a unit are folded like this: every CTA publishes its record as 8-byte {value, epoch} cells -- no fence, no
// atomic: a reader that sees the epoch sees the value -- and then normalises 1/nsplit of the unit's outputs itself, polling
// the cells of its peers (all CTAs of the grid are resident, so every cell arrives; a watchdog traps instead of hanging).
__device__ __forceinline__ float attn_cell_wait(const unsigned long long* cell, unsigned epoch, int* err) {
	unsigned long long v;
	unsigned spins = 0;
	unsigned long long t0 = 0;
	for (;;) {
		asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(cell) : "memory");
		if ((unsigned)(v >> 32) == epoch) break;
		if ((++spins & 1023) == 0) {
			const unsigned long long now = globaltimer_ns();
			if (!t0) t0 = now;
			if (now - t0 > 5000000000ull) { // 5 s: a slice never arrived -- fail loudly, never hang the GPU
				if (err) *reinterpret_cast<volatile int*>(err) = 9200;
				__threadfence_system();
				__trap();
			}
		}
	}
	return __uint_as_float((unsigned)v);
}

// two adjacent cells (16-byte aligned) with ONE poll: a slice's (m, l)
__device__ __forceinline__ void attn_cell_pair_wait(const unsigned long long* cell, unsigned epoch, int* err, float& v0, float& v1) {
	unsigned long long c0, c1;
	unsigned spins = 0;
	unsigned long long t0 = 0;
	for (;;) {
		asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(c0), "=l"(c1) : "l"(cell) : "memory");
		if ((unsigned)(c0 >> 32) == epoch && (unsigned)(c1 >> 32) == epoch) break;
		if ((++spins & 1023) == 0) {
			const unsigned long long now = globaltimer_ns();
			if (!t0) t0 = now;
			if (now - t0 > 5000000000ull) {
				if (err) *reinterpret_cast<volatile int*>(err) = 9201;
				__threadfence_system();
				__trap();
			}
		}
	}
	v0 = __uint_as_float((unsigned)c0), v1 = __uint_as_float((unsigned)c1);
}

// d += A B, m16n8k16, f16 x f16 -> f32
__device__ __forceinline__ void mma_f16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
	asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
	    : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
	    : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Cache elements -> f16 MMA operands.  e5m2 is the high byte of an f16, so its expansion is a byte permutation (exact).
template <typename KVT>
struct KvMma;
template <>
struct KvMma<__half> {
	// 8 consecutive dims of one position -> 4 pairs (dims 0-1, 2-3, 4-5, 6-7)
	static __device__ __forceinline__ void dims8(const __half* p, uint32_t (&w)[4]) {
		const uint4 r = *reinterpret_cast<const uint4*>(p);
		w[0] = r.x, w[1] = r.y, w[2] = r.z, w[3] = r.w;
	}
	// dims (d, d + 1) of positions p and p + 1 -> (V[p][d], V[p+1][d]) and (V[p][d+1], V[p+1][d+1])
	static __device__ __forceinline__ void pos2(const __half* p0, const __half* p1, uint32_t& b0, uint32_t& b1) {
		const uint32_t x = *reinterpret_cast<const uint32_t*>(p0), y = *reinterpret_cast<const uint32_t*>(p1);
		b0 = __byte_perm(x, y, 0x5410), b1 = __byte_perm(x, y, 0x7632);
	}
};
template <>
struct KvMma<uint8_t> {
	static __device__ __forceinline__ void dims8(const uint8_t* p, uint32_t (&w)[4]) {
		const uint2 r = *reinterpret_cast<const uint2*>(p);
		w[0] = __byte_perm(r.x, 0, 0x1404), w[1] = __byte_perm(r.x, 0, 0x3424);
		w[2] = __byte_perm(r.y, 0, 0x1404), w[3] = __byte_perm(r.y, 0, 0x3424);
	}
	static __device__ __forceinline__ void pos2(const uint8_t* p0, const uint8_t* p1, uint32_t& b0, uint32_t& b1) {
		const uint32_t x = *reinterpret_cast<const uint16_t*>(p0), y = *reinterpret_cast<const uint16_t*>(p1); // bytes 2, 3 are zero
		b0 = __byte_perm(x, y, 0x4202), b1 = __byte_perm(x, y, 0x5212);
	}
};

// One warp patches the shared-memory copy of block [t0, t0 + ATTN2_BP) once it has landed: the slot k_qkv wrote this token
// and the sinks k_embed re-rotated are not in the early copy (read from global memory), and V rows at positions >= kv_len are
// zeroed -- their probability is 0, but the cache there need not hold finite values, and inside an MMA 0 * NaN = NaN.
template <typename KVT, int HD>
__device__ __forceinline__ void attn2_fix_block(KVT* kb, KVT* vb, const KVT* kglob, const KVT* vglob, int t0, int kv_len, int kv_pos, int kv_sink, int lane) {
	constexpr int PPR = HD * (int)sizeof(KVT) / 16; // 16-byte pieces per row
	for (int i = lane; i < ATTN2_BP * PPR; i += 32) {
		const int o = i / PPR, t = t0 + o;
		uint4* ks = reinterpret_cast<uint4*>(kb + (size_t)o * HD) + i % PPR;
		uint4* vs = reinterpret_cast<uint4*>(vb + (size_t)o * HD) + i % PPR;
		if (t >= kv_len) {
			*vs = make_uint4(0, 0, 0, 0);
		} else if (t == kv_pos || t < kv_sink) {
			*ks = __ldcg(reinterpret_cast<const uint4*>(kglob + (size_t)t * HD) + i % PPR);
			*vs = __ldcg(reinterpret_cast<const uint4*>(vglob + (size_t)t * HD) + i % PPR);
		}
	}
}

template <typename KVT, int HG, int HD>
__global__ void __launch_bounds__(ATTN_THREADS, 1) k_attn2(__grid_constant__ const AttnArgs a) {
	constexpr int NW = ATTN_THREADS / 32, KS = HD / 16, NVW = HD / 16, REC = HD + 2;
	static_assert((HG == 2 || HG == 4 || HG == 8) && (HD == 64 || HD == 128) && NVW <= NW, "unsupported attention shape");
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ __align__(8) uint64_t bars[ATTN2_MAXB];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int g = lane >> 2, t4 = lane & 3; // MMA fragment coordinates: row / column group
	const int nbmax = a.nbmax, nsplit = a.nsplit, np = nbmax * ATTN2_BP, PS = np + 8;
	const int unit = blockIdx.x / nsplit, split = blockIdx.x % nsplit;
	const int kvh = unit / a.qgroups;
	const int hbase = kvh * a.kv_mul + (unit % a.qgroups) * HG;
	KVT* Ks = reinterpret_cast<KVT*>(smem_raw);
	KVT* Vs = Ks + (size_t)np * HD;
	float* S = reinterpret_cast<float*>(Vs + (size_t)np * HD); // [HG][np]
	__half* Ph = reinterpret_cast<__half*>(S + HG * np);        // [2 HG][PS]
	float* myrec = reinterpret_cast<float*>(Ph + 2 * HG * PS);  // [HG][REC]
	const KVT* kglob = reinterpret_cast<const KVT*>(a.kc) + (size_t)kvh * a.seq_len * HD;
	const KVT* vglob = reinterpret_cast<const KVT*>(a.vc) + (size_t)kvh * a.seq_len * HD;

#define ATTN_DBG(i)                                                          \
	do {                                                                     \
		if (a.dbg && blockIdx.x == 0 && tid == 0) a.dbg[i] = globaltimer_ns(); \
	} while (0)
	ATTN_DBG(0);
	pdl_launch_next();
	if (tid == 0) {
		for (int j = 0; j < nbmax; ++j) mbar_init(&bars[j], 1);
		mbar_init_fence();
	}
	__syncthreads();
	// request the slice while the previous kernel (k_qkv of this layer) is still running: thread j owns block j
	bool issued = false;
	auto request = [&](int j) {
		const int b = split + j * nsplit;
		const uint32_t bytes = (uint32_t)min(ATTN2_BP, a.seq_len - b * ATTN2_BP) * HD * sizeof(KVT);
		mbar_expect_tx(&bars[j], 2 * bytes);
		tma_load_1d(Ks + (size_t)j * ATTN2_BP * HD, kglob + (size_t)b * ATTN2_BP * HD, bytes, &bars[j]);
		tma_load_1d(Vs + (size_t)j * ATTN2_BP * HD, vglob + (size_t)b * ATTN2_BP * HD, bytes, &bars[j]);
	};
	if (tid < nbmax) {
		const int hint = min(*reinterpret_cast<const volatile int*>(&a.tp->kv_len), a.seq_len);
		if ((split + tid * nsplit) * ATTN2_BP < hint) request(tid), issued = true;
	}
	pdl_wait_prev();
	stamp_begin(a.stamp);
	ATTN_DBG(1);
	if (a.dbg && tid == 0) atomicMin(a.dbg + 10, globaltimer_ns());
	// this lane's query values: head g % HG (rows g and g + 8 of the A operand are the hi / lo parts of one head when HG = 8;
	// when HG < 8, row g < HG is hi, HG <= g < 2 HG lo, the rest zero), dims 32 c + 8 t4 + [0, 8) -- the quad of lanes with the
	// same g holds the whole head; q and the token parameters are requested together (one L2 round trip, not two)
	const int hq = g % HG;
	const bool qrow = g < 2 * HG;
	float qv[HD / 32][8];
#pragma unroll
	for (int c = 0; c < HD / 32; ++c) {
		float4 x0 = make_float4(0.f, 0.f, 0.f, 0.f), x1 = x0;
		if (qrow) {
			const float4* qp = reinterpret_cast<const float4*>(a.q + (size_t)(hbase + hq) * HD + 32 * c + 8 * t4);
			x0 = __ldcg(qp), x1 = __ldcg(qp + 1);
		}
		qv[c][0] = x0.x, qv[c][1] = x0.y, qv[c][2] = x0.z, qv[c][3] = x0.w, qv[c][4] = x1.x, qv[c][5] = x1.y, qv[c][6] = x1.z, qv[c][7] = x1.w;
	}
	const int kv_len = a.tp->kv_len, kv_pos = a.tp->kv_pos, kv_sink = a.tp->kv_sink;
	const unsigned epoch = (unsigned)a.tp->tp_seq * a.epoch_stride + a.epoch_idx;
	if (tid < nbmax && !issued && (split + tid * nsplit) * ATTN2_BP < kv_len) request(tid), issued = true;
	// per-head power-of-two scale: max |q| * scale in [2^13, 2^14), so hi never overflows f16 and lo stays normal; the score
	// multiplier inv = inv_sqrt_hd / scale undoes it exactly
	float qmax = 0.f;
#pragma unroll
	for (int c = 0; c < HD / 32; ++c)
#pragma unroll
		for (int i = 0; i < 8; ++i) qmax = fmaxf(qmax, fabsf(qv[c][i]));
	qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, 1));
	qmax = fmaxf(qmax, __shfl_xor_sync(0xffffffffu, qmax, 2));
	// (qmax = 2^e * [0.5, 1) for the biased exponent e + 126; the shift is bounded only so that both powers of two stay normal)
	const int qsh = min(max(14 - ((int)((__float_as_uint(qmax) >> 23) & 0xff) - 126), -100), 100);
	const float qscale = __uint_as_float((uint32_t)(127 + qsh) << 23), inv = a.inv_sqrt_hd * __uint_as_float((uint32_t)(127 - qsh) << 23);
	// A fragments of the score MMAs; step s = 2 c + e covers dims 32 c + 8 t4 + 4 e + [0, 4): (0, 1) in column pair t4, (2, 3) in t4 + 4
	uint32_t qa[KS][4];
#pragma unroll
	for (int c = 0; c < HD / 32; ++c)
#pragma unroll
		for (int e = 0; e < 2; ++e) {
			uint32_t hw[2], lw[2]; // dims (0, 1) and (2, 3) of the step
#pragma unroll
			for (int k = 0; k < 2; ++k) {
				__half h0, l0, h1, l1;
				split_hl(qv[c][4 * e + 2 * k] * qscale, h0, l0);
				split_hl(qv[c][4 * e + 2 * k + 1] * qscale, h1, l1);
				hw[k] = pack_h2(h0, h1), lw[k] = pack_h2(l0, l1);
			}
			uint32_t* f = qa[2 * c + e];
			if (HG == 8) { // row g: hi, row g + 8: lo
				f[0] = hw[0], f[2] = hw[1], f[1] = lw[0], f[3] = lw[1];
			} else {
				f[0] = !qrow ? 0u : g < HG ? hw[0] : lw[0];
				f[2] = !qrow ? 0u : g < HG ? hw[1] : lw[1];
				f[1] = f[3] = 0u;
			}
		}
	ATTN_DBG(2);

	// blocks of this CTA that hold cached positions
	const int nblk = (kv_len + ATTN2_BP - 1) / ATTN2_BP;
	const int nb = nblk > split ? (nblk - split + nsplit - 1) / nsplit : 0;
	const int nslots = nb * ATTN2_BP;
	if (a.dbg && blockIdx.x == 0 && tid == 0) { // debug: when the last of CTA 0's blocks landed (splits the passes into waiting for bytes and arithmetic)
		for (int j = 0; j < nb; ++j) mbar_wait(&bars[j], 0);
		a.dbg[8] = globaltimer_ns();
	}

	// ---- scores: block j is warp j % NW's; lane (g, t4) reads position 8 u + g of the block
	for (int j = warp; j < nb; j += NW) {
		mbar_wait(&bars[j], 0);
		if (j == 0) ATTN_DBG(3);
		const int t0 = (split + j * nsplit) * ATTN2_BP;
		KVT* kb = Ks + (size_t)j * ATTN2_BP * HD;
		if ((kv_pos >= t0 && kv_pos < t0 + ATTN2_BP) || t0 < kv_sink || t0 + ATTN2_BP > kv_len) {
			attn2_fix_block<KVT, HD>(kb, Vs + (size_t)j * ATTN2_BP * HD, kglob, vglob, t0, kv_len, kv_pos, kv_sink, lane);
			__syncwarp();
		}
#pragma unroll
		for (int u = 0; u < 2; ++u) {
			float sc[4] = {0.f, 0.f, 0.f, 0.f};
			const KVT* kr = kb + (size_t)(8 * u + g) * HD + 8 * t4;
#pragma unroll
			for (int c = 0; c < HD / 32; ++c) {
				uint32_t w[4];
				KvMma<KVT>::dims8(kr + 32 * c, w);
				mma_f16_16816(sc, qa[2 * c], w[0], w[1]);
				mma_f16_16816(sc, qa[2 * c + 1], w[2], w[3]);
			}
			// head g's score = row g (hi) + row HG + g (lo); lane (g, t4) holds positions 8 u + 2 t4 + {0, 1}
			float s0, s1;
			if (HG == 8) s0 = sc[0] + sc[2], s1 = sc[1] + sc[3];
			else s0 = sc[0] + __shfl_xor_sync(0xffffffffu, sc[0], 4 * HG), s1 = sc[1] + __shfl_xor_sync(0xffffffffu, sc[1], 4 * HG);
			const int o = 8 * u + 2 * t4;
			if (g < HG)
				*reinterpret_cast<float2*>(S + g * np + j * ATTN2_BP + o) = make_float2(t0 + o < kv_len ? s0 * inv : -FLT_MAX, t0 + o + 1 < kv_len ? s1 * inv : -FLT_MAX);
		}
	}
	__syncthreads();

	// ---- softmax: warp h owns head h
	if (warp < HG) {
		const float* sh = S + warp * np;
		float mx = -FLT_MAX;
		for (int i = lane; i < nslots; i += 32) mx = fmaxf(mx, sh[i]);
#pragma unroll
		for (int o = 16; o >= 1; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
		float sum = 0.f;
		for (int i = lane; i < nslots; i += 32) {
			const float p = __expf(sh[i] - mx);
			sum += p;
			split_hl(p, Ph[warp * PS + i], Ph[(HG + warp) * PS + i]);
		}
#pragma unroll
		for (int o = 16; o >= 1; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
		if (lane == 0) myrec[warp * REC + HD] = mx, myrec[warp * REC + HD + 1] = sum;
	}
	__syncthreads();
	ATTN_DBG(11);

	// ---- values: warp w owns dims [16 w, 16 w + 16); MMA u's column g is dim 16 w + 2 g + u, its K is the 16 positions of a block
	if (warp < NVW) {
		const int d0 = 16 * warp;
		float oc[2][4] = {};
		const __half* pr0 = Ph + g * PS + 2 * t4;
		const __half* pr1 = Ph + (g + 8) * PS + 2 * t4;
		for (int j = 0; j < nb; ++j) {
			mbar_wait(&bars[j], 0); // (completed: its score warp has seen it; this makes the bulk copy visible to this warp too)
			uint32_t pa[4];
			pa[0] = qrow ? *reinterpret_cast<const uint32_t*>(pr0 + j * ATTN2_BP) : 0u;
			pa[2] = qrow ? *reinterpret_cast<const uint32_t*>(pr0 + j * ATTN2_BP + 8) : 0u;
			pa[1] = HG == 8 ? *reinterpret_cast<const uint32_t*>(pr1 + j * ATTN2_BP) : 0u;
			pa[3] = HG == 8 ? *reinterpret_cast<const uint32_t*>(pr1 + j * ATTN2_BP + 8) : 0u;
			const KVT* vr = Vs + (size_t)(j * ATTN2_BP + 2 * t4) * HD + d0 + 2 * g;
			uint32_t b00, b10, b01, b11; // b<u><k half>
			KvMma<KVT>::pos2(vr, vr + HD, b00, b10);
			KvMma<KVT>::pos2(vr + 8 * HD, vr + 9 * HD, b01, b11);
			mma_f16_16816(oc[0], pa, b00, b01);
			mma_f16_16816(oc[1], pa, b10, b11);
		}
		// head g = row g (hi) + row HG + g (lo); lane (g, t4) holds columns 2 t4, 2 t4 + 1 = dims d0 + 4 t4 + u, d0 + 4 t4 + 2 + u
#pragma unroll
		for (int u = 0; u < 2; ++u) {
			float v0, v1;
			if (HG == 8) v0 = oc[u][0] + oc[u][2], v1 = oc[u][1] + oc[u][3];
			else v0 = oc[u][0] + __shfl_xor_sync(0xffffffffu, oc[u][0], 4 * HG), v1 = oc[u][1] + __shfl_xor_sync(0xffffffffu, oc[u][1], 4 * HG);
			if (g < HG) myrec[g * REC + d0 + 4 * t4 + u] = v0, myrec[g * REC + d0 + 4 * t4 + 2 + u] = v1;
		}
	}
	__syncthreads();
	ATTN_DBG(4);

	// ---- fold the unit's slices
	__shared__ float mls[ATTN2_MAXB + 4][HG][2]; // (m, l) of every slice, then the coefficient in place  (nsplit <= 36)
	__shared__ float invl[HG];
	unsigned long long* cells = a.cells + (size_t)unit * nsplit * HG * REC;
	for (int i = tid; i < HG * REC; i += ATTN_THREADS) { // publish: ONE 8-byte store per value
		const unsigned long long c = ((unsigned long long)epoch << 32) | __float_as_uint(myrec[i]);
		asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(cells + (size_t)split * HG * REC + i), "l"(c) : "memory");
	}
	for (int i = tid; i < nsplit * HG; i += ATTN_THREADS) {
		const int s = i / HG, h = i % HG;
		const unsigned long long* c = cells + (size_t)s * HG * REC + h * REC + HD;
		if (s == split) mls[s][h][0] = myrec[h * REC + HD], mls[s][h][1] = myrec[h * REC + HD + 1];
		else attn_cell_pair_wait(c, epoch, a.err, mls[s][h][0], mls[s][h][1]); // (REC and HD are even: the pair is 16-byte aligned)
	}
	__syncthreads();
	__shared__ float cfs[ATTN2_MAXB + 4][HG]; // exp(m_s - M): one exponential per (slice, head), in parallel
	for (int i = tid; i < nsplit * HG; i += ATTN_THREADS) {
		const int s = i / HG, h = i % HG;
		float M = -FLT_MAX;
		for (int s2 = 0; s2 < nsplit; ++s2) M = fmaxf(M, mls[s2][h][0]);
		cfs[s][h] = expf(mls[s][h][0] - M);
	}
	__syncthreads();
	if (tid < HG) {
		float L = 0.f;
		for (int s = 0; s < nsplit; ++s) L = fmaf(mls[s][tid][1], cfs[s][tid], L); // slice order: deterministic
		invl[tid] = 1.0f / L;
	}
	for (int i = tid; i < nsplit * HG; i += ATTN_THREADS) mls[i / HG][i % HG][0] = cfs[i / HG][i % HG]; // the output loop reads the coefficient from mls
	__syncthreads();
	ATTN_DBG(6);
	// CTA `split` normalises outputs [split * per, (split + 1) * per): 8 adjacent lanes share an output, each sums every 8th slice
	const int nout = HG * HD, per = (nout + nsplit - 1) / nsplit;
	const int o_end = min(nout, (split + 1) * per);
	for (int o0 = split * per; o0 < o_end; o0 += ATTN_THREADS / 8) {
		const int o = o0 + tid / 8, sg = tid & 7;
		float v = 0.f;
		if (o < o_end) {
			const int h = o / HD, e = o % HD;
			// all of this lane's cells are requested before the first is looked at (their slices' (m, l) have been seen: they are
			// almost always there) -- one L2 round trip instead of one per slice; a cell that is not there yet is polled as before
			constexpr int NS8 = (ATTN2_MAXB + 4 + 7) / 8;
			unsigned long long c[NS8];
#pragma unroll
			for (int k = 0; k < NS8; ++k) {
				const int s = sg + 8 * k;
				c[k] = 0;
				if (s < nsplit && s != split) asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(c[k]) : "l"(cells + (size_t)s * HG * REC + h * REC + e) : "memory");
			}
#pragma unroll
			for (int k = 0; k < NS8; ++k) {
				const int s = sg + 8 * k;
				if (s < nsplit) {
					float x;
					if (s == split) x = myrec[h * REC + e];
					else if ((unsigned)(c[k] >> 32) == epoch) x = __uint_as_float((unsigned)c[k]);
					else x = attn_cell_wait(cells + (size_t)s * HG * REC + h * REC + e, epoch, a.err);
					v = fmaf(x, mls[s][h][0], v); // slice order per lane: deterministic
				}
			}
		}
		v += __shfl_xor_sync(0xffffffffu, v, 1), v += __shfl_xor_sync(0xffffffffu, v, 2), v += __shfl_xor_sync(0xffffffffu, v, 4);
		if (o < o_end && sg == 0) __stcg(a.out + (size_t)hbase * HD + o, v * invl[o / HD]);
	}
	// no bulk copy may still be in flight into this CTA's shared memory when it exits (a block requested on a stale hint)
	if (tid < nbmax && issued) mbar_wait(&bars[tid], 0);
	ATTN_DBG(7);
	if (a.dbg && tid == 0) atomicMax(a.dbg + 9, globaltimer_ns());
	stamp_end(a.stamp);
}
