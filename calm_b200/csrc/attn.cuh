// attn.cuh -- k_attn2: flash-decoding with the KV slice brought into shared memory by bulk TMA copies that are issued
// BEFORE the dependency wait.
//
// Why: the cache prefix of a layer is immutable while k_qkv of the same layer runs (k_qkv only writes slot kv_pos), so the
// attention kernel -- resident early thanks to programmatic dependent launch -- can request its whole K/V slice while the
// q/k/v matvec is still streaming weights.  When the dependency wait returns, the 16.8 MB a Llama-3-8B layer reads at
// position 4095 are already on chip, and what remains on the critical path is q -> scores -> softmax -> values out of
// shared memory (no DRAM round trips) plus the slice merge of stages.cuh (attn_tail).
//
// Work split: unit = kv head x group of HG query heads (as k_attn); the positions of a unit are cut into blocks of
// ATTN2_BP = 16 positions and dealt round-robin to the unit's `nsplit` CTAs (block b belongs to CTA b % nsplit), so the
// split is balanced for every kv_len and does NOT depend on kv_len -- which the pre-wait code only knows as a hint
// (TokenParams may still be about to be rewritten by the previous token's tail; the hint decides what to request early,
// never what is computed).  One mbarrier per block; a 16-position K block and V block are one bulk copy each
// ([position][head_dim] is contiguous per (layer, kv head)).  The slot written this step and the attention sinks that
// k_embed re-rotates are read from global memory after the wait instead of from the early copy.
//
// Lane layout and arithmetic are k_attn's transposing score path: LPP = head_dim / 8 lanes own a position (8 dims per
// lane), P = LPP / HG positions per lane group and step, so the HG * P partial dot products of a step transpose onto the
// LPP lanes of the group (one complete score per lane), the two exponentials are evaluated once per lane, and the
// probabilities are broadcast back for the value accumulation.  Reference arithmetic: infer.c:238-267.
#pragma once

#include "stages.cuh"

#define ATTN2_BP 16   // positions per block (one bulk copy of K, one of V)
#define ATTN2_MAXB 32 // blocks per CTA

// ---- thread-block cluster helpers (the CTAs of a unit form one cluster when CLUSTER: nsplit <= 16)
__device__ __forceinline__ void cluster_sync_all() { // every thread of every CTA of the cluster; release / acquire at cluster scope
	asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
	asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ float ld_dsmem(const float* local_ptr, uint32_t cta_rank) { // the same shared-memory location in CTA `cta_rank` of this cluster
	uint32_t raddr;
	float v;
	asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(smem_u32(local_ptr)), "r"(cta_rank));
	asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(raddr) : "memory");
	return v;
}

#define ATTN2_MAX_CLUSTER 16

// shared memory: K blocks | V blocks | q [HG][head_dim] | merge scratch | this CTA's merged record [HG][head_dim + 2]
template <typename KVT>
__host__ __device__ inline size_t attn2_smem_bytes(int hg, int head_dim, int nbmax, int nsplit) {
	size_t kv = (size_t)2 * nbmax * ATTN2_BP * head_dim * sizeof(KVT);
	size_t scratch = (size_t)(ATTN_THREADS / 32) * hg * (head_dim + 2);
	size_t scratch2 = (size_t)(2 * nsplit + 1) * hg;
	if (scratch2 > scratch) scratch = scratch2;
	return kv + ((size_t)hg * head_dim + scratch + (size_t)hg * (head_dim + 2)) * sizeof(float);
}

// How the slices of a unit are folded (with global partials, a grid-scope fence, an atomic counter and a last-CTA pass the
// fold is a serial tail on the last CTA):
//   CLUSTER = false (default): every CTA publishes its record as 8-byte {value, epoch} cells -- no fence, no atomic: a reader
//     that sees the epoch sees the value -- and then normalises 1/nsplit of the unit's outputs itself, polling the cells
//     of its peers (all CTAs of the grid are resident, so every cell arrives; a watchdog traps instead of hanging).
//   CLUSTER = true: the nsplit CTAs of a unit are one thread-block cluster and read each other's records through
//     distributed shared memory (a 16-CTA cluster has to wait for 16 free SMs of one GPC; kept selectable, off by default).
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

template <typename KVT, int HG, int LPP, bool CLUSTER>
__global__ void __launch_bounds__(ATTN_THREADS) k_attn2(const AttnArgs a) {
	typedef typename KvRaw<KVT>::type raw_t;
	constexpr int HD = LPP * 8, P = LPP / HG, G = 32 / LPP, NW = ATTN_THREADS / 32, NC = LPP;
	static_assert(HG * P == LPP && P >= 1 && P <= 4 && ATTN2_BP % P == 0, "unsupported head grouping");
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ __align__(8) uint64_t bars[ATTN2_MAXB];
	__shared__ int flag;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int nbmax = a.nbmax, nsplit = a.nsplit;
	const int unit = blockIdx.x / nsplit, split = blockIdx.x % nsplit;
	const int kvh = unit / a.qgroups;
	const int hbase = kvh * a.kv_mul + (unit % a.qgroups) * HG;
	constexpr uint32_t BLK = ATTN2_BP * HD * sizeof(KVT); // bytes of a whole block
	KVT* Ks = reinterpret_cast<KVT*>(smem_raw);
	KVT* Vs = Ks + (size_t)nbmax * ATTN2_BP * HD;
	float* qs = reinterpret_cast<float*>(Vs + (size_t)nbmax * ATTN2_BP * HD);
	float* scratch = qs + HG * HD;
	float* myrec = scratch + max(NW * HG * (HD + 2), (2 * nsplit + 1) * HG); // [HG][HD + 2]
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
	// q and the token parameters are requested together (one L2 round trip, not two)
	constexpr int QPT = (HG * HD + ATTN_THREADS - 1) / ATTN_THREADS;
	float qreg[QPT];
#pragma unroll
	for (int i = 0; i < QPT; ++i) qreg[i] = (tid + i * ATTN_THREADS < HG * HD) ? __ldcg(a.q + (size_t)hbase * HD + tid + i * ATTN_THREADS) : 0.f;
	const int kv_len = a.tp->kv_len, kv_pos = a.tp->kv_pos, kv_sink = a.tp->kv_sink;
	const unsigned epoch = (unsigned)a.tp->tp_seq * a.epoch_stride + a.epoch_idx;
	if (tid < nbmax && !issued && (split + tid * nsplit) * ATTN2_BP < kv_len) request(tid), issued = true;
#pragma unroll
	for (int i = 0; i < QPT; ++i)
		if (tid + i * ATTN_THREADS < HG * HD) qs[tid + i * ATTN_THREADS] = qreg[i];
	__syncthreads();
	ATTN_DBG(2);

	// blocks of this CTA that hold cached positions
	const int nblk = (kv_len + ATTN2_BP - 1) / ATTN2_BP;
	const int nb = nblk > split ? (nblk - split + nsplit - 1) / nsplit : 0;
	const int nslots = nb * ATTN2_BP;
	const int grp = lane / LPP, li = lane % LPP;

	float acc[HG][8], m[HG], l[HG];
#pragma unroll
	for (int h = 0; h < HG; ++h) {
		m[h] = -FLT_MAX, l[h] = 0.f;
#pragma unroll
		for (int d = 0; d < 8; ++d) acc[h][d] = 0.f;
	}
	float mh = -FLT_MAX, lh = 0.f; // running max / sum of THIS lane's head (li / P)

	// Steps are taken SC at a time: first ALL scores of the chunk (independent dot products and transposing reductions: no
	// serial softmax state between them), then one max / exp / sum for the chunk, then the value pass.  With 8 warps per SM
	// the per-step online softmax is a latency chain (max / exp / rescale per step); this form rescales the
	// accumulators once per chunk.
	constexpr int SC = 4, STEP = NW * G * P;
	const int gbase = grp * LPP;
	auto slot_of = [&](int s0, int& j, int& o, int& t0) {
		j = s0 / ATTN2_BP, o = s0 % ATTN2_BP;
		t0 = (split + j * nsplit) * ATTN2_BP + o;
	};
	for (int sb = (warp * G + grp) * P; sb - grp * P < nslots; sb += SC * STEP) { // warp-uniform trip count (full-warp shuffles inside)
		float sc[SC];
		bool val[SC], fast[SC];
#pragma unroll
		for (int c = 0; c < SC; ++c) {
			const int s0 = sb + c * STEP;
			const bool inr = s0 < nslots;
			int j = 0, o = 0, t0 = 0;
			if (inr) slot_of(s0, j, o, t0);
			if (inr) mbar_wait(&bars[j], 0);
			if (s0 == 0) ATTN_DBG(3);
			// the common case for a whole warp -- P cached positions, none of them written during this token -- needs no per-position tests
			fast[c] = __all_sync(0xffffffffu, inr && t0 + P <= kv_len && (kv_pos < t0 || kv_pos >= t0 + P) && t0 >= kv_sink);
			float part[NC]; // combo h * P + i: partial dot product of this lane's 8 dims
			{
				float kf[P][8];
				if (fast[c]) {
					const KVT* kp = Ks + ((size_t)j * ATTN2_BP + o) * HD + li * 8;
#pragma unroll
					for (int i = 0; i < P; ++i) KvRaw<KVT>::unpack(*reinterpret_cast<const raw_t*>(kp + i * HD), kf[i]);
				} else {
#pragma unroll
					for (int i = 0; i < P; ++i) {
						const int t = t0 + i;
						raw_t kr = KvRaw<KVT>::zero();
						if (inr && t < kv_len)
							kr = (t == kv_pos || t < kv_sink) ? KvRaw<KVT>::load(kglob + (size_t)t * HD + li * 8) // written during this token: not in the early copy
							                                  : *reinterpret_cast<const raw_t*>(Ks + ((size_t)j * ATTN2_BP + o + i) * HD + li * 8);
						KvRaw<KVT>::unpack(kr, kf[i]);
					}
				}
#pragma unroll
				for (int h = 0; h < HG; ++h) {
					const float4 q0 = *reinterpret_cast<const float4*>(qs + h * HD + li * 8), q1 = *reinterpret_cast<const float4*>(qs + h * HD + li * 8 + 4);
#pragma unroll
					for (int i = 0; i < P; ++i) {
						float d = q0.x * kf[i][0];
						d = fmaf(q0.y, kf[i][1], d), d = fmaf(q0.z, kf[i][2], d), d = fmaf(q0.w, kf[i][3], d);
						d = fmaf(q1.x, kf[i][4], d), d = fmaf(q1.y, kf[i][5], d), d = fmaf(q1.z, kf[i][6], d), d = fmaf(q1.w, kf[i][7], d);
						part[h * P + i] = d;
					}
				}
			}
			// transposing reduction over the LPP lanes of the group: after the step with stride s a lane keeps the half selected by bit s
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
			// lane li owns combo li: head li / P, position li % P
			val[c] = inr && (t0 + li % P) < kv_len;
			sc[c] = val[c] ? part[0] * a.inv_sqrt_hd : -FLT_MAX;
		}
		float gmax = sc[0];
#pragma unroll
		for (int c = 1; c < SC; ++c) gmax = fmaxf(gmax, sc[c]);
#pragma unroll
		for (int o2 = 1; o2 < P; o2 <<= 1) gmax = fmaxf(gmax, __shfl_xor_sync(0xffffffffu, gmax, o2));
		const float mnew = fmaxf(mh, gmax);
		const float corr = __expf(mh - mnew);
		float pr[SC], ps = 0.f;
#pragma unroll
		for (int c = 0; c < SC; ++c) pr[c] = val[c] ? __expf(sc[c] - mnew) : 0.f, ps += pr[c];
#pragma unroll
		for (int o2 = 1; o2 < P; o2 <<= 1) ps += __shfl_xor_sync(0xffffffffu, ps, o2);
		lh = fmaf(lh, corr, ps);
		mh = mnew;
#pragma unroll
		for (int h = 0; h < HG; ++h) {
			const float ch = __shfl_sync(0xffffffffu, corr, gbase + h * P);
#pragma unroll
			for (int e = 0; e < 8; ++e) acc[h][e] *= ch;
		}
#pragma unroll
		for (int c = 0; c < SC; ++c) {
			const int s0 = sb + c * STEP;
			const bool inr = s0 < nslots;
			int j = 0, o = 0, t0 = 0;
			if (inr) slot_of(s0, j, o, t0);
			float vf[P][8];
			if (fast[c]) {
				const KVT* vp = Vs + ((size_t)j * ATTN2_BP + o) * HD + li * 8;
#pragma unroll
				for (int i = 0; i < P; ++i) KvRaw<KVT>::unpack(*reinterpret_cast<const raw_t*>(vp + i * HD), vf[i]);
			} else {
#pragma unroll
				for (int i = 0; i < P; ++i) {
					const int t = t0 + i;
					raw_t vr = KvRaw<KVT>::zero();
					if (inr && t < kv_len)
						vr = (t == kv_pos || t < kv_sink) ? KvRaw<KVT>::load(vglob + (size_t)t * HD + li * 8)
						                                  : *reinterpret_cast<const raw_t*>(Vs + ((size_t)j * ATTN2_BP + o + i) * HD + li * 8);
					KvRaw<KVT>::unpack(vr, vf[i]);
				}
			}
#pragma unroll
			for (int h = 0; h < HG; ++h) {
				float pw[P];
#pragma unroll
				for (int i = 0; i < P; ++i) pw[i] = __shfl_sync(0xffffffffu, pr[c], gbase + h * P + i);
#pragma unroll
				for (int e = 0; e < 8; ++e) {
					float v = acc[h][e];
#pragma unroll
					for (int i = 0; i < P; ++i) v = fmaf(pw[i], vf[i][e], v);
					acc[h][e] = v;
				}
			}
		}
	}
	ATTN_DBG(4);
#pragma unroll
	for (int h = 0; h < HG; ++h) { // running max / sum live in the lanes that own the head: hand them to every lane of the group
		m[h] = __shfl_sync(0xffffffffu, mh, grp * LPP + h * P);
		l[h] = __shfl_sync(0xffffffffu, lh, grp * LPP + h * P);
	}
	if constexpr (CLUSTER) {
		constexpr int REC = HD + 2;
		__shared__ float mls[ATTN2_MAX_CLUSTER][HG][2]; // (m, l) of every slice, then (coefficient, -) in place
		__shared__ float invl[HG];
		attn_cta_merge<HG>(a, HG, 0, HG, warp, NW, m, l, acc, scratch, myrec);
		cluster_sync_all(); // every CTA's record is complete and visible cluster-wide
		for (int i = tid; i < nsplit * HG; i += ATTN_THREADS) {
			const int s = i / HG, h = i % HG;
			mls[s][h][0] = ld_dsmem(myrec + h * REC + HD, s), mls[s][h][1] = ld_dsmem(myrec + h * REC + HD + 1, s);
		}
		__syncthreads();
		if (tid < HG) {
			float M = -FLT_MAX;
			for (int s = 0; s < nsplit; ++s) M = fmaxf(M, mls[s][tid][0]);
			float L = 0.f;
			for (int s = 0; s < nsplit; ++s) {
				const float c = expf(mls[s][tid][0] - M);
				L = fmaf(mls[s][tid][1], c, L);
				mls[s][tid][0] = c;
			}
			invl[tid] = 1.0f / L;
		}
		__syncthreads();
		// CTA `split` normalises outputs [split * per, (split + 1) * per): 8 adjacent lanes share an output, each sums every 8th slice
		const int nout = HG * HD, per = (nout + nsplit - 1) / nsplit;
		const int o_end = min(nout, (split + 1) * per);
		for (int o0 = split * per; o0 < o_end; o0 += ATTN_THREADS / 8) {
			const int o = o0 + tid / 8, sg = tid & 7;
			float v = 0.f;
			if (o < o_end) {
				const int h = o / HD, e = o % HD;
				for (int s = sg; s < nsplit; s += 8) v = fmaf(ld_dsmem(myrec + h * REC + e, s), mls[s][h][0], v);
			}
			v += __shfl_xor_sync(0xffffffffu, v, 1), v += __shfl_xor_sync(0xffffffffu, v, 2), v += __shfl_xor_sync(0xffffffffu, v, 4);
			if (o < o_end && sg == 0) __stcg(a.out + (size_t)hbase * HD + o, v * invl[o / HD]);
		}
		cluster_sync_all(); // no CTA may exit (and free its shared memory) while a peer still reads its record
	} else {
		constexpr int REC = HD + 2;
		__shared__ float mls[ATTN2_MAXB + 4][HG][2]; // (m, l) of every slice, then the coefficient in place  (nsplit <= 36)
		__shared__ float invl[HG];
		(void)flag;
		attn_cta_merge<HG>(a, HG, 0, HG, warp, NW, m, l, acc, scratch, myrec);
		__syncthreads();
		ATTN_DBG(5);
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
	}
	// no bulk copy may still be in flight into this CTA's shared memory when it exits (a block requested on a stale hint)
	if (tid < nbmax && issued) mbar_wait(&bars[tid], 0);
	ATTN_DBG(7);
	if (a.dbg && tid == 0) atomicMax(a.dbg + 9, globaltimer_ns());
	stamp_end(a.stamp);
}
