// ring.cuh -- the two largest matvec stages (FFN up, FFN down; and wo) fed by warp-private bulk-TMA rings.
//
// Why: the register-fed stage kernels keep their bytes in flight in registers --
// a warp requests one batch (8 x 16 B per lane), waits a DRAM round trip, consumes it, and only then requests the next --
// so the bytes in flight per SM are duty-cycled, bounded by the register file, and nothing can be requested before the
// dependency wait without costing a CTA of occupancy.  Here every warp owns a small ring of shared-memory slots that it
// fills itself with cp.async.bulk (one elected lane, completion on the slot's mbarrier, L2::evict_first: every weight byte
// is read once per token): requests run RING_NS chunks ahead of the arithmetic, continuously, across task boundaries, and
// the first RING_NS chunks are requested BEFORE griddepcontrol.wait (weights are immutable), i.e. while the previous kernel
// drains and the activation vector is staged.  There is no producer warp and no CTA-wide hand-off: a warp waits only on
// its own mbarriers.  Slots per warp and warps per CTA are the best of the H100 sweep in profiles/README.md.
//
// Work split: one CTA owns a contiguous range of "tasks"; its warps take tasks from a shared-memory counter, so all warps
// of an SM finish within one chunk of each other whatever the task count (the static row-pair stride of k_ffn_up costs a
// nearly empty fifth round: 14336 pairs over 3552 warps).  A task is a row pair (R = 2 rows share every activation load)
// restricted to a K-slice of S chunks; kernels with few long rows (w2: 2048 pairs of 14336 weights) use S = 1 and
// fold the slices of a pair in slice order (deterministic) through shared memory -- the last slice to finish does it.
//
// Arithmetic is dot_vec<> of common.cuh on the same vectors in the same per-lane order as warp_dot_rows, so results are
// bit-identical to the register-fed kernels for whole rows.  Rows must be whole 1 KB chunks.  The rings serve dense
// models, with or without tensor parallelism: k_matres_ring carries the in-kernel exchange of stages.cuh TpExchange, and
// only the NCCL all-reduce path keeps k_matres for wo / w2.  MoE layers (expert rows known only after the router) and
// other row lengths keep k_ffn_up / k_matres.
#pragma once

#include "stages.cuh"

#define RING_NS 2         // slots per warp
#define RING_UP_WARPS 8   // FFN up: two CTAs of 8 warps per SM
#define RING_RES_WARPS 16 // wo / w2: one CTA of 16 warps per SM (the activation vector is long: w2)
#define RING_MAX_PAIRS 48 // row pairs per CTA when K-slices are folded through shared memory
#define RING_MAX_SLICES 32

struct RingCtl {
	uint64_t bar[RING_RES_WARPS][RING_NS];
	int slot_task[RING_RES_WARPS][RING_NS];
	int slot_piece[RING_RES_WARPS][RING_NS];
	int ctr; // next task of this CTA
};

// shared memory of a ring kernel: [32 floats block-reduce][activation vector][ring: warps x RING_NS x 2 rows x CH bytes]
template <int DBITS>
__host__ __device__ inline size_t ring_smem_bytes(int n, int u, int warps) {
	size_t xs = ((size_t)(32 + xs_all_floats<DBITS>(n)) * sizeof(float) + 127) & ~(size_t)127;
	return xs + (size_t)warps * RING_NS * 2 * u * 512;
}

// The streaming loop of one warp.  rows(task, rp0, rp1, chunk0): byte pointers of the task's two rows and its first chunk
// index inside the row; done(task, v0, v1): the two finished dot products (called by every lane, values valid in all).
// issue_prologue() must be called (warp-uniformly) before consume_all(); in between the caller waits for the previous grid
// and stages the activation vector.
template <int DBITS, int U, typename RowsFn, typename DoneFn>
struct RingWarp {
	static constexpr int CH = U * 512; // bytes per row and chunk
	RingCtl* ctl;
	unsigned char* ring; // this warp's RING_NS slots
	int warp, lane;
	int t_hi, S; // end of the CTA's task range; chunks per task
	uint64_t policy;
	int issued = 0, consumed = 0, cur_task = 0, cur_piece = 0;
	bool more = true;
	RowsFn rows;
	DoneFn done;

	__device__ __forceinline__ RingWarp(RingCtl* c, unsigned char* ring_base, int t_hi_, int S_, RowsFn r, DoneFn d)
	    : ctl(c), warp(threadIdx.x >> 5), lane(threadIdx.x & 31), t_hi(t_hi_), S(S_), rows(r), done(d) {
		ring = ring_base + (size_t)warp * RING_NS * 2 * CH;
		policy = l2_policy_evict_first();
		cur_piece = S; // forces a task grab
	}

	__device__ __forceinline__ void issue_one() { // warp-uniform control flow
		if (cur_piece == S) {
			int t = 0;
			if (lane == 0) t = atomicAdd(&ctl->ctr, 1);
			t = __shfl_sync(0xffffffffu, t, 0);
			if (t >= t_hi) {
				more = false;
				return;
			}
			cur_task = t, cur_piece = 0;
		}
		const int slot = issued % RING_NS;
		if (lane == 0) {
			const unsigned char *rp0, *rp1;
			int chunk0;
			rows(cur_task, rp0, rp1, chunk0);
			const size_t off = (size_t)(chunk0 + cur_piece) * CH;
			ctl->slot_task[warp][slot] = cur_task, ctl->slot_piece[warp][slot] = cur_piece;
			uint64_t* bar = &ctl->bar[warp][slot];
			mbar_expect_tx(bar, 2 * CH);
			tma_load_1d_hint(ring + (size_t)slot * 2 * CH, rp0 + off, CH, bar, policy);
			tma_load_1d_hint(ring + (size_t)slot * 2 * CH + CH, rp1 + off, CH, bar, policy);
		}
		++issued, ++cur_piece;
	}

	__device__ __forceinline__ void issue_prologue() {
#pragma unroll
		for (int i = 0; i < RING_NS; ++i)
			if (more) issue_one();
		__syncwarp();
	}

	__device__ __forceinline__ void consume_all(const float4* __restrict__ xs4, int n) { // n: length of the staged vector
		const float4* xg4 = xs4 + (xs_floats<DBITS>(n) >> 2); // gf4: the group sums behind the vector (common.cuh xs_aux_floats)
		constexpr int Q = WFmt<DBITS>::VW / 4;
		float acc0 = 0.f, acc1 = 0.f;
		while (consumed < issued) {
			const int slot = consumed % RING_NS;
			mbar_wait(&ctl->bar[warp][slot], (consumed / RING_NS) & 1);
			const int task = ctl->slot_task[warp][slot], piece = ctl->slot_piece[warp][slot];
			int chunk0;
			{
				const unsigned char *rp0, *rp1;
				rows(task, rp0, rp1, chunk0);
			}
			const uint4* s0 = reinterpret_cast<const uint4*>(ring + (size_t)slot * 2 * CH);
			const uint4* s1 = s0 + CH / 16;
			const float4* xp = xs4 + (size_t)((chunk0 + piece) * U) * Q * 32; // chunk = U groups of 32 vectors
			uint4 w0[U], w1[U];
#pragma unroll
			for (int u = 0; u < U; ++u) w0[u] = s0[32 * u + lane], w1[u] = s1[32 * u + lane];
#pragma unroll
			for (int u = 0; u < U; ++u) {
				float4 xv[Q];
#pragma unroll
				for (int q = 0; q < Q; ++q) xv[q] = xp[(u * Q + q) * 32 + (lane ^ xs_swz<DBITS>(q))];
				float4 g3 = make_float4(0.f, 0.f, 0.f, 0.f);
				if (DBITS == 4) g3 = xg4[((chunk0 + piece) * U + u) * 32 + lane];
				acc0 = dot_vec<DBITS>(w0[u], xv, g3, acc0);
				acc1 = dot_vec<DBITS>(w1[u], xv, g3, acc1);
			}
			++consumed;
			__syncwarp(); // every lane has read the slot (its values are in registers): the slot may be refilled
			if (more) issue_one();
			if (piece == S - 1) {
				const float v0 = warp_sum(acc0), v1 = warp_sum(acc1);
				done(task, v0, v1);
				acc0 = acc1 = 0.f;
			}
		}
	}
};

__device__ __forceinline__ void ring_init(RingCtl* ctl, int t_lo) {
	if (threadIdx.x == 0) ctl->ctr = t_lo;
	if (threadIdx.x < (blockDim.x >> 5) * RING_NS) mbar_init(&ctl->bar[threadIdx.x / RING_NS][threadIdx.x % RING_NS], 1);
	if (threadIdx.x == 0) mbar_init_fence();
	__syncthreads();
}

// ------------------------------------------------------------------------------------------------
// FFN up: hb[i] = act(w1[i] . xn) * (w3[i] . xn)   (reference infer.c:437-450); task i = rows (w1[i], w3[i]), whole rows.

template <int DBITS, int U>
__global__ void __launch_bounds__(RING_UP_WARPS * 32, 2) k_ffn_up_ring(const FfnUpArgs a) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ RingCtl ctl;
	float* red = reinterpret_cast<float*>(smem_raw);
	float* xs = red + 32;
	unsigned char* ring = smem_raw + (((size_t)(32 + xs_all_floats<DBITS>(a.dim)) * sizeof(float) + 127) & ~(size_t)127);
	const size_t rowbytes = (size_t)a.dim * DBITS / 8;
	const int cpt = (int)(rowbytes / (U * 512));
	const int t_lo = (int)(((long long)blockIdx.x * a.hidden) / gridDim.x), t_hi = (int)(((long long)(blockIdx.x + 1) * a.hidden) / gridDim.x);
	pdl_launch_next();
	ring_init(&ctl, t_lo);
	float post = 1.f;
	const unsigned char* w1 = reinterpret_cast<const unsigned char*>(a.w1);
	const unsigned char* w3 = reinterpret_cast<const unsigned char*>(a.w3);
	auto rows = [&](int t, const unsigned char*& rp0, const unsigned char*& rp1, int& chunk0) {
		rp0 = w1 + (size_t)t * rowbytes, rp1 = w3 + (size_t)t * rowbytes, chunk0 = 0;
	};
	auto done = [&](int t, float v0, float v1) {
		if ((threadIdx.x & 31) == 0) {
			const float u1 = v0 * post, u3 = v1 * post;
			a.hb[t] = (a.gelu ? act_gelu(u1) : act_silu(u1)) * u3;
		}
	};
	RingWarp<DBITS, U, decltype(rows), decltype(done)> rw(&ctl, ring, t_hi, cpt, rows, done);
	rw.issue_prologue(); // the first RING_NS chunks of every warp are in flight before the previous kernel has finished
	pdl_wait_prev();
	stamp_begin(a.stamp);
	post = stage_vector<DBITS>(xs, red, a.x, a.dim, a.normw, a.eps, a.ln != 0, nullptr);
	rw.consume_all(reinterpret_cast<const float4*>(xs), a.dim);
	stamp_end(a.stamp);
}

// ------------------------------------------------------------------------------------------------
// y[row] += W[row] . xin  (wo, w2; dense).  Task = (row pair p, K-slice s of S chunks), t = p * nsl + s; with nsl > 1 the
// slices of a pair land in part[][] and the last one to arrive adds them up in slice order.

template <int DBITS, int U>
__global__ void __launch_bounds__(RING_RES_WARPS * 32, 1) k_matres_ring(const MatResArgs a) {
	extern __shared__ __align__(128) unsigned char smem_raw[];
	__shared__ RingCtl ctl;
	__shared__ float2 part[RING_MAX_PAIRS][RING_MAX_SLICES];
	__shared__ int cnt[RING_MAX_PAIRS];
	__shared__ __align__(8) float ypart[2 * RING_MAX_PAIRS]; // tensor parallelism: this rank's partial of the CTA's rows, summed over the ranks at the end
	float* red = reinterpret_cast<float*>(smem_raw);
	float* xs = red + 32;
	unsigned char* ring = smem_raw + (((size_t)(32 + xs_all_floats<DBITS>(a.n)) * sizeof(float) + 127) & ~(size_t)127);
	const size_t rowbytes = (size_t)a.n * DBITS / 8;
	const int S = a.S, cpt = (int)(rowbytes / (U * 512)), nsl = cpt / S;
	const int npairs = a.d / 2;
	const int p_lo = (int)(((long long)blockIdx.x * npairs) / gridDim.x), p_hi = (int)(((long long)(blockIdx.x + 1) * npairs) / gridDim.x);
	pdl_launch_next();
	if (threadIdx.x < RING_MAX_PAIRS) cnt[threadIdx.x] = 0;
	ring_init(&ctl, p_lo * nsl);
	const unsigned char* w = reinterpret_cast<const unsigned char*>(a.w);
	auto rows = [&](int t, const unsigned char*& rp0, const unsigned char*& rp1, int& chunk0) {
		const int p = t / nsl, s = t - p * nsl;
		rp0 = w + (size_t)(2 * p) * rowbytes, rp1 = rp0 + rowbytes, chunk0 = s * S;
	};
	auto done = [&](int t, float v0, float v1) {
		if ((threadIdx.x & 31) != 0) return;
		const int p = t / nsl, s = t - p * nsl;
		if (nsl > 1) {
			const int pl = p - p_lo;
			part[pl][s] = make_float2(v0, v1);
			__threadfence_block();
			if (atomicAdd(&cnt[pl], 1) != nsl - 1) return;
			__threadfence_block();
			v0 = 0.f, v1 = 0.f;
			for (int k = 0; k < nsl; ++k) v0 += part[pl][k].x, v1 += part[pl][k].y; // slice order: deterministic
		}
		if (a.tpx.world > 1) { // the matvec -> all-reduce fusion of stages.cuh TpExchange, on this kernel's contiguous row ranges
			ypart[2 * (p - p_lo)] = v0, ypart[2 * (p - p_lo) + 1] = v1;
			return;
		}
		float2* dst = reinterpret_cast<float2*>(a.y + 2 * p);
		float2 cur = a.accumulate ? *dst : make_float2(0.f, 0.f);
		cur.x += v0, cur.y += v1;
		*dst = cur;
	};
	RingWarp<DBITS, U, decltype(rows), decltype(done)> rw(&ctl, ring, p_hi * nsl, S, rows, done);
	rw.issue_prologue();
	pdl_wait_prev();
	stamp_begin(a.stamp);
	stage_vector<DBITS, 16>(xs, red, a.xin, a.n, nullptr, 0.f, false, nullptr);
	rw.consume_all(reinterpret_cast<const float4*>(xs), a.n);
	if (a.tpx.world > 1) tp_exchange_rows(a.tpx, ypart, 2 * p_lo, 2 * (p_hi - p_lo), a.y, a.d);
	stamp_end(a.stamp);
}

