// sample_n.cuh -- the attention of calm_b200_decode_sample_n: nseq sequences that continue one shared prompt, one token
// each per step, through the short-block pass (verify.cuh's k_vf_gemm for the projections and the classifier).
//
// Cache layout.  The prompt is in slots [0, pos0).  At step j every row b (one per sequence) is at RoPE position pos0 + j
// and writes slot pos0 + j * nseq + b, so a step is an ordinary short block at slot base pos0 + j * nseq and the QKV
// epilogue appends its keys unchanged.  Row b's keys at step j, in order, are the prompt's slots 0 .. pos0 - 1 and then
// its own slots pos0 + i * nseq + b for i = 0 .. j: its virtual key index v = 0 .. pos0 + j.
//
//   k_sn_attn   split-KV, multi-query attention over fixed chunks of SN_CHUNK virtual keys.  A chunk wholly inside the
//               prompt holds the same keys for every row, so one CTA per (kv head, chunk) stages its K and V tiles in
//               shared memory once and computes a partial (m, l, acc[HD]) for every row and query head of the kv head.
//               A chunk that reaches past the prompt is computed per row, over that row's own virtual keys.  fp32 math
//               on the fp16 / e5m2 cache entries, as k_pf_attn.  A warp takes KM query heads of one row at a time; its
//               lanes own the chunk's keys lane + 32 i for the scores and head dims for the values.
//   k_sn_fold   one warp per (row, query head): the row's chunk partials folded in ascending chunk order against their
//               common maximum, written as the f16 hi + lo pair that wo's k_vf_gemm reads.
//
// A row's output depends on its query, its keys and the chunking only, never on how many rows run beside it: which chunks
// are shared depends on pos0 and j alone, a query's arithmetic does not depend on the warp that runs it, and nothing is
// added with atomics.
//
// BATCH (calm_b200_decode_sample_batch): every row continues its own prompt.  The prompts were packed by the prompt pass
// from slot 0, row b's L_b prompt entries at slots s_b .. s_b + L_b - 1 (rows[b] = (s_b, L_b)), and the region ends at
// slot pos0 = G.  Step j writes row b to slot G + j * nseq + b, so row b's keys at step j are v = 0 .. L_b + j: v < L_b is
// slot s_b + v, v >= L_b is slot G + (v - L_b) * nseq + b.  No chunk is shared: CTA x is chunk x % nch of row x / nch
// (nch = gridDim.x / nseq, the longest row's chunk count), and a CTA past its row's chunks returns.  A query's staging,
// scores, chunk softmax, value pass and fold are the plain kernels' operations in the same order, so row b gives what
// calm_b200_decode_sample_n gives one sequence over the same keys at pos0 = L_b.
//
// QUEUE (with BATCH; calm_b200_decode_sample_queue): rows run requests that were admitted at different steps, so each row
// has its own step count and its own generated slots.  qrows[r] = (s, L, t, j): the row's prompt entries are at slots
// s .. s + L - 1, its generated entries at slots t, t + 1, .., and it is at its own step j, so its keys are v = 0 .. L + j:
// v < L is slot s + v, v >= L is slot t + (v - L).  Grid, chunking and every floating-point operation are BATCH's, so a row
// gives what decode_sample_batch gives its sequence over the same keys at step j.
//
// GROUPS (with QUEUE; calm_b200_decode_sample_queue_context): a row's prompt is a context of nc entries at slots c ..
// followed by its own L - nc entries at slots s .., so v < nc is slot c + v, nc <= v < L is slot s + (v - nc) and v >= L is
// slot t + (v - L) (SqGroups.ctx[r] = (c, nc); nc = 0 is QUEUE's mapping).  The rows in flight that name one context form
// a group.  A chunk wholly inside the context, (k + 1) * SN_CHUNK <= nc, holds the same keys for every row of the group,
// so one CTA per (group, chunk, kv head) stages it once and writes the partials of every row of the group, as the shared
// prompt chunks above; every other chunk is computed per row, over the row's own virtual keys.  Grid (shared chunks +
// nseq x nsuf, kv heads): CTA x < the shared chunks' count is shared chunk x - chunk0[g] of the group g that holds it, the
// others are per-row chunk nc / SN_CHUNK + x' % nsuf of row x' / nsuf.  Which chunks are shared depends on nc alone and a
// query's arithmetic does not depend on the CTA or warp that runs it, so a row gives what QUEUE gives it over the same keys.
//
// BEAM (calm_b200_decode_beam): the plain layout, but a row reads its generated keys through its ancestry.  Step j writes
// row b to slot pos0 + j * nbeam + b (step 0 runs one row), and anc[b * anc_stride + i] is the row of step i whose key
// row b reads as its virtual key pos0 + i, so v >= pos0 is slot pos0 + (v - pos0) * nbeam + anc[b][v - pos0].  With
// anc[b][i] = b and nbeam = nseq that is the plain mapping, and grid, chunking and every floating-point operation are
// the plain kernels', so a beam's row gives what decode_sample_n gives a sequence over the same keys.
#pragma once

#include "prefill.cuh"

#define SN_CHUNK 128 // virtual keys per chunk: four per lane in the score pass
#define SN_WARPS 8
#define SQ_ROWS 16   // rows of a queue step: one token tile of k_vf_gemm

// The context groups of one queue step (GROUPS), rows in the step's admission order.  Passed by value to k_sq_groups,
// which keeps it where k_sn_attn reads it.
struct SqGroups {
	int2 ctx[SQ_ROWS];        // row r's context: its first slot and its length nc (0: none)
	int chunk0[SQ_ROWS + 1];  // group g's shared chunks are the CTAs chunk0[g] .. chunk0[g + 1] - 1
	int first[SQ_ROWS + 1];   // group g's rows are rows[first[g] .. first[g + 1])
	int rows[SQ_ROWS];
	int ng;                   // groups; chunk0[ng] is the shared chunks' count
};

struct SnAttnArgs {
	const float* Q;  // [nseq][q_dim] the step's rotated queries
	const void* kc;  // this layer
	const void* vc;
	float* part;     // [nseq][n_heads][nchmax][HD + 2] per chunk: m, l, acc[HD]
	__half* Ohi;     // [nseq][q_dim]
	__half* Olo;
	int pos0, step, nseq, seq_len, q_dim, kv_mul, n_heads, nchmax;
	float inv_sqrt_hd;
	const int2* rows; // [nseq] (BATCH) row b's prompt: its first slot s_b and its length L_b; read by no other variant
	const int4* qrows; // [nseq] (QUEUE) row b's (s, L, t, j); read by no other variant
	const SqGroups* groups; // (GROUPS) the step's contexts and groups; read by no other variant
	const int* anc;   // (BEAM) [nseq][anc_stride] each row's ancestor row at every step; read by no other variant
	int nbeam, anc_stride; // (BEAM) the slot stride of a step and anc's row length
};

// dynamic shared memory of k_sn_attn: the K tile (padded rows), the V tile, each warp's KM queries
template <typename KVT, int HD, int KM>
constexpr size_t sn_smem_bytes() {
	return (size_t)SN_CHUNK * (HD * sizeof(KVT) + 16) + (size_t)SN_CHUNK * HD * sizeof(KVT) + (size_t)SN_WARPS * KM * HD * sizeof(float);
}

// grid (prompt chunks + nseq x suffix chunks, kv heads): CTA x < pos0 / SN_CHUNK is prompt chunk x for every row, the
// others are suffix chunk x' % nsuf of row x' / nsuf (x' = x - prompt chunks).  BATCH (and QUEUE): grid (nseq x nch, kv
// heads).  GROUPS: the grid above its header comment says.
template <typename KVT, int HD, int KM, bool BATCH = false, bool QUEUE = false, bool GROUPS = false, bool BEAM = false>
__global__ void __launch_bounds__(SN_WARPS * 32) k_sn_attn(const SnAttnArgs a) {
	static_assert(BATCH || !QUEUE, "a queue step is a batch step with per-row step counts");
	static_assert(QUEUE || !GROUPS, "context groups are rows of a queue step");
	static_assert(!(BEAM && BATCH), "beams share one prompt");
	pdl_enter();
	constexpr int DPL = HD / 32, KPL = SN_CHUNK / 32;
	constexpr int VSTR = HD * sizeof(KVT), KSTR = VSTR + 16; // padded key row, as k_pf_attn's
	extern __shared__ __align__(16) unsigned char sn_smem[];
	unsigned char* ks = sn_smem;
	unsigned char* vs = ks + SN_CHUNK * KSTR;
	float* qs = reinterpret_cast<float*>(vs + SN_CHUNK * VSTR) + (threadIdx.x >> 5) * KM * HD;
	const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, kvh = blockIdx.y;
	int nkeys, c, b0, nrows; // (GROUPS) b0 = -1 - f for a shared chunk, whose rows are groups->rows[f ..]
	if constexpr (GROUPS) {
		const SqGroups* gt = a.groups;
		const int nsh = __ldg(gt->chunk0 + __ldg(&gt->ng));
		if ((int)blockIdx.x < nsh) { // chunk c of group gi's context, for every row of the group
			int gi = 0;
			while ((int)blockIdx.x >= __ldg(gt->chunk0 + gi + 1)) ++gi;
			const int f = __ldg(gt->first + gi);
			c = blockIdx.x - __ldg(gt->chunk0 + gi), nrows = __ldg(gt->first + gi + 1) - f;
			b0 = -1 - f, nkeys = (c + 1) * SN_CHUNK;
		} else {
			const int nsuf = (gridDim.x - nsh) / a.nseq, x = blockIdx.x - nsh;
			b0 = x / nsuf, nrows = 1;
			const int4 qr = __ldg(a.qrows + b0);
			nkeys = qr.y + qr.w + 1, c = __ldg(&gt->ctx[b0].y) / SN_CHUNK + x % nsuf;
			if (c * SN_CHUNK >= nkeys) return;
		}
	} else if constexpr (BATCH) {
		const int nch = gridDim.x / a.nseq;
		b0 = blockIdx.x / nch, c = blockIdx.x % nch, nrows = 1;
		if constexpr (QUEUE) {
			const int4 qr = __ldg(a.qrows + b0);
			nkeys = qr.y + qr.w + 1;
		} else nkeys = __ldg(&a.rows[b0].y) + a.step + 1;
		if (c * SN_CHUNK >= nkeys) return;
	} else {
		nkeys = a.pos0 + a.step + 1, c = blockIdx.x, b0 = 0, nrows = a.nseq;
		const int npre = a.pos0 / SN_CHUNK, nsuf = (nkeys + SN_CHUNK - 1) / SN_CHUNK - npre;
		if (c >= npre) {
			const int x = c - npre;
			b0 = x / nsuf, c = npre + x % nsuf, nrows = 1;
		}
	}
	const int v0 = c * SN_CHUNK, nk = min(SN_CHUNK, nkeys - v0);
	const KVT* kbase = reinterpret_cast<const KVT*>(a.kc) + (size_t)kvh * a.seq_len * HD;
	const KVT* vbase = reinterpret_cast<const KVT*>(a.vc) + (size_t)kvh * a.seq_len * HD;
	for (int i = threadIdx.x; i < SN_CHUNK * (VSTR / 16); i += blockDim.x) {
		const int row = i / (VSTR / 16), cc = i % (VSTR / 16), v = v0 + row;
		const bool in = row < nk;
		int slot;
		if constexpr (GROUPS) { // (a shared chunk maps its keys through its group's first row: they are in its context)
			const int br = b0 >= 0 ? b0 : __ldg(a.groups->rows - 1 - b0);
			const int* qr = reinterpret_cast<const int*>(a.qrows + br);
			const int2 cx = __ldg(a.groups->ctx + br);
			const int L = __ldg(qr + 1);
			slot = v < cx.y ? cx.x + v : v < L ? __ldg(qr) + (v - cx.y) : __ldg(qr + 2) + (v - L);
		} else if constexpr (QUEUE) { // (scalar loads: the whole int4 held through the score pass adds spills)
			const int* qr = reinterpret_cast<const int*>(a.qrows + b0);
			const int L = __ldg(qr + 1);
			slot = v < L ? __ldg(qr) + v : __ldg(qr + 2) + (v - L);
		} else if constexpr (BATCH) { // (read per key: held in registers through the score pass, they add spills)
			const int2 pr = __ldg(a.rows + b0);
			slot = v < pr.y ? pr.x + v : a.pos0 + (v - pr.y) * a.nseq + b0;
		} else if constexpr (BEAM) { // (only a key the chunk holds reads its ancestor: anc ends at the row's last key)
			slot = v < a.pos0 || !in ? v : a.pos0 + (v - a.pos0) * a.nbeam + __ldg(a.anc + (size_t)b0 * a.anc_stride + (v - a.pos0));
		} else slot = v < a.pos0 ? v : a.pos0 + (v - a.pos0) * a.nseq + b0;
		const uint4 z = make_uint4(0, 0, 0, 0);
		*reinterpret_cast<uint4*>(ks + row * KSTR + cc * 16) = in ? __ldcg(reinterpret_cast<const uint4*>(kbase + (size_t)slot * HD) + cc) : z;
		*reinterpret_cast<uint4*>(vs + row * VSTR + cc * 16) = in ? __ldcg(reinterpret_cast<const uint4*>(vbase + (size_t)slot * HD) + cc) : z;
	}
	__syncthreads();

	const int groups = nrows * a.kv_mul / KM;
	for (int gq = warp; gq < groups; gq += SN_WARPS) {
		const int b = GROUPS && b0 < 0 ? __ldg(a.groups->rows + (-1 - b0) + gq * KM / a.kv_mul) : b0 + gq * KM / a.kv_mul, h0 = kvh * a.kv_mul + gq * KM % a.kv_mul;
		__syncwarp(); // the previous group's queries are no longer being read
		for (int i = lane; i < KM * HD; i += 32) qs[i] = a.Q[(size_t)b * a.q_dim + (size_t)h0 * HD + i];
		__syncwarp();
		// scores of keys lane + 32 i against the KM heads
		float sc[KM][KPL];
#pragma unroll
		for (int h = 0; h < KM; ++h)
#pragma unroll
			for (int i = 0; i < KPL; ++i) sc[h][i] = 0.f;
#pragma unroll 2
		for (int c8 = 0; c8 < HD / 8; ++c8) {
			float4 q[KM][2];
#pragma unroll
			for (int h = 0; h < KM; ++h) q[h][0] = *reinterpret_cast<const float4*>(qs + h * HD + c8 * 8), q[h][1] = *reinterpret_cast<const float4*>(qs + h * HD + c8 * 8 + 4);
#pragma unroll
			for (int i = 0; i < KPL; ++i) {
				float kf[8];
				kv_load8(reinterpret_cast<const KVT*>(ks + (lane + 32 * i) * KSTR) + c8 * 8, kf);
#pragma unroll
				for (int h = 0; h < KM; ++h) {
					float s = sc[h][i];
					s = fmaf(q[h][0].x, kf[0], s), s = fmaf(q[h][0].y, kf[1], s), s = fmaf(q[h][0].z, kf[2], s), s = fmaf(q[h][0].w, kf[3], s);
					s = fmaf(q[h][1].x, kf[4], s), s = fmaf(q[h][1].y, kf[5], s), s = fmaf(q[h][1].z, kf[6], s), s = fmaf(q[h][1].w, kf[7], s);
					sc[h][i] = s;
				}
			}
		}
		// the chunk's softmax numerators against its own maximum, and their sum
		float m[KM], l[KM];
#pragma unroll
		for (int h = 0; h < KM; ++h) {
			float mx = -FLT_MAX;
#pragma unroll
			for (int i = 0; i < KPL; ++i) {
				sc[h][i] = lane + 32 * i < nk ? sc[h][i] * a.inv_sqrt_hd : -FLT_MAX;
				mx = fmaxf(mx, sc[h][i]);
			}
			mx = warp_max(mx);
			float s = 0.f;
#pragma unroll
			for (int i = 0; i < KPL; ++i) {
				sc[h][i] = lane + 32 * i < nk ? expf(sc[h][i] - mx) : 0.f;
				s += sc[h][i];
			}
			m[h] = mx, l[h] = warp_sum(s);
		}
		// values: lane owns head dims [lane * DPL, lane * DPL + DPL), keys in ascending order
		float acc[KM][DPL];
#pragma unroll
		for (int h = 0; h < KM; ++h)
#pragma unroll
			for (int d = 0; d < DPL; ++d) acc[h][d] = 0.f;
#pragma unroll
		for (int i = 0; i < KPL; ++i) {
			const int jn = min(32, nk - 32 * i);
			for (int j = 0; j < jn; ++j) {
				float vf[DPL];
				pf_load_dims<DPL>(reinterpret_cast<const KVT*>(vs + (32 * i + j) * VSTR) + lane * DPL, vf);
#pragma unroll
				for (int h = 0; h < KM; ++h) {
					const float pj = __shfl_sync(0xffffffffu, sc[h][i], j);
#pragma unroll
					for (int d = 0; d < DPL; ++d) acc[h][d] = fmaf(pj, vf[d], acc[h][d]);
				}
			}
		}
#pragma unroll
		for (int h = 0; h < KM; ++h) {
			float* o = a.part + (((size_t)b * a.n_heads + h0 + h) * a.nchmax + c) * (HD + 2);
			if (lane == 0) o[0] = m[h], o[1] = l[h];
#pragma unroll
			for (int d = 0; d < DPL; ++d) o[2 + lane * DPL + d] = acc[h][d];
		}
	}
}

// grid (cdiv(n_heads, SN_WARPS), nseq): warp = query head, lane = head dims [lane * DPL, lane * DPL + DPL)
template <int HD, bool BATCH = false, bool QUEUE = false>
__global__ void __launch_bounds__(SN_WARPS * 32) k_sn_fold(const SnAttnArgs a) {
	pdl_enter();
	constexpr int DPL = HD / 32;
	const int lane = threadIdx.x & 31, h = blockIdx.x * SN_WARPS + (threadIdx.x >> 5), b = blockIdx.y;
	if (h >= a.n_heads) return;
	int last; // the row's last virtual key
	if constexpr (QUEUE) last = a.qrows[b].y + a.qrows[b].w;
	else last = (BATCH ? a.rows[b].y : a.pos0) + a.step;
	const int nch = (last + SN_CHUNK) / SN_CHUNK;
	const float* p = a.part + ((size_t)b * a.n_heads + h) * a.nchmax * (HD + 2);
	float mx = -FLT_MAX;
	for (int c = lane; c < nch; c += 32) mx = fmaxf(mx, __ldcg(p + (size_t)c * (HD + 2)));
	mx = warp_max(mx);
	float l = 0.f, acc[DPL];
#pragma unroll
	for (int d = 0; d < DPL; ++d) acc[d] = 0.f;
	for (int c = 0; c < nch; ++c) {
		const float* pc = p + (size_t)c * (HD + 2);
		const float w = expf(__ldcg(pc) - mx);
		l = fmaf(__ldcg(pc + 1), w, l);
#pragma unroll
		for (int d = 0; d < DPL; ++d) acc[d] = fmaf(__ldcg(pc + 2 + lane * DPL + d), w, acc[d]);
	}
	const float inv = 1.0f / l;
#pragma unroll
	for (int d = 0; d < DPL; ++d) {
		__half hh, hl;
		split_hl(acc[d] * inv, hh, hl);
		const size_t o = (size_t)b * a.q_dim + (size_t)h * HD + lane * DPL + d;
		a.Ohi[o] = hh, a.Olo[o] = hl;
	}
}

// ---------------------------------------------------------------- calm_b200_decode_sample_queue's rows

// The rows of one queue step, row r in admission order.  Passed by value to k_sq_begin, which keeps it where the step's
// kernels read it.
struct SqRows {
	int4 q[SQ_ROWS];          // (s, L, t, j): k_sn_attn<.., QUEUE>'s key mapping
	int pos[SQ_ROWS];         // RoPE position L + j (k_pf_rope_rows)
	int slot[SQ_ROWS];        // cache slot t + j of the row's keys and values (k_vf_gemm<PF_QKV_SLOTS>)
	int src[SQ_ROWS];         // the previous step's row this row continues, or -1 for a row admitted before this step
	int tok0[SQ_ROWS];        // (src -1) the last token of the row's prompt
	SampleState st0[SQ_ROWS]; // (src -1) the row's sampler state
	int out[SQ_ROWS];         // where the row's token goes in pf.sqout
	int req[SQ_ROWS];         // the row's request, its slot in pf.sqst
	int greedy[SQ_ROWS];      // 1: the row takes the argmax (pf.greedy), 0: the sampler's token (pf.vsampled)
	int n;
};

// one warp, before a step: keep the table, then give each row its token and sampler state, taken from the previous step's
// row it continues or from the table.  Rows only move down, onto rows other lanes read, so every lane reads first.
__global__ void __launch_bounds__(32) k_sq_begin(const SqRows r, SqRows* tab, const int* prev, int* tokens, SampleState* st) {
	pdl_enter();
	const int i = threadIdx.x;
	for (int k = i; k < (int)(sizeof(SqRows) / sizeof(int)); k += 32) reinterpret_cast<int*>(tab)[k] = reinterpret_cast<const int*>(&r)[k];
	int tok = 0;
	SampleState s = {};
	if (i < r.n) {
		const int from = r.src[i];
		tok = from >= 0 ? prev[from] : r.tok0[i];
		s = from >= 0 ? st[from] : r.st0[i];
	}
	__syncwarp();
	if (i < r.n) tokens[i] = tok, st[i] = s;
}

// one warp, before a step whose rows have contexts: keep the step's groups table
__global__ void __launch_bounds__(32) k_sq_groups(const SqGroups gr, SqGroups* tab) {
	pdl_enter();
	for (int k = threadIdx.x; k < (int)(sizeof(SqGroups) / sizeof(int)); k += 32) reinterpret_cast<int*>(tab)[k] = reinterpret_cast<const int*>(&gr)[k];
}

// one warp, after a step: each row's token (the argmax or the sampler's) to the step's tokens and to the row's output
// slot, and a sampled row's generator state to its request
__global__ void __launch_bounds__(32) k_sq_end(const SqRows* tab, const int* greedy, const int* sampled, const SampleState* st, int* step_tok, int* out,
                                               unsigned long long* rng) {
	pdl_enter();
	const int i = threadIdx.x;
	if (i >= tab->n) return;
	const bool gr = tab->greedy[i];
	const int tok = gr ? greedy[i] : sampled[i];
	step_tok[i] = tok, out[tab->out[i]] = tok;
	if (!gr) rng[tab->req[i]] = st[i].rng;
}

// ---------------------------------------------------------------- calm_b200_decode_sample_queue_lookup

// The token each row's successor was fed, its draft (src -1 in SqRows), or -1 for a request's last row.  Passed by value
// to k_sq_accept.
struct SqNext {
	int tok[SQ_ROWS];
};

// one warp, in place of k_sq_end after a step with draft rows (a request's rows are contiguous, its draft rows after its
// first): row i is emitted when every earlier row of its request gave the token its successor was fed.  A row whose token
// differs from its successor's draft, or a request's last row, ends its request's run, so row i is emitted exactly when
// the nearest earlier run end (the ballot's highest bit below i) belongs to another request or there is none.  Every row's
// token goes to the step's tokens and its emitted flag to emitted[i]; an emitted row's token goes to its output slot, and
// a sampled request's generator state comes from its last emitted row alone, so each word has one writer.
__global__ void __launch_bounds__(32) k_sq_accept(const SqRows* tab, const SqNext nx, const int* greedy, const int* sampled, const SampleState* st,
                                                  int* step_tok, int* emitted, int* out, unsigned long long* rng) {
	pdl_enter();
	const int i = threadIdx.x;
	const bool in = i < tab->n;
	const bool gr = in && tab->greedy[i];
	const int tok = !in ? -1 : gr ? greedy[i] : sampled[i], req = in ? tab->req[i] : -1;
	const bool ends = in && tok != nx.tok[i];
	const unsigned below = __ballot_sync(0xffffffffu, ends) & ((1u << i) - 1u);
	const int h = 31 - __clz(below); // -1: no earlier run end
	const int hreq = __shfl_sync(0xffffffffu, req, h < 0 ? 0 : h);
	if (!in) return;
	const bool em = h < 0 || hreq != req;
	step_tok[i] = tok, emitted[i] = em;
	if (!em) return;
	out[tab->out[i]] = tok;
	if (ends && !gr) rng[req] = st[i].rng;
}

// ---------------------------------------------------------------- calm_b200_decode_sample_queue_logprobs

// one warp per row, after the sampler and before the merge of a step with log-probabilities: the row's target logit
// becomes its emitted token's, so that k_pf_logprob's tgt - M - ln S is that token's log-probability.  A sampled row's
// logit is its sampled token's entry of its logit row; a greedy row's token is the argmax, whose logit is the largest tile
// maximum (fmaxf is exact, so the order of the maxima does not matter).
__global__ void __launch_bounds__(32) k_sq_tgt(const SqRows* tab, const float2* part, int nvt, const float* logits, int vocab, const int* sampled,
                                               float* tgt) {
	pdl_enter();
	const int i = blockIdx.x, lane = threadIdx.x;
	if (tab->greedy[i]) {
		float m = -FLT_MAX;
		for (int v = lane; v < nvt; v += 32) m = fmaxf(m, part[(size_t)i * nvt + v].x);
		m = warp_max(m);
		if (lane == 0) tgt[i] = m;
	} else if (lane == 0) {
		tgt[i] = logits[(size_t)i * vocab + sampled[i]];
	}
}

// one warp, after the merge of a step with log-probabilities: each row's log-probability, and its k top ids and
// log-probabilities, to the row's output slot (its token's slot in pf.sqout; the top-k entries at k times that)
__global__ void __launch_bounds__(32) k_sq_lp(const SqRows* tab, const float* logprob, const int* top_ids, const float* top_lp, int k, float* out_lp,
                                              int* out_ids, float* out_tlp) {
	pdl_enter();
	const int n = tab->n;
	for (int i = threadIdx.x; i < n; i += 32) out_lp[tab->out[i]] = logprob[i];
	for (int e = threadIdx.x; e < n * k; e += 32) {
		const size_t o = (size_t)tab->out[e / k] * k + e % k;
		out_ids[o] = top_ids[e], out_tlp[o] = top_lp[e];
	}
}

// ---------------------------------------------------------------- calm_b200_decode_sample_queue_penalties

// A step's penalty lane (-1: a neutral request's row) and automaton state (-1: an unconstrained request's row) of each
// row, passed by value to k_sq_lanes
struct SqLanes {
	int lane[SQ_ROWS];
	int state[SQ_ROWS];
};
static_assert(sizeof(SqLanes) == 32 * sizeof(int), "one word per thread of k_sq_lanes' warp");

// one warp, before a step with a non-neutral or constrained row: keep the step's lanes and states, lanes[0 .. 16) and
// lanes[16 .. 32), where k_vf_gemm<.., PEN> (and <.., PEN, MASK>) and k_sq_pen_step read them
__global__ void __launch_bounds__(32) k_sq_lanes(const SqLanes l, int* lanes) {
	pdl_enter();
	lanes[threadIdx.x] = reinterpret_cast<const int*>(&l)[threadIdx.x];
}

// What k_sq_pen_admit needs of the request it admits to a lane: where its context, prompt and bias list lie in the
// call's uploaded tokens and bias arrays, and its (presence, frequency, repetition, 0)
struct SqPenAdmit {
	int lane, ctx_off, ctx_len, off, len, bias_off, bias_len;
	float4 par;
};

#define SQ_PEN_SPAN 1024 // vocabulary entries per CTA of k_sq_pen_admit

// one launch per non-neutral request a round admits, CTA b owning the lane's entries [b SQ_PEN_SPAN, (b + 1) SQ_PEN_SPAN):
// it clears them in the count and bias rows, then marks the tokens of ctx ++ prompt that fall among them seen and writes
// the bias list's values there (ids are distinct within a list), so that nothing of the lane's previous occupant
// remains.  Each entry is written by its own CTA only, the marks after the clear (__syncthreads orders a block's writes).
__global__ void __launch_bounds__(256) k_sq_pen_admit(const SqPenAdmit q, const int* tokens, const int* bias_ids, const float* bias_val, int vocab, int* cnt,
                                                      float* bias, float4* par) {
	pdl_enter();
	const int v0 = blockIdx.x * SQ_PEN_SPAN, v1 = min(v0 + SQ_PEN_SPAN, vocab);
	int* c = cnt + (size_t)q.lane * vocab;
	float* b = bias + (size_t)q.lane * vocab;
	for (int v = v0 + threadIdx.x; v < v1; v += blockDim.x) c[v] = 0, b[v] = 0.0f;
	__syncthreads();
	for (int i = threadIdx.x; i < q.ctx_len + q.len; i += blockDim.x) {
		const int tok = i < q.ctx_len ? tokens[q.ctx_off + i] : tokens[q.off + i - q.ctx_len];
		if (tok >= v0 && tok < v1) c[tok] = SQ_PEN_SEEN;
	}
	for (int i = threadIdx.x; i < q.bias_len; i += blockDim.x) {
		const int id = bias_ids[q.bias_off + i];
		if (id >= v0 && id < v1) b[id] = bias_val[q.bias_off + i];
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) par[q.lane] = q.par;
}

// one warp, after k_sq_end of a step with non-neutral rows: each such row's token counts once more in its lane, so the
// next step's classifier sees c(v) over the tokens of steps 0 .. j (a count > 0 also makes the token seen)
__global__ void __launch_bounds__(32) k_sq_pen_step(const int* lanes, const int* step_tok, int vocab, int* cnt) {
	pdl_enter();
	const int i = threadIdx.x;
	if (i < SQ_ROWS && lanes[i] >= 0) ++cnt[(size_t)lanes[i] * vocab + step_tok[i]];
}

// ---------------------------------------------------------------- calm_b200_decode_beam

#define BM_MAX 10      // CALM_B200_BEAM_MAX
#define BM_THREADS 256 // k_bm_select: one thread per candidate, at most BM_MAX x PF_TOPK_MAX of them

// A finished hypothesis: the tokens of row `row` of step `step` (its history), then `token` with log-probability `lp`
// (-1: none, a live beam entering the pool after the last step); `order` counts the call's entries into the pool
struct BmHyp {
	float score, sum, lp;
	int step, row, token, order;
};

// The pool of at most B finished hypotheses, and each live beam's running sum; zeroed before a call's first step
struct BmState {
	float sum[BM_MAX];
	BmHyp pool[BM_MAX];
	int npool, nadded, done;
};

// The row and token a live beam of step j + 1 continues, and the token's log-probability
struct BmBack {
	int parent, token;
	float lp;
};

// The pool rule of calm_b200_decode_beam (include/calm_b200.h): h enters while the pool holds fewer than B, or when its
// score is strictly greater than the worst; past B the worst leaves, the earliest added among equal worst scores.  The
// device's walk and the host's last step share it, so both keep the same pool.
__host__ __device__ inline int bm_worst(const BmState& s) {
	int w = 0;
	for (int i = 1; i < s.npool; ++i)
		if (s.pool[i].score < s.pool[w].score || (s.pool[i].score == s.pool[w].score && s.pool[i].order < s.pool[w].order)) w = i;
	return w;
}
__host__ __device__ inline void bm_add(BmState& s, int B, BmHyp h) {
	if (s.npool == B && !(h.score > s.pool[bm_worst(s)].score)) return;
	h.order = s.nadded++;
	if (s.npool < B) {
		s.pool[s.npool++] = h;
		return;
	}
	s.pool[bm_worst(s)] = h; // (one in, the worst out: the pool never holds more than B)
}

// What k_bm_select needs of one step
struct BmArgs {
	const int* tid;    // [rows][K] the step's merged top-K ids and log-probabilities (pf.sqtid / pf.sqtlp)
	const float* tlp;
	const int* anc;    // [B][max_new] the ancestry the step read, and the one the next step reads
	int* anc_next;
	BmState* st;
	BmBack* back;      // [max_new][B]
	int* trace_id;     // [max_new][B][K] every step's lists (rows past `rows`: id -1, -inf)
	float* trace_lp;
	int* tokens;       // [B] the next step's tokens (pf.tokens)
	int stop[PF_TOPK_MAX];
	int n_stop, j, rows, B, K, max_new, early;
	float norm_j, norm_next; // norm[max(1, j)] and norm[j + 1]
};

// one CTA, after the merge of step j: each candidate's score c = S_b + lp and its place in the walk order (c descending,
// beam ascending, rank ascending, found by counting the candidates before it), then the walk on one thread, then the next
// ancestry: anc'[b'][i] = anc[parent][i] for i <= j, and b' at j + 1
__global__ void __launch_bounds__(BM_THREADS) k_bm_select(const BmArgs a) {
	pdl_enter();
	__shared__ float cs[BM_MAX * PF_TOPK_MAX];
	__shared__ int walk[PF_TOPK_MAX], par[BM_MAX];
	__shared__ float S[BM_MAX]; // the next beams' sums
	const int n = a.rows * a.K, t = threadIdx.x;
	BmState* st = a.st;
	if (t < a.K) walk[t] = 0; // (places in the walk are distinct unless a score is NaN: no entry is left unset)
	if (t < a.B) par[t] = 0;
	for (int e = t; e < a.B * a.K; e += blockDim.x) {
		const bool in = e < n;
		const size_t o = ((size_t)a.j * a.B) * a.K + e;
		a.trace_id[o] = in ? a.tid[e] : -1, a.trace_lp[o] = in ? a.tlp[e] : -INFINITY;
		if (in) cs[e] = st->sum[e / a.K] + a.tlp[e];
	}
	__syncthreads();
	for (int e = t; e < n; e += blockDim.x) {
		const float c = cs[e];
		int q = 0; // (e / K, e % K) order as e does: beam, then rank
		for (int f = 0; f < n; ++f) q += cs[f] > c || (cs[f] == c && f < e);
		if (q < a.K) walk[q] = e;
	}
	__syncthreads();
	if (t == 0) {
		for (int b = 0; b < a.B; ++b) S[b] = -INFINITY;
		int taken = 0;
		for (int q = 0; q < a.K && taken < a.B; ++q) {
			const int e = walk[q], tok = a.tid[e];
			const float lp = a.tlp[e], c = cs[e];
			bool stop = false;
			for (int i = 0; i < a.n_stop; ++i) stop = stop || tok == a.stop[i];
			if (stop) {
				if (q < a.B) bm_add(*st, a.B, BmHyp{c / a.norm_j, c, lp, a.j, e / a.K, tok, 0});
				continue;
			}
			S[taken] = c, par[taken] = e / a.K, a.tokens[taken] = tok;
			a.back[(size_t)a.j * a.B + taken] = BmBack{e / a.K, tok, lp};
			++taken;
		}
		for (int b = 0; b < a.B; ++b) st->sum[b] = S[b];
		st->done = st->npool == a.B && (a.early || st->pool[bm_worst(*st)].score >= S[0] / a.norm_next);
	}
	__syncthreads();
	if (a.j + 1 >= a.max_new) return;
	for (int x = t; x < a.B * (a.j + 2); x += blockDim.x) {
		const int b = x / (a.j + 2), i = x % (a.j + 2);
		a.anc_next[(size_t)b * a.max_new + i] = i <= a.j ? a.anc[(size_t)par[b] * a.max_new + i] : b;
	}
}
