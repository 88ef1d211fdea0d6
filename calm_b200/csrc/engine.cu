// engine.cu -- host side of libcalm_b200.so: the reference's CUDA backend boundary
// (upload_cuda / prepare_cuda / forward_cuda / perf_cuda, reference src/run.c:22-25 and
// src/infer.cu:69-131, 651-801) implemented over the sm_90a kernels in stages.cuh.
//
// The per-token kernel sequence is captured once into CUDA graphs and replayed; per-token scalars
// live in a device-resident TokenParams record that the host (forward_cuda) or the device
// (greedy decode) rewrites between replays.

#include "../../include/calm_b200.h"

#include <dlfcn.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <iterator>
#include <map>
#include <set>
#include <vector>

#include "stages.cuh"
#include "attn.cuh"
#include "ring.cuh"
#include "prefill.cuh"
#include "verify.cuh"
#include "sample_n.cuh"

namespace {

#define MAX_STAMPS (2 + 5 * MAX_LAYERS)
#define TP_MAX_CAND 2048 // greedy candidates (classifier CTAs) per rank in the tensor-parallel gather area
enum Stage { ST_EMBED, ST_QKV, ST_ATTN, ST_WO, ST_FFN_UP, ST_FFN_DOWN, ST_OUTPUT, ST_COUNT };
const char* const kStageNames[ST_COUNT] = {"embed", "matmul_qkv", "attention", "matmul_attn", "matmul_ffn_up", "matmul_ffn_down", "output"};

// a planned launch: the kernel chosen for a stage and its launch shape
template <typename A>
struct Launch {
	void (*kernel)(A) = nullptr;
	int grid = 0, block = 0;
	size_t smem = 0;
};
struct ResLaunch : Launch<MatResArgs> {
	int S = 1; // k_matres_ring: MatResArgs::S
};

struct Engine {
	bool ready = false;
	int device = -1;
	int sms = 0;
	cudaStream_t stream = nullptr;
	struct Config cfg;
	struct Weights w;
	int kvbits = 16;
	int nact = 1;
	int q_dim = 0, kv_dim = 0, kv_mul = 1;

	// device buffers
	float *x = nullptr, *xb = nullptr, *q = nullptr, *att = nullptr, *hb = nullptr, *logits_dev = nullptr;
	float* logits_host = nullptr; // pinned + mapped
	void *kc = nullptr, *vc = nullptr;
	float* rope_freq = nullptr;
	float2* rope_cs = nullptr; // (cos, sin) of the current token's RoPE angles, written by k_embed
	unsigned long long* attn_cells = nullptr; // k_attn2's slice fold: {value, epoch} cells
	int* dev_err = nullptr;                   // mapped host word: watchdog code of an in-kernel wait that gave up
	float* attn_partial = nullptr;
	unsigned* attn_counter = nullptr;
	MoeSel* moe_sel = nullptr;
	TokenParams* tp = nullptr;
	float* cand_val = nullptr;
	int* cand_idx = nullptr;
	int* out_tokens = nullptr;
	int out_tokens_cap = 0;
	int* last_token = nullptr; // pinned + mapped
	int ncand = 0;

	// attention launch shape
	int attn_hg = 1, attn_qgroups = 1, attn_nsplit = 1, attn_lpp = 1;
	int attn_nbmax = 0;

	// launch plan, fixed at prepare time: the kernel that serves each shape-dependent stage, and its launch shape
	Launch<AttnArgs> attn; // k_attn2 (attn.cuh) or k_attn
	ResLaunch wo, down;    // k_matres_ring (ring.cuh) or k_matres
	Launch<FfnUpArgs> up;  // k_ffn_up_ring or k_ffn_up
	int grid_qkv = 0, grid_out = 0;
	size_t smem_dim = 0;
	int cur_kv_len = 0; // host copy, for the perf table only
	int cur_pos = 0;

	// tensor parallelism (staged engine): this process owns 1/tp_world of the heads and of the FFN rows
	int tp_rank = 0, tp_world = 1;
	void* tp_comm = nullptr;         // ncclComm_t
	float* xpart = nullptr;          // partial of wo / w2 before the all-reduce (NCCL path)
	bool tp_fused = false;           // wo / w2 sum their partials inside k_matres over peer memory (stages.cuh TpExchange)
	size_t up_expert_stride = 0;     // 16-byte vectors between experts of w1 / w3 once the rows are sharded
	int out_row0 = 0, out_row1 = 0;  // classifier rows of this rank (vocabulary split; the whole vocabulary without tensor parallelism)
	size_t tp_off_logits = 0, tp_off_cval = 0, tp_off_cidx = 0, tp_off_flags = 0; // byte offsets of the gather area inside every rank's exchange area
	void* tp_area = nullptr;         // this rank's exchange area: {partial, epoch} cells, then the logits gather area
	void* tp_peer[TP_MAX_WORLD] = {}; // every rank's area as mapped here (own entry == tp_area)
	int* tp_err = nullptr;           // mapped host word for the exchange watchdog
	std::vector<void*> tp_owned;     // shard copies made by prepare_cuda (wo / w2 column slices, packed biases)


	// one graph per call mode: 0 KV only, 1 logits to host, 2 greedy loop, 3 logits + argmax, 4 min-p sampling loop;
	// [1][mode] = the same token with stage stamps (perf_cuda)
	cudaGraphExec_t graph[2][5] = {};
	int graph_launches[2][5] = {};
	// device-side min-p sampler (stages.cuh k_sample_*)
	SampleState* sample_state = nullptr;
	int sample_chunks = 0;
	int* sample_count = nullptr;
	float* sample_csum = nullptr;
	int* sample_idx = nullptr;
	float* sample_prob = nullptr;
	bool use_graph = true;
	bool use_pdl = true;

	// profiling (perf_cuda): in-kernel %globaltimer stamps per launch of the production graph (stages.cuh stamp_begin/end)
	bool perf = false;
	bool debug = false;
	unsigned long long* stamps = nullptr;    // device [MAX_STAMPS][2]: {min start, max end} of each launch of the current token
	unsigned long long* stamp_acc = nullptr; // device [MAX_STAMPS + 2]: summed durations; [MAX_STAMPS] token span, [MAX_STAMPS + 1] tokens
	int n_stamps = 0;                        // launches with a slot in the current token
	int stamp_stage[MAX_STAMPS] = {};        // launch -> Stage
	double stamp_bytes[MAX_STAMPS] = {};     // algorithmic bytes of that launch (KV bytes use the host copy of kv_len)
	double stage_ms[ST_COUNT] = {};
	double stage_bytes[ST_COUNT] = {};
	long stage_launches[ST_COUNT] = {};
	double token_span_ms = 0;
	int perf_runs = 0;
	cudaEvent_t timer[2] = {nullptr, nullptr};
};

Engine g;

static_assert(PF_TOPK_MAX == CALM_B200_TOPK_MAX, "the tile lists hold the largest k a call accepts");

// batched prompt pass (prefill.cuh): buffers for up to `cap` tokens, allocated on first use
struct Prefill {
	int cap = 0;
	float *X = nullptr, *Q = nullptr;
	__half *Nhi = nullptr, *Nlo = nullptr, *Ahi = nullptr, *Alo = nullptr, *Hhi = nullptr, *Hlo = nullptr;
	float2* rope = nullptr;
	int* tokens = nullptr;
	int *rowpos = nullptr, *seg = nullptr; // packed blocks (calm_b200_score_batch / _context): a row's RoPE position, its sequence's first row
	int2* ctx = nullptr; // packed blocks that hold a context: a row's context, its first row and length
	CUtensorMap tmN[2], tmA[2], tmH[2]; // (hi, lo) views of the three activation matrices the GEMMs read
	// scoring (calm_b200_score), allocated on its first call for `cap` rows: the classifier's per-tile records, the targets'
	// logits, the targets and the log-probabilities
	bool scoring = false;
	float2* part = nullptr; // [cap][cdiv(vocab, PF_BM)]
	float *tgt = nullptr, *logprob = nullptr;
	int* targets = nullptr;
	// greedy scoring (calm_b200_score_greedy and its siblings), allocated on its first call for `cap` rows: each tile's
	// argmax and the merged argmax of each row
	int* gidx = nullptr; // [cap][cdiv(vocab, PF_BM)]
	int* greedy = nullptr;
	// top-k scoring (calm_b200_score_topk and its siblings), allocated on its first call for `cap` rows and the largest k:
	// each tile's sorted top-k list, and each row's merged top-k ids and log-probabilities
	float* topv = nullptr; // [cap][cdiv(vocab, PF_BM)][PF_TOPK_MAX]
	int* topi = nullptr;
	int* top_ids = nullptr; // [cap][PF_TOPK_MAX]
	float* top_lp = nullptr;
	// short blocks (calm_b200_verify_greedy), allocated on its first call: k_vf_gemm's partial sums, sized for the largest
	// GEMM of the model, and its arrival counters, which are zero between launches
	float* vacc = nullptr;
	size_t vacc_floats = 0;
	unsigned* vcnt = nullptr;
	// sampled short blocks (calm_b200_verify_sample), allocated on its first call: the block's logit rows and each tile's
	// maximum, and per row the sampler's survivor lists, chunk sums and counts, its SampleState and its token
	float* vlogits = nullptr; // [VF_TOK][vocab]
	float* vtmax = nullptr;   // [VF_TOK][cdiv(vocab, PF_BM)]
	int* vsidx = nullptr;     // [VF_TOK][sample_chunks * SAMPLE_CHUNK]
	float* vsprob = nullptr;
	float* vcsum = nullptr;   // [VF_TOK][sample_chunks]
	int* vcount = nullptr;
	SampleState* vstate = nullptr; // [VF_TOK]
	int* vsampled = nullptr;       // [VF_TOK]
	int vrows = 0;                 // rows of the last sampled block (CALM_B200_STATE_PF_LOGITS)
	// n samples of one prompt (calm_b200_decode_sample_n), allocated on its first call: the attention's chunk partials
	// (regrown when a call needs more chunks), the RoPE position of every row of the call and the tokens of every step
	float* snpart = nullptr; // [VF_TOK][n_heads][snchunks][head_dim + 2]
	int snchunks = 0;
	int* snpos = nullptr;    // [seq_len]: step j's rows at [j * nseq, (j + 1) * nseq)
	int* sntok = nullptr;    // [seq_len]: step j's tokens at [j * nseq, (j + 1) * nseq)
	// different prompts decoded together (calm_b200_decode_sample_batch), allocated on its first call: each row's prompt
	// in the packed cache, its first slot and length (uploaded once per call)
	int2* sbrows = nullptr; // [VF_TOK]
	// requests generated from a queue (calm_b200_decode_sample_queue), allocated on its first call and regrown when a call
	// needs more: the step's row table (written by k_sq_begin), the step's tokens, and every request's tokens and state
	SqRows* sqrows = nullptr;
	SqGroups* sqgroups = nullptr;      // the step's context groups (written by k_sq_groups), on steps whose rows have contexts
	int* sqtok = nullptr;              // [2 VF_TOK]: the step's tokens, then (k_sq_accept) each row's emitted flag
	int* sqout = nullptr;              // [sqout_cap]: request i's tokens from O_i = max_new[0] + .. + max_new[i - 1]
	unsigned long long* sqst = nullptr; // [sqst_cap]: request i's generator state after its last sampled step
	size_t sqout_cap = 0, sqst_cap = 0;
	// the queue's log-probabilities (calm_b200_decode_sample_queue_logprobs), allocated on its first call: a step's tile
	// lists and merged top-k for VF_TOK rows and the largest k, and every request's outputs, regrown like pf.sqout
	float* sqtopv = nullptr; // [VF_TOK][cdiv(vocab, PF_BM)][PF_TOPK_MAX]
	int* sqtopi = nullptr;
	int* sqtid = nullptr;    // [VF_TOK][PF_TOPK_MAX]
	float* sqtlp = nullptr;
	float* sqlp = nullptr;   // [sqlp_cap]: request i's log-probabilities from O_i
	int* sqoid = nullptr;    // [sqtop_cap]: request i's top-k ids and log-probabilities from O_i * k
	float* sqolp = nullptr;
	size_t sqlp_cap = 0, sqtop_cap = 0;
	// the queue's logit processing (calm_b200_decode_sample_queue_penalties), allocated on its first call with a
	// non-neutral request: each of the 16 lanes' count and bias rows and parameters (VfArgs::pcnt / pbias / ppar), and
	// the call's tokens and bias lists, uploaded once per call and regrown like pf.sqout
	int* sqpcnt = nullptr;    // [16][vocab]
	float* sqpbias = nullptr; // [16][vocab]
	float4* sqppar = nullptr; // [16]
	int* sqlanes = nullptr;   // [32] the step's lane of each row, and its automaton state from 16 (k_sq_lanes), allocated with pf.sqrows
	int* sqptok = nullptr;    // [sqptok_cap]
	int* sqpbid = nullptr;    // [sqpb_cap]
	float* sqpbval = nullptr;
	size_t sqptok_cap = 0, sqpb_cap = 0;
	// the automaton of calm_b200_decode_sample_queue_constrained: its states' bitmasks (VfArgs::allow), uploaded once per
	// call with a constrained request and regrown like pf.sqout
	uint32_t* sqallow = nullptr; // [sqallow_cap]
	size_t sqallow_cap = 0;
	// beam search (calm_b200_decode_beam), allocated on its first call and regrown when a call needs more: the ancestry
	// tables (double-buffered), the per-step backpointers and candidate lists, the pool; and the last call's shape
	int* bmanc[2] = {nullptr, nullptr}; // [bmanc_cap] each: [B][max_new]
	BmBack* bmback = nullptr;           // [bmback_cap]: [max_new][B]
	int* bmtid = nullptr;               // [bmtrace_cap]: [max_new][B][K]
	float* bmtlp = nullptr;
	BmState* bmst = nullptr;
	size_t bmanc_cap = 0, bmback_cap = 0, bmtrace_cap = 0;
	int bm_steps = 0, bm_beams = 0, bm_k = 0, bm_max_new = 0, bm_last = 0; // bm_last: the bmanc table the last step read
};
Prefill pf;

void pf_free() {
	cudaFree(pf.X), cudaFree(pf.Q), cudaFree(pf.Nhi), cudaFree(pf.Nlo), cudaFree(pf.Ahi), cudaFree(pf.Alo), cudaFree(pf.Hhi), cudaFree(pf.Hlo), cudaFree(pf.rope), cudaFree(pf.tokens);
	cudaFree(pf.rowpos), cudaFree(pf.seg), cudaFree(pf.ctx);
	cudaFree(pf.part), cudaFree(pf.tgt), cudaFree(pf.logprob), cudaFree(pf.targets);
	cudaFree(pf.gidx), cudaFree(pf.greedy);
	cudaFree(pf.topv), cudaFree(pf.topi), cudaFree(pf.top_ids), cudaFree(pf.top_lp);
	cudaFree(pf.vacc), cudaFree(pf.vcnt);
	cudaFree(pf.vlogits), cudaFree(pf.vtmax), cudaFree(pf.vsidx), cudaFree(pf.vsprob), cudaFree(pf.vcsum), cudaFree(pf.vcount), cudaFree(pf.vstate), cudaFree(pf.vsampled);
	cudaFree(pf.snpart), cudaFree(pf.snpos), cudaFree(pf.sntok), cudaFree(pf.sbrows);
	cudaFree(pf.sqrows), cudaFree(pf.sqgroups), cudaFree(pf.sqtok), cudaFree(pf.sqout), cudaFree(pf.sqst);
	cudaFree(pf.sqtopv), cudaFree(pf.sqtopi), cudaFree(pf.sqtid), cudaFree(pf.sqtlp), cudaFree(pf.sqlp), cudaFree(pf.sqoid), cudaFree(pf.sqolp);
	cudaFree(pf.sqpcnt), cudaFree(pf.sqpbias), cudaFree(pf.sqppar), cudaFree(pf.sqlanes), cudaFree(pf.sqptok), cudaFree(pf.sqpbid), cudaFree(pf.sqpbval);
	cudaFree(pf.sqallow);
	cudaFree(pf.bmanc[0]), cudaFree(pf.bmanc[1]), cudaFree(pf.bmback), cudaFree(pf.bmtid), cudaFree(pf.bmtlp), cudaFree(pf.bmst);
	pf = Prefill();
}

int g_device_override = -1;
uint64_t g_launches = 0;

void select_device() {
	if (g.device >= 0) return;
	int dev = g_device_override;
	if (dev < 0) {
		const char* e = getenv("CALM_B200_DEVICE");
		dev = e ? atoi(e) : 0;
	}
	int count = 0;
	cudaError_t err = cudaGetDeviceCount(&count);
	if (err != cudaSuccess || count == 0) CALM_FATAL("no CUDA device available (%s); this backend has no CPU fallback", cudaGetErrorString(err));
	if (dev >= count) CALM_FATAL("device %d requested but only %d present", dev, count);
	CUDA_CHECK(cudaSetDevice(dev));
	g.device = dev;
}

void* dev_alloc(size_t bytes) {
	void* p = nullptr;
	CUDA_CHECK(cudaMalloc(&p, bytes ? bytes : 16));
	return p;
}

// let `kernel` take `smem` bytes of dynamic shared memory (outside stream capture).  The attribute only ever grows, so a
// kernel launched at several sizes keeps the largest.
template <typename F>
void smem_optin(F kernel, size_t smem) {
	if (smem > 227 * 1024) CALM_FATAL("kernel needs %zu bytes of shared memory per CTA (limit 227 KB)", smem);
	cudaFuncAttributes fa;
	CUDA_CHECK(cudaFuncGetAttributes(&fa, kernel));
	if (smem > (size_t)fa.maxDynamicSharedSizeBytes) CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
}

// CTAs of `kernel` resident on the device at once, each with `smem` bytes of dynamic shared memory (opted in here)
template <typename F>
int max_ctas(F kernel, int block, size_t smem) {
	smem_optin(kernel, smem);
	int per_sm = 0;
	CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem));
	if (per_sm < 1) CALM_FATAL("kernel does not fit on an SM (block %d, %zu bytes of shared memory)", block, smem);
	return per_sm * g.sms;
}

int imin(int a, int b) { return a < b ? a : b; }
int cdiv(int a, int b) { return (a + b - 1) / b; }
// grid for `units` equal CTA-sized work items when at most `cap` CTAs are resident: every CTA gets the same
// number of rounds (a 3.03-rounds grid costs 4 rounds on some SMs and idles the rest)
int balanced_grid(int units, int cap) {
	if (units <= cap) return units < 1 ? 1 : units;
	return cdiv(units, cdiv(units, cap));
}

template <int DBITS>
size_t xs_bytes(int n) {
	return (size_t)(32 + xs_all_floats<DBITS>(n)) * sizeof(float);
}


// ---------------------------------------------------------------------------------------------
// NCCL, bound at run time (the library stays loadable and linkable without it; only tensor-parallel runs need it)

struct NcclApi {
	void* lib = nullptr;
	int (*GetUniqueId)(void*) = nullptr;
	int (*CommInitRank)(void**, int, /* ncclUniqueId by value: 128 bytes */ struct Id128, int) = nullptr;
	int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
	int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
	int (*CommDestroy)(void*) = nullptr;
	const char* (*GetErrorString)(int) = nullptr;
};
struct Id128 {
	char bytes[128];
};
NcclApi g_nccl;
Id128 g_tp_id;
bool g_tp_pending = false;
int g_tp_rank = 0, g_tp_world = 1;

void nccl_load() {
	if (g_nccl.lib) return;
	const char* names[] = {"libnccl.so.2", "libnccl.so"};
	for (const char* n : names)
		if ((g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL))) break;
	if (!g_nccl.lib) CALM_FATAL("tensor parallelism needs NCCL (libnccl.so.2): %s", dlerror());
	g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.lib, "ncclGetUniqueId");
	g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(g_nccl.lib, "ncclCommInitRank");
	g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.lib, "ncclAllReduce");
	g_nccl.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(g_nccl.lib, "ncclAllGather");
	g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.lib, "ncclCommDestroy");
	g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.lib, "ncclGetErrorString");
	if (!g_nccl.GetUniqueId || !g_nccl.CommInitRank || !g_nccl.AllReduce || !g_nccl.AllGather || !g_nccl.CommDestroy) CALM_FATAL("libnccl lacks the expected entry points");
}

#define NCCL_CHECK(x)                                                                                              \
	do {                                                                                                           \
		int r_ = (x);                                                                                              \
		if (r_ != 0) CALM_FATAL("NCCL error %d (%s) at %s:%d", r_, g_nccl.GetErrorString ? g_nccl.GetErrorString(r_) : "?", __FILE__, __LINE__); \
	} while (0)

// sum over ranks of a float vector, in stream order (captured into the CUDA graph like any kernel)
void tp_allreduce(float* buf, size_t count) {
	NCCL_CHECK(g_nccl.AllReduce(buf, buf, count, /*ncclFloat32*/ 7, /*ncclSum*/ 0, g.tp_comm, g.stream));
}

// Exchange areas for the fused matvec -> all-reduce (stages.cuh TpExchange): one cudaMalloc per rank, mapped into
// every peer with CUDA IPC (one process per GPU); the 64-byte handles travel through an NCCL all-gather.  Falls
// back to ncclAllReduce + k_addvec when peer mapping is unavailable on ANY rank (the ranks agree via an all-reduce).
void tp_setup_exchange() {
	const int W = g.tp_world, dim = g.cfg.dim;
	// cell[slot][src][row] | logits[vocab] | cand_val[W][TP_MAX_CAND] | cand_idx[W][TP_MAX_CAND] | flags[W]
	auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
	g.tp_off_logits = up((size_t)2 * W * dim * sizeof(uint2));
	g.tp_off_cval = g.tp_off_logits + up((size_t)g.cfg.vocab_size * sizeof(float));
	g.tp_off_cidx = g.tp_off_cval + up((size_t)W * TP_MAX_CAND * sizeof(float));
	g.tp_off_flags = g.tp_off_cidx + up((size_t)W * TP_MAX_CAND * sizeof(int));
	const size_t bytes = g.tp_off_flags + up((size_t)W * sizeof(unsigned));
	bool ok = W <= TP_MAX_WORLD && !(getenv("CALM_B200_TP_FUSED") && atoi(getenv("CALM_B200_TP_FUSED")) == 0);
	g.tp_area = dev_alloc(bytes);
	CUDA_CHECK(cudaMemset(g.tp_area, 0, bytes));
	cudaIpcMemHandle_t mine;
	if (cudaIpcGetMemHandle(&mine, g.tp_area) != cudaSuccess) ok = false, (void)cudaGetLastError();
	static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
	char* hdev = (char*)dev_alloc((size_t)W * 64 + sizeof(int));
	CUDA_CHECK(cudaMemcpy(hdev + (size_t)g.tp_rank * 64, &mine, 64, cudaMemcpyHostToDevice));
	NCCL_CHECK(g_nccl.AllGather(hdev + (size_t)g.tp_rank * 64, hdev, 64, /*ncclInt8*/ 0, g.tp_comm, g.stream));
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	std::vector<cudaIpcMemHandle_t> all(W);
	CUDA_CHECK(cudaMemcpy(all.data(), hdev, (size_t)W * 64, cudaMemcpyDeviceToHost));
	for (int p = 0; p < W && ok; ++p) {
		if (p == g.tp_rank) {
			g.tp_peer[p] = g.tp_area;
			continue;
		}
		if (cudaIpcOpenMemHandle(&g.tp_peer[p], all[p], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
			fprintf(stderr, "calm_b200: rank %d cannot map rank %d's exchange area (%s); using ncclAllReduce\n", g.tp_rank, p, cudaGetErrorString(cudaGetLastError()));
			g.tp_peer[p] = nullptr;
			ok = false;
		}
	}
	// every rank must take the same path: min over ranks of `ok`
	int* okdev = (int*)(hdev + (size_t)W * 64);
	int okh = ok ? 1 : 0;
	CUDA_CHECK(cudaMemcpy(okdev, &okh, sizeof(int), cudaMemcpyHostToDevice));
	NCCL_CHECK(g_nccl.AllReduce(okdev, okdev, 1, /*ncclInt32*/ 2, /*ncclMin*/ 3, g.tp_comm, g.stream));
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	CUDA_CHECK(cudaMemcpy(&okh, okdev, sizeof(int), cudaMemcpyDeviceToHost));
	CUDA_CHECK(cudaFree(hdev));
	g.tp_fused = okh == 1;
	if (g.tp_fused) {
		CUDA_CHECK(cudaHostAlloc((void**)&g.tp_err, sizeof(int), cudaHostAllocMapped));
		*g.tp_err = 0;
	}
}

void tp_fill(TpExchange& t, int idx) {
	t.world = g.tp_world, t.rank = g.tp_rank, t.idx = (unsigned)idx, t.stride = 2u * g.cfg.n_layers, t.tp = g.tp, t.err = g.tp_err;
	for (int p = 0; p < g.tp_world; ++p) t.cell[p] = (uint2*)g.tp_peer[p];
}

// Launch on the library's stream with programmatic stream serialization (PDL), so that consecutive kernels
// of a token overlap their launch latency (the kernels order themselves with griddepcontrol.wait).  Counts the launch.
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kernel)(KArgs...), dim3 grid, int block, size_t smem, Args... args) {
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = grid, cfg.blockDim = dim3(block), cfg.dynamicSmemBytes = smem, cfg.stream = g.stream;
	cudaLaunchAttribute at[1];
	at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
	at[0].val.programmaticStreamSerializationAllowed = g.use_pdl ? 1 : 0;
	cfg.attrs = at, cfg.numAttrs = 1;
	CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, args...));
	++g_launches;
}

template <typename A>
void launch(const Launch<A>& p, const A& a) {
	launch_pdl(p.kernel, p.grid, p.block, p.smem, a);
}

// planned at prepare time (outside stream capture): the launch's shared memory is opted in here
template <typename A>
Launch<A> plan(void (*kernel)(A), int grid, int block, size_t smem) {
	smem_optin(kernel, smem);
	return {kernel, grid, block, smem};
}

// the model's weight bits and KV cache element as template arguments: with_formats calls f(Formats<DBITS, KVT>())
template <int DBITS, typename KVT>
struct Formats {};

template <typename F>
void with_formats(F&& f) {
	switch (g.w.dbits * 100 + g.kvbits) {
	case 1616: return f(Formats<16, __half>());
	case 1608: return f(Formats<16, uint8_t>());
	case 816: return f(Formats<8, __half>());
	case 808: return f(Formats<8, uint8_t>());
	case 416: return f(Formats<4, __half>());
	default: return f(Formats<4, uint8_t>());
	}
}

// ---------------------------------------------------------------------------------------------
// one token = this sequence of launches

// A stage launch: hands out the stamp slot when the profiling graph is being built (NULL in the production graph) and,
// under CALM_B200_DEBUG=1, synchronises after the launch to name the stage that faults or hangs.
struct StageScope {
	Stage st;
	unsigned long long* slot = nullptr;
	StageScope(Stage s, double bytes) : st(s) {
		if (g.perf && g.n_stamps < MAX_STAMPS) {
			g.stamp_stage[g.n_stamps] = s, g.stamp_bytes[g.n_stamps] = bytes;
			slot = g.stamps + 2 * (size_t)g.n_stamps++;
		}
	}
	~StageScope() {
		if (g.debug) {
			cudaError_t e = cudaStreamSynchronize(g.stream);
			fprintf(stderr, "calm_b200: stage %s -> %s\n", kStageNames[st], cudaGetErrorName(e));
		}
	}
};

// end of a profiled token: fold the launch stamps into the running sums (one thread per slot)
__global__ void k_stamp_accum(const unsigned long long* stamps, unsigned long long* acc, int n) {
	pdl_enter();
	__shared__ unsigned long long lo[256], hi[256];
	unsigned long long mn = ~0ull, mx = 0;
	for (int i = threadIdx.x; i < n; i += blockDim.x) {
		const unsigned long long b = stamps[2 * i], e = stamps[2 * i + 1];
		if (b != ~0ull && e > b) {
			acc[i] += e - b;
			mn = b < mn ? b : mn, mx = e > mx ? e : mx;
		}
	}
	lo[threadIdx.x] = mn, hi[threadIdx.x] = mx;
	__syncthreads();
	if (threadIdx.x == 0) {
		for (int i = 1; i < (int)blockDim.x; ++i) mn = lo[i] < mn ? lo[i] : mn, mx = hi[i] > mx ? hi[i] : mx;
		if (mx > mn) acc[MAX_STAMPS] += mx - mn;
		acc[MAX_STAMPS + 1] += 1;
	}
}

// shared memory of k_attn<., HG>: the per-warp records of the in-CTA merge, or the coefficient tables of the slice merge
size_t attn_smem(int hg, int head_dim, int nsplit) {
	size_t smem = (size_t)(ATTN_THREADS / 32) * hg * (head_dim + 2) * sizeof(float);
	size_t smem2 = (size_t)(2 * nsplit + 1) * hg * sizeof(float);
	return smem2 > smem ? smem2 : smem;
}

// shapes k_attn2 is instantiated for: head_dim 128 with 4 or 8 query heads per kv head, head_dim 64 with 2, 4 or 8
bool attn2_shape_ok(int hg, int lpp, int head_dim) {
	return head_dim == lpp * 8 && ((lpp == 16 && (hg == 4 || hg == 8)) || (lpp == 8 && (hg == 2 || hg == 4 || hg == 8)));
}

typedef void (*AttnKernel)(AttnArgs);

template <typename KVT>
AttnKernel attn2_kernel(int hg, int lpp) {
	switch (lpp * 100 + hg) {
	case 1604: return k_attn2<KVT, 4, 128>;
	case 1608: return k_attn2<KVT, 8, 128>;
	case 802: return k_attn2<KVT, 2, 64>;
	case 804: return k_attn2<KVT, 4, 64>;
	case 808: return k_attn2<KVT, 8, 64>;
	}
	return nullptr;
}

template <typename KVT>
AttnKernel attn_kernel(int hg) {
	switch (hg) {
	case 1: return k_attn<KVT, 1>;
	case 2: return k_attn<KVT, 2>;
	case 3: return k_attn<KVT, 3>;
	case 4: return k_attn<KVT, 4>;
	case 5: return k_attn<KVT, 5>;
	case 6: return k_attn<KVT, 6>;
	case 7: return k_attn<KVT, 7>;
	default: return k_attn<KVT, 8>;
	}
}

// wo / w2: y += W . xin over this rank's share; under tensor parallelism the partials are summed over the ranks, inside the
// kernel over peer memory or by an NCCL all-reduce after it.  idx: the exchange slot of this projection.
void launch_res(const ResLaunch& p, MatResArgs& a, int idx) {
	const int dim = g.cfg.dim;
	a.S = p.S;
	if (g.tp_fused) tp_fill(a.tpx, idx);
	else if (g.tp_world > 1) a.y = g.xpart, a.accumulate = 0;
	launch(p, a);
	if (g.tp_world > 1 && !g.tp_fused) {
		tp_allreduce(g.xpart, dim);
		launch_pdl(k_addvec, cdiv(dim, 256), 256, 0, g.x, (const float*)g.xpart, dim);
	}
}

// mode: 0 kv only, 1 logits -> host, 2 logits -> device + advance (greedy loop), 3 logits -> host + argmax, 4 logits -> device + min-p sample + advance
template <int DBITS, typename KVT>
void run_token(Formats<DBITS, KVT>, int mode) {
	const Config& c = g.cfg;
	const Weights& w = g.w;
	const int dim = c.dim, hidden = c.hidden_dim, hd = c.head_dim;
	const size_t wb = (size_t)DBITS; // bits per weight
	g.n_stamps = 0;
	const size_t kv_layer = (size_t)c.n_kv_heads * c.seq_len * hd; // elements per layer

	{
		StageScope t(ST_EMBED, 0);
		EmbedArgs<KVT> a = {};
		a.x = g.x, a.table = w.token_embedding_table, a.tp = g.tp, a.dim = dim;
		a.embed_blocks = cdiv(dim, 256);
		a.key_cache = (KVT*)g.kc, a.rope_freq = g.rope_freq, a.rope_cs = g.rope_cs;
		a.n_layers = c.n_layers, a.n_kv_heads = c.n_kv_heads, a.head_dim = hd, a.seq_len = c.seq_len;
		a.stamp = nullptr, a.stamp_reset = g.perf ? g.stamps : nullptr, a.n_stamps = MAX_STAMPS + 8; // + the 16 debug stamps
		launch_pdl(k_embed<DBITS, KVT>, a.embed_blocks + 8, 256, 0, a);
	}

	for (int l = 0; l < c.n_layers; ++l) {
		{
			StageScope t(ST_QKV, (double)(g.q_dim + 2 * g.kv_dim) * dim * wb / 8);
			QkvArgs<KVT> a = {};
			a.x = g.x, a.normw = w.rms_att_weight[l], a.wq = w.wq[l], a.wk = w.wk[l], a.wv = w.wv[l], a.bias = w.bqkv[l];
			a.q_out = g.q, a.kc = (KVT*)g.kc + l * kv_layer, a.vc = (KVT*)g.vc + l * kv_layer;
			a.rope_cs = g.rope_cs, a.xb_out = c.norm_par ? g.xb : nullptr, a.tp = g.tp;
			a.dim = dim, a.q_dim = g.q_dim, a.kv_dim = g.kv_dim, a.head_dim = hd, a.seq_len = c.seq_len;
			a.eps = c.norm_eps, a.clip = c.qkv_clip, a.ln = c.norm_ln;
			a.stamp = t.slot;
			launch_pdl(k_qkv<DBITS, KVT>, g.grid_qkv, QKV_THREADS, g.smem_dim, a);
		}
		{
			StageScope t(ST_ATTN, -1.0); // bytes depend on the position: accounted per token in launch_token()
			AttnArgs a = {};
			a.q = g.q, a.kc = (KVT*)g.kc + l * kv_layer, a.vc = (KVT*)g.vc + l * kv_layer;
			a.partial = g.attn_partial, a.counter = g.attn_counter, a.out = g.att, a.tp = g.tp;
			a.head_dim = hd, a.seq_len = c.seq_len, a.nsplit = g.attn_nsplit, a.lpp = g.attn_lpp;
			a.kv_mul = g.kv_mul, a.qgroups = g.attn_qgroups;
			a.inv_sqrt_hd = 1.0f / sqrtf((float)hd);
			a.nbmax = g.attn_nbmax;
			a.cells = g.attn_cells, a.epoch_stride = (unsigned)c.n_layers + 1, a.epoch_idx = (unsigned)l + 1, a.err = g.dev_err;
			a.dbg = (g.perf && l == c.n_layers / 2) ? g.stamps + 2 * (size_t)MAX_STAMPS : nullptr;
			a.stamp = t.slot;
			launch(g.attn, a);
		}
		{
			StageScope t(ST_WO, (double)dim * g.q_dim * wb / 8);
			MatResArgs a = {};
			a.xin = g.att, a.w = w.wo[l], a.y = g.x, a.sel = nullptr, a.n = g.q_dim, a.d = dim, a.nact = 1, a.accumulate = 1;
			a.stamp = t.slot;
			launch_res(g.wo, a, 2 * l); // partial over this rank's heads
		}
		{
			StageScope t(ST_FFN_UP, (double)2 * g.nact * hidden * dim * wb / 8);
			FfnUpArgs a = {};
			a.x = (c.norm_par ? g.xb : g.x), a.normw = c.norm_par ? nullptr : w.rms_ffn_weight[l];
			a.gate = c.n_experts ? w.moegate[l] : nullptr, a.w1 = w.w1[l], a.w3 = w.w3[l], a.hb = g.hb, a.sel = g.moe_sel;
			a.dim = dim, a.hidden = hidden, a.n_experts = c.n_experts, a.nact = g.nact;
			a.eps = c.norm_eps, a.ln = c.norm_ln, a.gelu = c.act_gelu;
			a.expert_stride = g.up_expert_stride;
			a.stamp = t.slot;
			launch(g.up, a);
		}
		{
			StageScope t(ST_FFN_DOWN, (double)g.nact * hidden * dim * wb / 8);
			MatResArgs a = {};
			a.xin = g.hb, a.w = w.w2[l], a.y = g.x, a.sel = c.n_experts ? g.moe_sel : nullptr;
			a.n = hidden, a.d = dim, a.nact = g.nact, a.accumulate = 1;
			a.stamp = t.slot;
			launch_res(g.down, a, 2 * l + 1); // partial over this rank's FFN rows
		}
	}

	if (mode != 0) {
		StageScope t(ST_OUTPUT, (double)c.vocab_size * dim * wb / 8);
		OutputArgs a = {};
		a.x = g.x, a.normw = w.rms_final_weight, a.wcls = w.wcls;
		a.logits = (mode == 2 || mode == 4) ? g.logits_dev : g.logits_host;
		a.cand_val = (mode >= 2) ? g.cand_val : nullptr, a.cand_idx = g.cand_idx;
		a.dim = dim, a.vocab = c.vocab_size, a.eps = c.norm_eps, a.ln = c.norm_ln;
		a.stamp = t.slot;
		int grid = g.grid_out;
		const bool split = g.tp_fused; // classifier rows divided over the ranks, slices pushed into every rank's gather area
		int ncand = grid;
		const float* cand_val = g.cand_val;
		const int* cand_idx = g.cand_idx;
		if (split) {
			a.row0 = g.out_row0, a.row1 = g.out_row1, a.world = g.tp_world, a.rank = g.tp_rank;
			for (int p = 0; p < g.tp_world; ++p) {
				char* area = (char*)g.tp_peer[p];
				a.peer_logits[p] = (float*)(area + g.tp_off_logits), a.peer_cand_val[p] = (float*)(area + g.tp_off_cval), a.peer_cand_idx[p] = (int*)(area + g.tp_off_cidx);
			}
			ncand = grid * g.tp_world;
			cand_val = (const float*)((char*)g.tp_area + g.tp_off_cval), cand_idx = (const int*)((char*)g.tp_area + g.tp_off_cidx);
		}
		launch_pdl(k_output<DBITS>, grid, 256, g.smem_dim, a);
		if (split) {
			TpGatherArgs ga = {};
			ga.world = g.tp_world, ga.rank = g.tp_rank, ga.tp = g.tp, ga.err = g.tp_err;
			for (int p = 0; p < g.tp_world; ++p) ga.flags[p] = (unsigned*)((char*)g.tp_peer[p] + g.tp_off_flags);
			ga.src = (const float*)((char*)g.tp_area + g.tp_off_logits), ga.dst = a.logits, ga.n = c.vocab_size;
			launch_pdl(k_tp_gather, 32, 256, 0, ga);
		}
		if (mode == 4) { // min-p sampling on the device (reference sampler.c:44-90), then the bookkeeping of k_advance
			SampleArgs sa;
			sa.logits = g.logits_dev, sa.cand_val = cand_val, sa.ncand = ncand, sa.vocab = c.vocab_size, sa.nchunks = g.sample_chunks;
			sa.st = g.sample_state, sa.count = g.sample_count, sa.csum = g.sample_csum, sa.sidx = g.sample_idx, sa.sprob = g.sample_prob;
			launch_pdl(k_sample_scan, g.sample_chunks, 256, 0, sa);
			launch_pdl(k_sample_pick, 1, 256, 0, sa, g.sample_state, g.tp, g.out_tokens, g.last_token, 1);
		} else if (mode >= 2) {
			launch_pdl(k_advance, 1, 256, 0, cand_val, cand_idx, ncand, g.tp, g.out_tokens, g.last_token, (int)(mode == 2), c.vocab_size);
		}
	}
	if (g.perf) launch_pdl(k_stamp_accum, 1, 256, 0, (const unsigned long long*)g.stamps, g.stamp_acc, g.n_stamps);
}


// Tensor-parallel view of the model for rank r of N (Megatron split; SURVEY.md s.8e): query/kv heads and FFN rows
// are divided, so wq/wk/wv/w1/w3 shards are contiguous row ranges of the uploaded tensors (no copy), while wo and w2
// need their COLUMN range, packed once into a contiguous (dim x n/N) matrix.  Embedding, norms and the classifier
// are replicated.  After this the engine runs unchanged on the "local" shapes; the two partial projections per layer
// are summed with one all-reduce each.
void tp_shard_model() {
	Config& c = g.cfg;
	Weights& w = g.w;
	const int N = g.tp_world, r = g.tp_rank;
	const int ne = c.n_experts ? c.n_experts : 1; // MoE: the same split inside every expert (all ranks serve both active experts)
	if (c.n_heads % N || c.n_kv_heads % N || c.hidden_dim % (32 * N)) CALM_FATAL("tensor parallelism: %d ranks do not divide heads %d/%d or hidden %d", N, c.n_heads, c.n_kv_heads, c.hidden_dim);
	const size_t wb = (size_t)w.dbits;
	const int q_dim = c.head_dim * c.n_heads, kv_dim = c.head_dim * c.n_kv_heads;
	const int ql = q_dim / N, kl = kv_dim / N, hl = c.hidden_dim / N;
	auto rows = [&](void* base, size_t row0, size_t cols) { return (void*)((char*)base + row0 * cols * wb / 8); };
	auto col_slice = [&](const void* base, int nrows, size_t cols, size_t col0, size_t ncols) {
		void* dst = dev_alloc((size_t)nrows * ncols * wb / 8);
		CUDA_CHECK(cudaMemcpy2D(dst, ncols * wb / 8, (const char*)base + col0 * wb / 8, cols * wb / 8, ncols * wb / 8, nrows, cudaMemcpyDeviceToDevice));
		g.tp_owned.push_back(dst);
		return dst;
	};
	for (int l = 0; l < c.n_layers; ++l) {
		w.wq[l] = rows(w.wq[l], (size_t)r * ql, c.dim);
		w.wk[l] = rows(w.wk[l], (size_t)r * kl, c.dim);
		w.wv[l] = rows(w.wv[l], (size_t)r * kl, c.dim);
		w.w1[l] = rows(w.w1[l], (size_t)r * hl, c.dim); // expert e's rows start e * (full hidden) rows further: up_expert_stride
		w.w3[l] = rows(w.w3[l], (size_t)r * hl, c.dim);
		w.wo[l] = col_slice(w.wo[l], c.dim, q_dim, (size_t)r * ql, ql);
		w.w2[l] = col_slice(w.w2[l], ne * c.dim, c.hidden_dim, (size_t)r * hl, hl); // [expert][dim][hl], packed
		if (w.bqkv[l]) { // [q | k | v] -> this rank's [q_r | k_r | v_r]
			float* b = (float*)dev_alloc((size_t)(ql + 2 * kl) * sizeof(float));
			CUDA_CHECK(cudaMemcpy(b, w.bqkv[l] + (size_t)r * ql, ql * sizeof(float), cudaMemcpyDeviceToDevice));
			CUDA_CHECK(cudaMemcpy(b + ql, w.bqkv[l] + q_dim + (size_t)r * kl, kl * sizeof(float), cudaMemcpyDeviceToDevice));
			CUDA_CHECK(cudaMemcpy(b + ql + kl, w.bqkv[l] + q_dim + kv_dim + (size_t)r * kl, kl * sizeof(float), cudaMemcpyDeviceToDevice));
			g.tp_owned.push_back(b);
			w.bqkv[l] = b;
		}
	}
	if (c.n_experts) g.up_expert_stride = (size_t)c.hidden_dim * c.dim * wb / 8 / 16;
	c.n_heads /= N, c.n_kv_heads /= N, c.hidden_dim = hl;
}

// Choose the kernel and launch shape of every stage for this model and opt each kernel in to its shared memory (called once
// from prepare_cuda).  Kernels are first touched here in the order the library has always used: k_matres, attention, k_qkv,
// FFN up, the wo / w2 rings, k_output.  Under lazy module loading that order decides where their code is placed, and on an
// H100 (700 W) other orders moved decode by 0.2-0.3 % (Llama-3-8B faster, Mixtral-8x7B slower).
template <int DBITS, typename KVT>
void make_plan(Formats<DBITS, KVT>) {
	const Config& c = g.cfg;
	g.smem_dim = xs_bytes<DBITS>(c.dim);
	const size_t smem_qdim = xs_bytes<DBITS>(g.q_dim), smem_hidden = xs_bytes<DBITS>(c.hidden_dim);
	if (smem_qdim > 227 * 1024 || smem_hidden > 227 * 1024 || g.smem_dim > 227 * 1024) CALM_FATAL("activation vector does not fit in shared memory (dim %d, hidden %d)", c.dim, c.hidden_dim);
	const int grid_wo = balanced_grid(cdiv(c.dim / 2, 8), max_ctas(k_matres<DBITS>, 256, smem_qdim));
	const int grid_down = balanced_grid(cdiv(c.dim / 2, 8), max_ctas(k_matres<DBITS>, 256, smem_hidden));
	if (g.tp_fused) { // the in-kernel exchange needs co-resident grids (they are: balanced_grid stays under the cap) within its tables
		for (int grid : {grid_wo, grid_down})
			if (cdiv(c.dim / 2, grid * 8) > TP_MAX_ITERS) CALM_FATAL("tensor parallelism: grid %d outside the exchange tables for dim %d", grid, c.dim);
	}
	{
		// k_attn2 when the shape is instantiated, the CTA's share of the context fits in shared memory and the whole grid is
		// resident at once (the cell fold polls its peers); otherwise k_attn (global partials, last-CTA fold)
		const int units = c.n_kv_heads * g.attn_qgroups, grid = units * g.attn_nsplit;
		g.attn_nbmax = cdiv(cdiv(c.seq_len, ATTN2_BP), g.attn_nsplit);
		const size_t smem2 = attn2_smem_bytes<KVT>(g.attn_hg, c.head_dim, g.attn_nbmax);
		AttnKernel k2 = nullptr;
		if (attn2_shape_ok(g.attn_hg, g.attn_lpp, c.head_dim) && g.attn_nbmax <= ATTN2_MAXB && smem2 <= 200 * 1024) {
			k2 = attn2_kernel<KVT>(g.attn_hg, g.attn_lpp);
			if (max_ctas(k2, ATTN_THREADS, smem2) < grid) k2 = nullptr;
		}
		if (k2) g.attn = plan(k2, grid, ATTN_THREADS, smem2);
		else g.attn = plan(attn_kernel<KVT>(g.attn_hg), grid, ATTN_THREADS, attn_smem(g.attn_hg, c.head_dim, g.attn_nsplit));
		if (!getenv("CALM_B200_QUIET")) {
			printf("# plan: attention %s, %d units x %d slices\n", k2 ? "k_attn2" : "k_attn", units, g.attn_nsplit);
			fflush(stdout);
		}
	}
	g.grid_qkv = balanced_grid(cdiv((g.q_dim + 2 * g.kv_dim) / 2, 8), max_ctas(k_qkv<DBITS, KVT>, QKV_THREADS, g.smem_dim));
	// TMA-ring kernels for the dense stages whose rows are whole 1 KB / 2 KB chunks (ring.cuh)
	const bool ring_up_on = c.n_experts == 0; // MoE: the expert rows are known only after the router (row shards of w1 / w3 under tensor parallelism are fine)
	const bool ring_res_on = ring_up_on && (g.tp_world == 1 || g.tp_fused); // the ring kernels carry the in-kernel exchange too (gf4 too)
	auto chunk_units = [](size_t rowbytes) { return rowbytes % 2048 == 0 ? 4 : (rowbytes % 1024 == 0 ? 2 : 0); };
	// FFN up: k_ffn_up_ring or k_ffn_up (the long FFN-up stage gets a full grid with uneven rounds rather than balanced_grid's
	// even ones)
	g.up = {k_ffn_up<DBITS>, imin(max_ctas(k_ffn_up<DBITS>, 256, g.smem_dim), cdiv(g.nact * c.hidden_dim, 8)), 256, g.smem_dim};
	if (const int u = ring_up_on ? chunk_units((size_t)c.dim * DBITS / 8) : 0) {
		const size_t smem = ring_smem_bytes<DBITS>(c.dim, u, RING_UP_WARPS);
		if (smem <= 200 * 1024) {
			const int grid = imin(g.sms * imin(2, (int)(220 * 1024 / smem)), c.hidden_dim); // two CTAs per SM where they fit
			g.up = plan(u == 2 ? k_ffn_up_ring<DBITS, 2> : k_ffn_up_ring<DBITS, 4>, grid < 1 ? 1 : grid, RING_UP_WARPS * 32, smem);
		}
	}
	// wo (n = q_dim) and w2 (n = hidden): k_matres_ring when the rows are whole chunks and the ring fits, else k_matres
	auto plan_res = [&](int n, int grid_reg, size_t smem_reg) -> ResLaunch {
		const ResLaunch reg = {{k_matres<DBITS>, grid_reg, 256, smem_reg}};
		const size_t rowbytes = (size_t)n * DBITS / 8;
		int u = ring_res_on ? chunk_units(rowbytes) : 0;
		if (!u) return reg;
		size_t smem = ring_smem_bytes<DBITS>(n, u, RING_RES_WARPS);
		if (smem > 220 * 1024 && u == 4) u = 2, smem = ring_smem_bytes<DBITS>(n, u, RING_RES_WARPS); // long activation vectors (70B w2: 112 KB): 1 KB chunks
		if (smem > 220 * 1024) return reg;
		const int grid = imin(g.sms, c.dim / 2); // one CTA per SM
		const int cpt = (int)(rowbytes / (u * 512));
		if (g.tp_world > 1 && cdiv(c.dim / 2, grid) + 1 > RING_MAX_PAIRS) return reg; // the exchange keeps a CTA's rows in shared memory
		const bool split = cdiv(c.dim / 2, grid) + 1 <= RING_MAX_PAIRS && cpt <= RING_MAX_SLICES; // K-slices of one chunk, folded in shared memory
		return {plan(u == 2 ? k_matres_ring<DBITS, 2> : k_matres_ring<DBITS, 4>, grid < 1 ? 1 : grid, RING_RES_WARPS * 32, smem), split ? 1 : cpt};
	};
	g.wo = plan_res(g.q_dim, grid_wo, smem_qdim);
	g.down = plan_res(c.hidden_dim, grid_down, smem_hidden);
	if (!getenv("CALM_B200_QUIET")) {
		auto res_name = [](const ResLaunch& r) { return r.kernel == k_matres<DBITS> ? "k_matres" : "k_matres_ring"; };
		printf("# plan: matvec up %s, wo %s, down %s\n", g.up.kernel == k_ffn_up<DBITS> ? "k_ffn_up" : "k_ffn_up_ring", res_name(g.wo), res_name(g.down));
		fflush(stdout);
	}
	g.out_row0 = 0, g.out_row1 = c.vocab_size;
	if (g.tp_fused) { // vocabulary split: equal slices of whole 32-row CTA iterations (the last rank's may be short)
		const int per = cdiv(cdiv(c.vocab_size, g.tp_world), 32) * 32;
		g.out_row0 = imin(c.vocab_size, g.tp_rank * per), g.out_row1 = imin(c.vocab_size, g.out_row0 + per);
		g.grid_out = balanced_grid(cdiv(per, 32), max_ctas(k_output<DBITS>, 256, g.smem_dim)); // the same grid on every rank
		if (g.grid_out > TP_MAX_CAND) CALM_FATAL("tensor parallelism: %d classifier CTAs exceed the gather area", g.grid_out);
	} else {
		g.grid_out = balanced_grid(cdiv(c.vocab_size, 32), max_ctas(k_output<DBITS>, 256, g.smem_dim));
	}
	g.ncand = g.grid_out;
}

void launch_token(int mode) {
	const int pv = g.perf ? 1 : 0; // the profiling variant is the same graph with stamp slots
	auto run = [mode] { with_formats([mode](auto f) { run_token(f, mode); }); };
	if (!g.use_graph) {
		run();
		CUDA_CHECK(cudaGetLastError());
	} else {
		if (!g.graph[pv][mode]) {
			const uint64_t n0 = g_launches;
			cudaGraph_t graph;
			CUDA_CHECK(cudaStreamBeginCapture(g.stream, cudaStreamCaptureModeThreadLocal));
			run();
			CUDA_CHECK(cudaStreamEndCapture(g.stream, &graph));
			CUDA_CHECK(cudaGraphInstantiate(&g.graph[pv][mode], graph, 0));
			CUDA_CHECK(cudaGraphDestroy(graph));
			g.graph_launches[pv][mode] = (int)(g_launches - n0);
			g_launches = n0; // a captured launch counts when the graph runs
		}
		CUDA_CHECK(cudaGraphLaunch(g.graph[pv][mode], g.stream));
		g_launches += g.graph_launches[pv][mode];
	}
	if (g.perf) { // algorithmic bytes of this token per stage (the reference's accounting, infer.cu:683-699)
		const int n = g.cfg.n_layers * 5 + (mode != 0 ? 1 : 0) + 1;
		for (int i = 0; i < n && i < MAX_STAMPS; ++i) {
			const int st = g.stamp_stage[i];
			g.stage_bytes[st] += g.stamp_bytes[i] >= 0 ? g.stamp_bytes[i] : 2.0 * g.kv_dim * g.cur_kv_len * (g.kvbits / 8);
			g.stage_launches[st] += 1;
		}
		++g.perf_runs;
	}
}

void set_params(int token, int pos, int step) {
	g.cur_kv_len = pos >= g.cfg.seq_len ? g.cfg.seq_len : pos + 1;
	g.cur_pos = pos;
	k_set_params<<<1, 1, 0, g.stream>>>(g.tp, token, pos, g.cfg.seq_len, step);
	++g_launches;
}

} // namespace

// =================================================================================================
// C ABI

extern "C" int calm_b200_abi_version(void) {
	return CALM_B200_ABI_VERSION;
}

extern "C" void calm_b200_set_device(int device) {
	g_device_override = device;
}

extern "C" void* upload_cuda(void* host, size_t size) {
	select_device();
	void* dev = dev_alloc(size);
	CUDA_CHECK(cudaMemcpyAsync(dev, host, size, cudaMemcpyHostToDevice));
	return dev;
}

extern "C" void calm_b200_free(void* device_ptr) {
	if (device_ptr) CUDA_CHECK(cudaFree(device_ptr));
}

extern "C" void prepare_cuda(struct Transformer* transformer) {
	select_device();
	if (g.ready) CALM_FATAL("prepare_cuda called twice; call calm_b200_release() first (one model per process, as in the reference)");

	Config c = transformer->config; // copies: under tensor parallelism they become this rank's shard view
	Weights w = transformer->weights;
	RunState* s = &transformer->state;

	cudaDeviceProp prop;
	CUDA_CHECK(cudaGetDeviceProperties(&prop, g.device));
	if (prop.major != 9 || prop.minor != 0) CALM_FATAL("device %s is sm_%d%d; this library contains sm_90a code only and has no fallback", prop.name, prop.major, prop.minor);
	g.sms = prop.multiProcessorCount;
	if (!getenv("CALM_B200_QUIET"))
		printf("# CUDA: %s, compute %d.%d, %d SMs, %.1f GiB, peak bandwidth %.0f GB/s (ECC %d)\n", prop.name, prop.major, prop.minor, prop.multiProcessorCount,
		       (double)prop.totalGlobalMem / (1024 * 1024 * 1024), (double)prop.memoryClockRate * (prop.memoryBusWidth / 8) * 2 / 1e6, prop.ECCEnabled);

	// configuration checks (the reference asserts the same alignment, infer.cu:670, 755)
	if (w.dbits != 4 && w.dbits != 8 && w.dbits != 16) CALM_FATAL("unsupported dbits %d: must be 4, 8 or 16", w.dbits);
	if (s->kvbits != 8 && s->kvbits != 16) CALM_FATAL("unsupported kvbits %d: must be 8 or 16", s->kvbits);
	int q_dim = c.head_dim * c.n_heads, kv_dim = c.head_dim * c.n_kv_heads;
	if (c.dim % 32 || kv_dim % 32 || c.hidden_dim % 32 || q_dim % 32) CALM_FATAL("dim, q_dim, kv_dim and hidden_dim must be multiples of 32");
	if (c.head_dim % 8 || c.head_dim > 256) CALM_FATAL("head_dim %d unsupported (multiple of 8, <= 256)", c.head_dim);
	if (c.n_heads % c.n_kv_heads) CALM_FATAL("n_heads must be a multiple of n_kv_heads");
	if (c.n_layers > MAX_LAYERS) CALM_FATAL("too many layers");
	if (c.n_experts > MAX_EXPERTS || c.n_experts_ac > CALM_MAX_ACTIVE) CALM_FATAL("too many experts (%d, %d active)", c.n_experts, c.n_experts_ac);
	if (c.seq_len <= KV_SINKS) CALM_FATAL("seq_len too small");

	g.cfg = c;
	g.w = w;
	g.kvbits = s->kvbits;
	g.nact = c.n_experts ? c.n_experts_ac : 1;
	g.tp_rank = g_tp_rank, g.tp_world = g_tp_world;
	if (g.tp_world > 1) {
		nccl_load();
		NCCL_CHECK(g_nccl.CommInitRank(&g.tp_comm, g.tp_world, g_tp_id, g.tp_rank));
		tp_shard_model(); // g.cfg / g.w now describe this rank's shard
		c = g.cfg, w = g.w;
		q_dim = c.head_dim * c.n_heads, kv_dim = c.head_dim * c.n_kv_heads;
		if (kv_dim % 32 || c.hidden_dim % 32 || q_dim % 32) CALM_FATAL("tensor parallelism: per-rank q_dim, kv_dim and hidden_dim must be multiples of 32");
		g.xpart = (float*)dev_alloc(c.dim * sizeof(float));
	}
	g.q_dim = q_dim, g.kv_dim = kv_dim, g.kv_mul = g.cfg.n_heads / g.cfg.n_kv_heads;
	g.use_graph = !(getenv("CALM_B200_GRAPH") && atoi(getenv("CALM_B200_GRAPH")) == 0);
	g.use_pdl = !(getenv("CALM_B200_PDL") && atoi(getenv("CALM_B200_PDL")) == 0);
	g.debug = getenv("CALM_B200_DEBUG") && atoi(getenv("CALM_B200_DEBUG"));
	if (g.debug) g.use_graph = false;
	g.perf = (getenv("CALM_B200_PERF") && atoi(getenv("CALM_B200_PERF"))) || getenv("CUDA_INJECTION64_PATH");
	if (getenv("CALM_B200_PERF") && atoi(getenv("CALM_B200_PERF"))) { // the reference driver only calls perf_cuda under a CUPTI injection (run.c:630): print at exit
		static bool registered = false;
		if (!registered) atexit(perf_cuda), registered = true;
	}

	CUDA_CHECK(cudaStreamCreateWithFlags(&g.stream, cudaStreamNonBlocking));
	for (int i = 0; i < 2; ++i) CUDA_CHECK(cudaEventCreate(&g.timer[i]));
	g.stamps = (unsigned long long*)dev_alloc((size_t)(MAX_STAMPS * 2 + 16) * sizeof(unsigned long long));
	g.stamp_acc = (unsigned long long*)dev_alloc((size_t)(MAX_STAMPS + 2) * sizeof(unsigned long long));
	CUDA_CHECK(cudaMemset(g.stamps, 0, (size_t)(MAX_STAMPS * 2 + 16) * sizeof(unsigned long long)));
	CUDA_CHECK(cudaMemset(g.stamp_acc, 0, (size_t)(MAX_STAMPS + 2) * sizeof(unsigned long long)));
	if (g.tp_world > 1) { // first collective outside any graph capture: NCCL sets up its channels and buffers here
		CUDA_CHECK(cudaMemsetAsync(g.xpart, 0, c.dim * sizeof(float), g.stream));
		tp_allreduce(g.xpart, c.dim);
		CUDA_CHECK(cudaStreamSynchronize(g.stream));
		tp_setup_exchange();
	}

	g.x = (float*)dev_alloc(c.dim * sizeof(float));
	g.xb = (float*)dev_alloc(c.dim * sizeof(float));
	g.q = (float*)dev_alloc(q_dim * sizeof(float));
	g.att = (float*)dev_alloc(q_dim * sizeof(float));
	g.hb = (float*)dev_alloc((size_t)g.nact * c.hidden_dim * sizeof(float));
	g.logits_dev = (float*)dev_alloc((size_t)c.vocab_size * sizeof(float));
	CUDA_CHECK(cudaHostAlloc((void**)&g.logits_host, (size_t)c.vocab_size * sizeof(float), cudaHostAllocMapped));
	CUDA_CHECK(cudaHostAlloc((void**)&g.last_token, sizeof(int), cudaHostAllocMapped));
	memset(g.logits_host, 0, (size_t)c.vocab_size * sizeof(float));

	size_t kvbytes = (size_t)c.n_layers * c.seq_len * kv_dim * (g.kvbits / 8);
	g.kc = dev_alloc(kvbytes);
	g.vc = dev_alloc(kvbytes);
	CUDA_CHECK(cudaMemsetAsync(g.kc, 0, kvbytes, g.stream));
	CUDA_CHECK(cudaMemsetAsync(g.vc, 0, kvbytes, g.stream));

	// RoPE frequencies with the host libm, exactly as the CPU reference forms them (infer.c:225-226)
	std::vector<float> freq(c.head_dim / 2);
	for (int i = 0; i < c.head_dim; i += 2) freq[i / 2] = i >= c.rotary_dim ? 0.f : 1.0f / powf(c.rope_theta, (float)i / (float)c.rotary_dim);
	g.rope_cs = (float2*)dev_alloc(freq.size() * sizeof(float2));
	g.rope_freq = (float*)dev_alloc(freq.size() * sizeof(float));
	CUDA_CHECK(cudaMemcpyAsync(g.rope_freq, freq.data(), freq.size() * sizeof(float), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaStreamSynchronize(g.stream)); // freq is a local

	// attention shape: query-head group per CTA (largest divisor of kv_mul <= 8), lanes per position, slices
	g.attn_hg = 1;
	for (int h = 8; h >= 1; --h)
		if (g.kv_mul % h == 0) {
			g.attn_hg = h;
			break;
		}
	g.attn_qgroups = g.kv_mul / g.attn_hg;
	g.attn_lpp = 1;
	while (g.attn_lpp * 8 < c.head_dim) g.attn_lpp *= 2;
	int units = c.n_kv_heads * g.attn_qgroups;
	int want = g.sms / units; // about one 256-thread CTA per SM
	int maxsplit = cdiv(c.seq_len, 64);                 // at least 64 positions per slice at full context
	g.attn_nsplit = want < 1 ? 1 : (want > maxsplit ? maxsplit : want);
	if (g.attn_nsplit > ATTN2_MAXB + 4) g.attn_nsplit = ATTN2_MAXB + 4; // k_attn2 keeps one (m, l) pair per slice in static shared memory
	g.attn_partial = (float*)dev_alloc((size_t)units * g.attn_nsplit * g.attn_hg * (c.head_dim + 2) * sizeof(float));
	{
		const size_t cell_bytes = (size_t)units * g.attn_nsplit * g.attn_hg * (c.head_dim + 2) * sizeof(unsigned long long);
		// (the attention grid must be co-resident for the cell fold: units * nsplit CTAs of <= 1/2 SM each)
		g.attn_cells = (unsigned long long*)dev_alloc(cell_bytes);
		CUDA_CHECK(cudaMemset(g.attn_cells, 0, cell_bytes));
		CUDA_CHECK(cudaHostAlloc((void**)&g.dev_err, sizeof(int), cudaHostAllocMapped));
		*g.dev_err = 0;
	}
	g.attn_counter = (unsigned*)dev_alloc(units * sizeof(unsigned));
	CUDA_CHECK(cudaMemset(g.attn_counter, 0, units * sizeof(unsigned)));

	g.moe_sel = (MoeSel*)dev_alloc(sizeof(MoeSel));
	CUDA_CHECK(cudaMemset(g.moe_sel, 0, sizeof(MoeSel)));
	g.tp = (TokenParams*)dev_alloc(sizeof(TokenParams));
	CUDA_CHECK(cudaMemset(g.tp, 0, sizeof(TokenParams)));

	with_formats([](auto f) { make_plan(f); });
	g.cand_val = (float*)dev_alloc(g.ncand * sizeof(float));
	g.cand_idx = (int*)dev_alloc(g.ncand * sizeof(int));
	g.out_tokens_cap = 1 << 16;
	g.out_tokens = (int*)dev_alloc(g.out_tokens_cap * sizeof(int));
	g.sample_chunks = cdiv(c.vocab_size, SAMPLE_CHUNK);
	g.sample_state = (SampleState*)dev_alloc(sizeof(SampleState));
	g.sample_count = (int*)dev_alloc(g.sample_chunks * sizeof(int));
	g.sample_csum = (float*)dev_alloc(g.sample_chunks * sizeof(float));
	g.sample_idx = (int*)dev_alloc((size_t)g.sample_chunks * SAMPLE_CHUNK * sizeof(int));
	g.sample_prob = (float*)dev_alloc((size_t)g.sample_chunks * SAMPLE_CHUNK * sizeof(float));

	// what the reference backend publishes in RunState (infer.cu:99-112)
	s->x = g.x, s->hb = g.hb, s->he = g.hb, s->q = g.q, s->att = g.att;
	s->key_cache = g.kc, s->value_cache = g.vc;
	s->logits = g.logits_host;

	g.ready = true;
	CUDA_CHECK(cudaDeviceSynchronize());
}

extern "C" void calm_b200_tp_unique_id(void* out128) {
	select_device();
	nccl_load();
	Id128 id;
	memset(&id, 0, sizeof(id));
	NCCL_CHECK(g_nccl.GetUniqueId(&id));
	memcpy(out128, &id, sizeof(id));
}

extern "C" void calm_b200_tp_init(int rank, int world, const void* id128) {
	if (g.ready) CALM_FATAL("calm_b200_tp_init must precede prepare_cuda");
	if (world < 1 || rank < 0 || rank >= world) CALM_FATAL("calm_b200_tp_init: bad rank %d of %d", rank, world);
	g_tp_rank = rank, g_tp_world = world;
	if (world > 1) memcpy(&g_tp_id, id128, sizeof(g_tp_id));
}

extern "C" int calm_b200_tp_world(void) {
	return g.ready ? g.tp_world : g_tp_world;
}

extern "C" int calm_b200_tp_mode(void) {
	return !g.ready || g.tp_world <= 1 ? 0 : (g.tp_fused ? 2 : 1);
}

extern "C" void calm_b200_release(struct Transformer* transformer) {
	if (!g.ready) return;
	CUDA_CHECK(cudaDeviceSynchronize());
	for (int v = 0; v < 2; ++v)
		for (int i = 0; i < 5; ++i)
			if (g.graph[v][i]) CUDA_CHECK(cudaGraphExecDestroy(g.graph[v][i]));
	cudaFree(g.stamps), cudaFree(g.stamp_acc), cudaFree(g.attn_cells);
	if (g.dev_err) cudaFreeHost(g.dev_err);
	pf_free();
	cudaFree(g.x), cudaFree(g.xb), cudaFree(g.q), cudaFree(g.att), cudaFree(g.hb), cudaFree(g.logits_dev);
	cudaFreeHost(g.logits_host), cudaFreeHost(g.last_token);
	cudaFree(g.kc), cudaFree(g.vc), cudaFree(g.rope_freq), cudaFree(g.rope_cs), cudaFree(g.attn_partial), cudaFree(g.attn_counter);
	cudaFree(g.moe_sel), cudaFree(g.tp), cudaFree(g.cand_val), cudaFree(g.cand_idx), cudaFree(g.out_tokens);
	for (int p = 0; p < TP_MAX_WORLD; ++p)
		if (g.tp_peer[p] && g.tp_peer[p] != g.tp_area) cudaIpcCloseMemHandle(g.tp_peer[p]);
	if (g.tp_area) cudaFree(g.tp_area);
	if (g.tp_err) cudaFreeHost(g.tp_err);
	cudaFree(g.sample_state), cudaFree(g.sample_count), cudaFree(g.sample_csum), cudaFree(g.sample_idx), cudaFree(g.sample_prob);
	if (g.tp_comm) g_nccl.CommDestroy(g.tp_comm);
	if (g.xpart) cudaFree(g.xpart);
	for (void* p : g.tp_owned) cudaFree(p);
	g_tp_world = 1, g_tp_rank = 0; // a new communicator needs a new calm_b200_tp_init
	for (int i = 0; i < 2; ++i) cudaEventDestroy(g.timer[i]);
	cudaStreamDestroy(g.stream);
	int dev = g.device;
	g = Engine();
	g.device = dev;
	if (transformer) {
		int kvbits = transformer->state.kvbits;
		memset(&transformer->state, 0, sizeof(transformer->state));
		transformer->state.kvbits = kvbits;
	}
}

static void sync_stream() {
	cudaError_t e = cudaStreamSynchronize(g.stream);
	if (e != cudaSuccess) {
		int code = g.tp_err ? *(volatile int*)g.tp_err : 0; // 9000 + the rank never heard from
		if (!code && g.dev_err) code = *(volatile int*)g.dev_err; // 9200: a slice of the attention fold never arrived
		fprintf(stderr, "calm_b200: device failure: %s (%s); watchdog code %d\n", cudaGetErrorString(e), cudaGetErrorName(e), code);
		abort();
	}
}

static void check_call(struct Transformer* transformer, int token, int pos) {
	if (!g.ready) CALM_FATAL("forward before prepare_cuda");
	(void)transformer;
	if (token < 0 || token >= g.cfg.vocab_size) CALM_FATAL("token %d out of range", token);
	if (pos < 0) CALM_FATAL("negative position");
}

extern "C" float* forward_cuda(struct Transformer* transformer, int token, int pos, unsigned flags) {
	check_call(transformer, token, pos);
	set_params(token, pos, 0);
	if (flags & FF_UPDATE_KV_ONLY) {
		launch_token(0);
		return NULL; // no synchronisation: prompt tokens pipeline (reference infer.cu:724-727)
	}
	launch_token(1);
	sync_stream();
	CUDA_CHECK(cudaGetLastError());
	return g.logits_host;
}

extern "C" int calm_b200_forward_argmax(struct Transformer* transformer, int token, int pos) {
	check_call(transformer, token, pos);
	set_params(token, pos, 0);
	launch_token(3);
	sync_stream();
	return *(volatile int*)g.last_token;
}

extern "C" void calm_b200_decode_greedy(struct Transformer* transformer, int token0, int pos0, int n_tokens, int* out_tokens) {
	check_call(transformer, token0, pos0);
	if (n_tokens > g.out_tokens_cap) CALM_FATAL("decode_greedy: at most %d tokens per call", g.out_tokens_cap);
	set_params(token0, pos0, 0);
	for (int i = 0; i < n_tokens; ++i) {
		g.cur_pos = pos0 + i, g.cur_kv_len = g.cur_pos >= g.cfg.seq_len ? g.cfg.seq_len : g.cur_pos + 1;
		launch_token(2);
	}
	sync_stream();
	CUDA_CHECK(cudaMemcpy(out_tokens, g.out_tokens, n_tokens * sizeof(int), cudaMemcpyDeviceToHost));
}

// min-p / temperature sampling without a host round trip per token (reference sample(), sampler.c:80-90)
extern "C" void calm_b200_decode_sample(struct Transformer* transformer, int token0, int pos0, int n_tokens, float temperature, float minp,
                                        unsigned long long* rng_state, int* out_tokens) {
	if (temperature == 0.0f || minp >= 1.0f) { // greedy: the reference does not touch the generator either
		calm_b200_decode_greedy(transformer, token0, pos0, n_tokens, out_tokens);
		return;
	}
	check_call(transformer, token0, pos0);
	if (n_tokens > g.out_tokens_cap) CALM_FATAL("decode_sample: at most %d tokens per call", g.out_tokens_cap);
	SampleState st;
	st.rng = *rng_state, st.temperature = temperature, st.cut_delta = logf(minp) * temperature;
	CUDA_CHECK(cudaMemcpyAsync(g.sample_state, &st, sizeof(st), cudaMemcpyHostToDevice, g.stream));
	set_params(token0, pos0, 0);
	for (int i = 0; i < n_tokens; ++i) {
		g.cur_pos = pos0 + i, g.cur_kv_len = g.cur_pos >= g.cfg.seq_len ? g.cfg.seq_len : g.cur_pos + 1;
		launch_token(4);
	}
	sync_stream();
	CUDA_CHECK(cudaMemcpy(out_tokens, g.out_tokens, n_tokens * sizeof(int), cudaMemcpyDeviceToHost));
	CUDA_CHECK(cudaMemcpy(&st, g.sample_state, sizeof(st), cudaMemcpyDeviceToHost));
	*rng_state = st.rng;
}

extern "C" int calm_b200_forward_sample(struct Transformer* transformer, int token, int pos, float temperature, float minp, unsigned long long* rng_state) {
	int tok = 0;
	calm_b200_decode_sample(transformer, token, pos, 1, temperature, minp, rng_state, &tok);
	return tok;
}

// The state step of the reference's xorshift* generator (sampler.c:7-13), which k_sample_pick takes once per draw: the
// states of a run of draws do not depend on the logits, so the host can form them
static unsigned long long xorshift_step(unsigned long long s) {
	s ^= s >> 12;
	s ^= s << 25;
	s ^= s >> 27;
	return s;
}

// k_sample_trunc_rows over grid (TRUNC_CTAS, rows) on `st`, each CTA staging its ceil(vocab / TRUNC_CTAS) logits
static void trunc_launch(dim3 grid, cudaStream_t st, const SampleArgs& sa, const TruncRows& tr, int vocab) {
	const size_t smem = (size_t)(cdiv(vocab, TRUNC_CTAS) + 8) * sizeof(float);
	static size_t opted = 0;
	if (smem > opted) {
		CUDA_CHECK(cudaFuncSetAttribute(k_sample_trunc_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		opted = smem;
	}
	if (st == g.stream) {
		launch_pdl(k_sample_trunc_rows, grid, 256, smem, sa, tr);
		return;
	}
	k_sample_trunc_rows<<<grid, 256, smem, st>>>(sa, tr);
}

// abort unless top_k >= 0 and top_p is finite in (0, 1] (request i's, in `who`)
static void trunc_check(const char* who, int i, int top_k, float top_p) {
	if (top_k < 0) CALM_FATAL("%s: request %d's top_k %d is negative", who, i, top_k);
	if (!(top_p > 0.0f && top_p <= 1.0f)) CALM_FATAL("%s: request %d's top_p %g is not in (0, 1]", who, i, (double)top_p);
}

// The device sampler on its own: logits given by the host, any vocabulary size; returns the token and advances *rng_state.
// Same kernels as the decode loop (k_sample_scan + k_sample_pick); device_us (optional) receives their mean duration.
// `masked` (the fallback of calm_b200_decode_sample_queue_constrained): k_sample_scan_rows_masked on the one row instead
// of k_sample_scan, so that a -inf logit never survives.  top_k > 0 or top_p < 1 (calm_b200_sample_logits_truncated):
// k_sample_trunc_rows on the row first, then the masked scan; out_row (may be NULL) receives the row it left.
static int sample_logits(const float* logits_host, int vocab, float temperature, float minp, unsigned long long* rng_state, float* device_us, bool masked,
                         int top_k = 0, float top_p = 1.0f, float* out_row = nullptr) {
	select_device();
	if (vocab <= 0) CALM_FATAL("sample_logits: empty vocabulary");
	if (out_row) std::copy(logits_host, logits_host + vocab, out_row);
	if (temperature == 0.0f || minp >= 1.0f) { // greedy, first maximum (sampler.c:34-42); the generator is not touched
		int best = 0;
		for (int i = 1; i < vocab; ++i)
			if (logits_host[i] > logits_host[best]) best = i;
		if (device_us) *device_us = 0.f;
		return best;
	}
	const bool trunc = top_k > 0 || top_p < 1.0f;
	if (trunc && vocab > TRUNC_VOCAB_MAX) CALM_FATAL("sample_logits: truncation serves vocabularies up to %d tokens, not %d", TRUNC_VOCAB_MAX, vocab);
	masked = masked || trunc;
	const int nchunks = cdiv(vocab, SAMPLE_CHUNK);
	cudaStream_t st;
	CUDA_CHECK(cudaStreamCreate(&st));
	float* logits = (float*)dev_alloc((size_t)vocab * sizeof(float));
	float* cmax = (float*)dev_alloc(nchunks * sizeof(float));
	SampleState* sst = (SampleState*)dev_alloc(sizeof(SampleState));
	int* count = (int*)dev_alloc(nchunks * sizeof(int));
	float* csum = (float*)dev_alloc(nchunks * sizeof(float));
	int* sidx = (int*)dev_alloc((size_t)nchunks * SAMPLE_CHUNK * sizeof(int));
	float* sprob = (float*)dev_alloc((size_t)nchunks * SAMPLE_CHUNK * sizeof(float));
	int* tok = (int*)dev_alloc(sizeof(int));
	TokenParams* tp = (TokenParams*)dev_alloc(sizeof(TokenParams));
	CUDA_CHECK(cudaMemcpyAsync(logits, logits_host, (size_t)vocab * sizeof(float), cudaMemcpyHostToDevice, st));
	SampleState hs;
	hs.rng = *rng_state, hs.temperature = temperature, hs.cut_delta = logf(minp) * temperature;
	SampleArgs sa;
	sa.logits = logits, sa.cand_val = cmax, sa.ncand = nchunks, sa.vocab = vocab, sa.nchunks = nchunks;
	sa.st = sst, sa.count = count, sa.csum = csum, sa.sidx = sidx, sa.sprob = sprob;
	cudaEvent_t e0, e1;
	CUDA_CHECK(cudaEventCreate(&e0));
	CUDA_CHECK(cudaEventCreate(&e1));
	const int reps = device_us ? 5 : 1;
	float ms = 0;
	for (int r = 0; r < reps; ++r) { // every repetition restarts from the caller's generator state: same draw
		CUDA_CHECK(cudaMemcpyAsync(sst, &hs, sizeof(hs), cudaMemcpyHostToDevice, st));
		if (trunc) CUDA_CHECK(cudaMemcpyAsync(logits, logits_host, (size_t)vocab * sizeof(float), cudaMemcpyHostToDevice, st)); // (truncated in place)
		k_chunk_max<<<nchunks, 256, 0, st>>>(logits, vocab, cmax);
		CUDA_CHECK(cudaEventRecord(e0, st));
		if (trunc) {
			TruncRows tr = {};
			tr.top_k[0] = top_k, tr.top_p[0] = top_p;
			trunc_launch(dim3(TRUNC_CTAS, 1), st, sa, tr, vocab);
			g_launches += 1;
		}
		if (masked) k_sample_scan_rows_masked<<<dim3(nchunks, 1), 256, 0, st>>>(sa);
		else k_sample_scan<<<nchunks, 256, 0, st>>>(sa);
		k_sample_pick<<<1, 256, 0, st>>>(sa, sst, tp, nullptr, tok, 0);
		CUDA_CHECK(cudaEventRecord(e1, st));
		CUDA_CHECK(cudaEventSynchronize(e1));
		CUDA_CHECK(cudaGetLastError());
		CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
		g_launches += 3;
	}
	if (device_us) *device_us = ms * 1e3f;
	int htok = 0;
	CUDA_CHECK(cudaMemcpy(&htok, tok, sizeof(int), cudaMemcpyDeviceToHost));
	CUDA_CHECK(cudaMemcpy(&hs, sst, sizeof(hs), cudaMemcpyDeviceToHost));
	if (trunc && out_row) CUDA_CHECK(cudaMemcpy(out_row, logits, (size_t)vocab * sizeof(float), cudaMemcpyDeviceToHost));
	*rng_state = hs.rng;
	cudaFree(logits), cudaFree(cmax), cudaFree(sst), cudaFree(count), cudaFree(csum), cudaFree(sidx), cudaFree(sprob), cudaFree(tok), cudaFree(tp);
	cudaEventDestroy(e0), cudaEventDestroy(e1), cudaStreamDestroy(st);
	return htok;
}

extern "C" int calm_b200_sample_logits(const float* logits_host, int vocab, float temperature, float minp, unsigned long long* rng_state, float* device_us) {
	return sample_logits(logits_host, vocab, temperature, minp, rng_state, device_us, false);
}

extern "C" int calm_b200_sample_logits_truncated(const float* logits_host, int vocab, float temperature, float minp, int top_k, float top_p,
                                                 unsigned long long* rng_state, float* out_row, float* device_us) {
	trunc_check("sample_logits_truncated", 0, top_k, top_p);
	return sample_logits(logits_host, vocab, temperature, minp, rng_state, device_us, false, top_k, top_p, out_row);
}

// ---------------------------------------------------------------------------------------------
// forward_prefill_cuda: the prompt as one batched pass (SURVEY.md s.8b "additive entry points"; reference run.c:206-209 calls
// forward(..., FF_UPDATE_KV_ONLY) once per prompt token).

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void pf_make_map(CUtensorMap* map, void* base, int rows, int cols) { // f16 [rows][cols], box = 128 rows x 64 columns, 128-byte swizzle
	static EncodeTiledFn encode = nullptr;
	if (!encode) {
		cudaDriverEntryPointQueryResult qres;
		void* fn = nullptr;
		CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
		if (!fn || qres != cudaDriverEntryPointSuccess) CALM_FATAL("cuTensorMapEncodeTiled is not available from this driver");
		encode = (EncodeTiledFn)fn;
	}
	const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
	const cuuint64_t strides[1] = {(cuuint64_t)cols * sizeof(__half)};
	const cuuint32_t box[2] = {PF_BK, PF_BN}, estr[2] = {1, 1};
	CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
	                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS) CALM_FATAL("cuTensorMapEncodeTiled failed (%d) for a %d x %d f16 matrix", (int)r, rows, cols);
}

static void pf_reserve(int n) {
	const Config& c = g.cfg;
	int cap = cdiv(n, PF_BN) * PF_BN;
	if (cap <= pf.cap) return;
	if (pf.cap) {
		CUDA_CHECK(cudaStreamSynchronize(g.stream));
		pf_free();
	}
	pf.cap = cap;
	auto zalloc = [&](size_t bytes) {
		void* p = dev_alloc(bytes);
		CUDA_CHECK(cudaMemset(p, 0, bytes)); // defined bytes for the first pass; later, padding rows of a partial token tile hold an earlier pass's values
		return p;
	};
	pf.X = (float*)zalloc((size_t)cap * c.dim * sizeof(float));
	pf.Q = (float*)zalloc((size_t)cap * g.q_dim * sizeof(float));
	pf.Nhi = (__half*)zalloc((size_t)cap * c.dim * sizeof(__half)), pf.Nlo = (__half*)zalloc((size_t)cap * c.dim * sizeof(__half));
	pf.Ahi = (__half*)zalloc((size_t)cap * g.q_dim * sizeof(__half)), pf.Alo = (__half*)zalloc((size_t)cap * g.q_dim * sizeof(__half));
	pf.Hhi = (__half*)zalloc((size_t)cap * c.hidden_dim * sizeof(__half)), pf.Hlo = (__half*)zalloc((size_t)cap * c.hidden_dim * sizeof(__half));
	pf.rope = (float2*)zalloc((size_t)cap * (c.head_dim / 2) * sizeof(float2));
	pf.tokens = (int*)zalloc((size_t)cap * sizeof(int));
	pf.rowpos = (int*)zalloc((size_t)cap * sizeof(int)), pf.seg = (int*)zalloc((size_t)cap * sizeof(int));
	pf.ctx = (int2*)zalloc((size_t)cap * sizeof(int2));
	pf_make_map(&pf.tmN[0], pf.Nhi, cap, c.dim), pf_make_map(&pf.tmN[1], pf.Nlo, cap, c.dim);
	pf_make_map(&pf.tmA[0], pf.Ahi, cap, g.q_dim), pf_make_map(&pf.tmA[1], pf.Alo, cap, g.q_dim);
	pf_make_map(&pf.tmH[0], pf.Hhi, cap, c.hidden_dim), pf_make_map(&pf.tmH[1], pf.Hlo, cap, c.hidden_dim);
}

// which models the tensor-core pass serves; everything else is fed token by token (still on the GPU)
static bool pf_supported() {
	const Config& c = g.cfg;
	return c.n_experts == 0 && g.tp_world == 1 && c.dim % PF_BM == 0 && g.q_dim % PF_BM == 0 && g.kv_dim % PF_BM == 0 && c.hidden_dim % PF_BM == 0 &&
	       (c.head_dim == 64 || c.head_dim == 128);
}

template <int MODE, int DBITS, typename KVT>
static void pf_gemm(const CUtensorMap* tm, const PfGemmArgs& a, int rows, int n) {
	smem_optin(k_pf_gemm<MODE, DBITS, KVT>, pf_smem_bytes<MODE>());
	launch_pdl(k_pf_gemm<MODE, DBITS, KVT>, dim3(rows / PF_BM, cdiv(n, PF_BN)), PF_THREADS, pf_smem_bytes<MODE>(), tm[0], tm[1], a);
}

template <typename KVT, int HD, bool SEG, bool CTX = false>
static void pf_attn(const PfAttnArgs& a, int n) {
	const dim3 grid(cdiv(n, PFA_WARPS), g.cfg.n_kv_heads);
	if (g.kv_mul % 4 == 0) launch_pdl(k_pf_attn<KVT, HD, 4, SEG, CTX>, grid, PFA_WARPS * 32, 0, a);
	else if (g.kv_mul % 2 == 0) launch_pdl(k_pf_attn<KVT, HD, 2, SEG, CTX>, grid, PFA_WARPS * 32, 0, a);
	else launch_pdl(k_pf_attn<KVT, HD, 1, SEG, CTX>, grid, PFA_WARPS * 32, 0, a);
}

static_assert(VF_TOK == CALM_B200_VERIFY_MAX, "a short block is one token tile of k_vf_gemm");

static int vf_slices(int K) {
	return cdiv(K, VF_KS);
}

// k_vf_gemm's partial sums, for the largest (K-slices x rows) of the model's GEMMs, and its arrival counters (zeroed once)
static void vf_reserve() {
	if (pf.vacc) return;
	const Config& c = g.cfg;
	const size_t qkv = g.q_dim + 2 * g.kv_dim, cls = (size_t)imin(cdiv(c.vocab_size, PF_BM), VF_CLS_UNITS) * VF_ROWS;
	const size_t rows = std::max({vf_slices(c.dim) * qkv, (size_t)vf_slices(g.q_dim) * c.dim, (size_t)vf_slices(c.dim) * 2 * c.hidden_dim,
	                              (size_t)vf_slices(c.hidden_dim) * c.dim, vf_slices(c.dim) * cls});
	const size_t units = std::max({qkv, (size_t)c.dim, (size_t)c.hidden_dim, cls}) / VF_ROWS;
	pf.vacc_floats = rows * VF_TOK;
	pf.vacc = (float*)dev_alloc(pf.vacc_floats * sizeof(float));
	pf.vcnt = (unsigned*)dev_alloc(units * sizeof(unsigned));
	CUDA_CHECK(cudaMemset(pf.vcnt, 0, units * sizeof(unsigned)));
}

// out = W . X^T over the rows of `a` for the n <= 16 rows of (hi, lo), in `units` row blocks of 128 (UP: of w1 and of w3
// each); the classifier from vocabulary tile `tile0` on; PF_QKV_SLOTS: row t's keys and values to cache slot slot[t].
// Every K-slice gets the same number of CTAs, as many as stay resident together, each walking row blocks with the same
// stride.  PEN: the rows' lanes as k_sq_lanes left them in pf.sqlanes; MASK: also their automaton states, after them.
template <int MODE, int DBITS, typename KVT, bool TOPK = false, bool PEN = false, bool MASK = false>
static void vf_gemm(const __half* hi, const __half* lo, const PfGemmArgs& a, int units, int tile0 = 0, const int* slot = nullptr) {
	static int cap = 0, sms = 0;
	if (sms != g.sms) cap = max_ctas(k_vf_gemm<MODE, DBITS, KVT, TOPK, PEN, MASK>, VF_THREADS, 0), sms = g.sms;
	VfArgs v = {};
	v.xhi = hi, v.xlo = lo, v.acc = pf.vacc, v.cnt = pf.vcnt;
	v.nsl = vf_slices(a.K), v.units = units, v.rows = (MODE == PF_UP ? 2 : 1) * units * VF_ROWS;
	v.tile0 = tile0, v.nvt = cdiv(g.cfg.vocab_size, PF_BM);
	v.logits = pf.vlogits, v.tmax = pf.vtmax, v.slot = slot;
	if constexpr (PEN) v.lane = pf.sqlanes, v.pcnt = pf.sqpcnt, v.pbias = pf.sqpbias, v.ppar = pf.sqppar;
	if constexpr (MASK) v.mstate = pf.sqlanes + SQ_ROWS, v.allow = pf.sqallow;
	const int tasks = (MODE == PF_UP ? 2 : 1) * units;
	launch_pdl(k_vf_gemm<MODE, DBITS, KVT, TOPK, PEN, MASK>, dim3(balanced_grid(tasks, cap / v.nsl > 0 ? cap / v.nsl : 1), v.nsl), VF_THREADS, 0, a, v);
}

// What the rows of a prompt-pass block are
enum PfRows {
	PF_ONE,      // one sequence at cache slots pos0 + t
	PF_SHORT,    // PF_ONE of at most VF_TOK rows (calm_b200_verify_greedy), whose GEMMs run on k_vf_gemm
	PF_SAMPLES,  // a step of calm_b200_decode_sample_n (PfSampleStep): PF_SHORT's GEMMs, per-row RoPE positions from
	             // pf.snpos and the shared-prompt attention of sample_n.cuh
	PF_BATCH,    // a step of calm_b200_decode_sample_batch (PfSampleStep): PF_SAMPLES, but every row continues its own prompt
	             // (pf.sbrows) through sample_n.cuh's BATCH attention
	PF_QUEUE,    // a step of calm_b200_decode_sample_queue (PfSampleStep): PF_BATCH, but every row has its own step count, its
	             // own generated slots and its own RoPE position (the table pf.sqrows), and writes its keys to its own slot
	PF_PACKED,   // a packed block that holds no context (the scoring calls at pos0 = 0, and decode_sample_batch's prompts at
	             // any slot base): per-row RoPE positions in pf.rowpos, each row's sequence start (its cache slot) in pf.seg
	PF_CONTEXTS, // PF_PACKED, and sequences continue contexts placed in the same block: each row's context in pf.ctx
	PF_BEAM,     // a step of calm_b200_decode_beam (PfSampleStep): PF_SAMPLES, but every row reads its generated keys through
	             // its ancestry (sample_n.cuh's BEAM attention)
};

// a short block: at most VF_TOK rows whose GEMMs run on k_vf_gemm
static bool pf_short(PfRows layout) {
	return layout == PF_SHORT || layout == PF_SAMPLES || layout == PF_BATCH || layout == PF_QUEUE || layout == PF_BEAM;
}

// A layer GEMM of the pass over `rows` output rows of `a` (UP: of w1 and of w3 each), whose activations are the f16 pair
// (hi, lo) behind the tensor maps tm: on k_vf_gemm for a short block, on k_pf_gemm for any other
template <int MODE, int DBITS, typename KVT>
static void pf_layer_gemm(PfRows layout, const CUtensorMap* tm, const __half* hi, const __half* lo, const PfGemmArgs& a, int rows) {
	if (pf_short(layout)) vf_gemm<MODE, DBITS, KVT>(hi, lo, a, rows / VF_ROWS);
	else pf_gemm<MODE, DBITS, KVT>(tm, a, rows, a.n_tokens);
}

// A step of calm_b200_decode_sample_n: its n = nseq rows are the sequences, all at RoPE position pos0 + step, row b in
// cache slot pos0 + step * nseq + b; the prompt is in slots [0, pos0).  A step of calm_b200_decode_sample_batch: the
// same slots from pos0 = G, the end of the packed prompts, and row b at RoPE position L_b + step; lmax = max_b L_b.  A
// step of calm_b200_decode_sample_queue: nseq rows, step 0, and lmax = the largest L + j of its rows (pf.sqrows).  A queue
// step whose rows have contexts (pf.sqgroups): nshared shared chunks and nsuf > 0 per-row chunks per row (sample_n.cuh,
// GROUPS); nsuf = 0 on every other step.  A step of calm_b200_decode_beam: nseq rows (1 at step 0) at slots pos0 + step *
// nbeam + b, reading their keys through the ancestry `anc` (sample_n.cuh, BEAM).
struct PfSampleStep {
	int pos0, step, nseq, lmax;
	int nshared = 0, nsuf = 0;
	const int* anc = nullptr;
	int nbeam = 0, anc_stride = 0;
};

// The attention of a PF_SAMPLES step (shared prompt) or, with BATCH, of a PF_BATCH step (a prompt per row), or with
// QUEUE as well, of a PF_QUEUE step (sample_n.cuh), with GROUPS of one whose rows have contexts: chunk partials, then
// their fold into pf.Ahi / pf.Alo
template <typename KVT, int HD, bool BATCH, bool QUEUE = false, bool GROUPS = false, bool BEAM = false>
static void sn_attn(const SnAttnArgs& a, const PfSampleStep& ss) {
	const int nkeys = a.pos0 + a.step + 1, npre = a.pos0 / SN_CHUNK, nsuf = cdiv(nkeys, SN_CHUNK) - npre;
	const dim3 grid(GROUPS ? ss.nshared + a.nseq * ss.nsuf : BATCH ? a.nseq * cdiv(ss.lmax + a.step + 1, SN_CHUNK) : npre + a.nseq * nsuf, g.cfg.n_kv_heads);
	auto run = [&](auto kernel, size_t smem) {
		smem_optin(kernel, smem);
		launch_pdl(kernel, grid, SN_WARPS * 32, smem, a);
	};
	if (g.kv_mul % 4 == 0) run(k_sn_attn<KVT, HD, 4, BATCH, QUEUE, GROUPS, BEAM>, sn_smem_bytes<KVT, HD, 4>());
	else if (g.kv_mul % 2 == 0) run(k_sn_attn<KVT, HD, 2, BATCH, QUEUE, GROUPS, BEAM>, sn_smem_bytes<KVT, HD, 2>());
	else run(k_sn_attn<KVT, HD, 1, BATCH, QUEUE, GROUPS, BEAM>, sn_smem_bytes<KVT, HD, 1>());
	launch_pdl(k_sn_fold<HD, BATCH, QUEUE>, dim3(cdiv(g.cfg.n_heads, SN_WARPS), a.nseq), SN_WARPS * 32, 0, a);
}

// The pass over the n rows in pf.tokens at cache slots pos0 + t, laid out as `layout` says (PF_SAMPLES and PF_BATCH: the
// step `ss`, whose slot base pos0 is ss->pos0 + ss->step * n; PF_QUEUE: the step `ss`, each row at its own slot).
template <int DBITS, typename KVT>
static void pf_run(Formats<DBITS, KVT>, int n, int pos0, PfRows layout, const PfSampleStep* ss = nullptr) {
	const bool packed = layout == PF_PACKED || layout == PF_CONTEXTS;
	const Config& c = g.cfg;
	const Weights& w = g.w;
	const size_t kv_layer = (size_t)c.n_kv_heads * c.seq_len * c.head_dim;
	launch_pdl(k_pf_embed<DBITS>, n, 256, 0, pf.X, (const void*)w.token_embedding_table, (const int*)pf.tokens, n, c.dim);
	if (layout == PF_SAMPLES || layout == PF_BATCH || layout == PF_BEAM) launch_pdl(k_pf_rope_rows, cdiv(n * (c.head_dim / 2), 256), 256, 0, pf.rope, (const float*)g.rope_freq, (const int*)pf.snpos + (size_t)ss->step * n, n, c.head_dim / 2);
	else if (layout == PF_QUEUE) launch_pdl(k_pf_rope_rows, cdiv(n * (c.head_dim / 2), 256), 256, 0, pf.rope, (const float*)g.rope_freq, (const int*)pf.sqrows->pos, n, c.head_dim / 2);
	else if (packed) launch_pdl(k_pf_rope_rows, cdiv(n * (c.head_dim / 2), 256), 256, 0, pf.rope, (const float*)g.rope_freq, (const int*)pf.rowpos, n, c.head_dim / 2);
	else launch_pdl(k_pf_rope, cdiv(n * (c.head_dim / 2), 256), 256, 0, pf.rope, (const float*)g.rope_freq, n, c.head_dim / 2, pos0);
	for (int l = 0; l < c.n_layers; ++l) {
		launch_pdl(k_pf_norm, n, 256, 0, (const float*)pf.X, (const float*)w.rms_att_weight[l], pf.Nhi, pf.Nlo, n, c.dim, c.norm_eps, (int)c.norm_ln);
		PfGemmArgs a = {};
		a.n_tokens = n;
		a.w[0] = w.wq[l], a.w[1] = w.wk[l], a.w[2] = w.wv[l], a.K = c.dim;
		a.Q = pf.Q, a.q_dim = g.q_dim, a.kv_dim = g.kv_dim, a.head_dim = c.head_dim, a.seq_len = c.seq_len, a.pos0 = pos0;
		a.bias = w.bqkv[l], a.clip = c.qkv_clip, a.rope = pf.rope;
		a.kc = (KVT*)g.kc + l * kv_layer, a.vc = (KVT*)g.vc + l * kv_layer;
		if (layout == PF_QUEUE) {
			vf_gemm<PF_QKV_SLOTS, DBITS, KVT>(pf.Nhi, pf.Nlo, a, (g.q_dim + 2 * g.kv_dim) / VF_ROWS, 0, pf.sqrows->slot);
		} else pf_layer_gemm<PF_QKV, DBITS, KVT>(layout, pf.tmN, pf.Nhi, pf.Nlo, a, g.q_dim + 2 * g.kv_dim);

		PfAttnArgs aa = {};
		aa.Q = pf.Q, aa.kc = a.kc, aa.vc = a.vc, aa.Ohi = pf.Ahi, aa.Olo = pf.Alo;
		aa.n_tokens = n, aa.pos0 = pos0, aa.seq_len = c.seq_len, aa.q_dim = g.q_dim, aa.kv_mul = g.kv_mul, aa.inv_sqrt_hd = 1.0f / sqrtf((float)c.head_dim);
		aa.seg = pf.seg, aa.ctx = pf.ctx;
		if (layout == PF_SAMPLES || layout == PF_BATCH || layout == PF_QUEUE || layout == PF_BEAM) {
			SnAttnArgs sa = {};
			sa.Q = pf.Q, sa.kc = a.kc, sa.vc = a.vc, sa.part = pf.snpart, sa.Ohi = pf.Ahi, sa.Olo = pf.Alo;
			sa.pos0 = ss->pos0, sa.step = ss->step, sa.nseq = ss->nseq, sa.seq_len = c.seq_len, sa.q_dim = g.q_dim, sa.kv_mul = g.kv_mul;
			sa.n_heads = c.n_heads, sa.nchmax = pf.snchunks, sa.inv_sqrt_hd = aa.inv_sqrt_hd, sa.rows = pf.sbrows;
			if (layout == PF_QUEUE && ss->nsuf) {
				sa.qrows = pf.sqrows->q, sa.groups = pf.sqgroups;
				if (c.head_dim == 128) sn_attn<KVT, 128, true, true, true>(sa, *ss);
				else sn_attn<KVT, 64, true, true, true>(sa, *ss);
			} else if (layout == PF_QUEUE) {
				sa.qrows = pf.sqrows->q;
				if (c.head_dim == 128) sn_attn<KVT, 128, true, true>(sa, *ss);
				else sn_attn<KVT, 64, true, true>(sa, *ss);
			} else if (layout == PF_BEAM) {
				sa.anc = ss->anc, sa.nbeam = ss->nbeam, sa.anc_stride = ss->anc_stride;
				if (c.head_dim == 128) sn_attn<KVT, 128, false, false, false, true>(sa, *ss);
				else sn_attn<KVT, 64, false, false, false, true>(sa, *ss);
			} else if (layout == PF_BATCH) {
				if (c.head_dim == 128) sn_attn<KVT, 128, true>(sa, *ss);
				else sn_attn<KVT, 64, true>(sa, *ss);
			} else {
				if (c.head_dim == 128) sn_attn<KVT, 128, false>(sa, *ss);
				else sn_attn<KVT, 64, false>(sa, *ss);
			}
		} else if (layout == PF_CONTEXTS) {
			if (c.head_dim == 128) pf_attn<KVT, 128, true, true>(aa, n);
			else pf_attn<KVT, 64, true, true>(aa, n);
		} else if (packed) {
			if (c.head_dim == 128) pf_attn<KVT, 128, true>(aa, n);
			else pf_attn<KVT, 64, true>(aa, n);
		} else {
			if (c.head_dim == 128) pf_attn<KVT, 128, false>(aa, n);
			else pf_attn<KVT, 64, false>(aa, n);
		}

		PfGemmArgs b = {};
		b.n_tokens = n, b.w[0] = w.wo[l], b.K = g.q_dim, b.X = pf.X, b.dim = c.dim;
		pf_layer_gemm<PF_WO, DBITS, KVT>(layout, pf.tmA, pf.Ahi, pf.Alo, b, c.dim);

		if (!c.norm_par) { // (parallel-norm models reuse the attention-norm output, reference infer.c:417-420)
			launch_pdl(k_pf_norm, n, 256, 0, (const float*)pf.X, (const float*)w.rms_ffn_weight[l], pf.Nhi, pf.Nlo, n, c.dim, c.norm_eps, (int)c.norm_ln);
		}
		PfGemmArgs u = {};
		u.n_tokens = n, u.w[0] = w.w1[l], u.w[1] = w.w3[l], u.K = c.dim, u.Hhi = pf.Hhi, u.Hlo = pf.Hlo, u.hidden = c.hidden_dim, u.gelu = c.act_gelu;
		pf_layer_gemm<PF_UP, DBITS, KVT>(layout, pf.tmN, pf.Nhi, pf.Nlo, u, c.hidden_dim);

		PfGemmArgs d = {};
		d.n_tokens = n, d.w[0] = w.w2[l], d.K = c.hidden_dim, d.X = pf.X, d.dim = c.dim;
		pf_layer_gemm<PF_DOWN, DBITS, KVT>(layout, pf.tmH, pf.Hhi, pf.Hlo, d, c.dim);
	}
}

// What a scoring call writes for each scored position: logprobs[i], with `greedy` its argmax, with k > 0 its k largest
// logits' indices and log-probabilities (top_ids / top_logprobs[i * k + r]).  Pointers are at the slot of position 0.
struct PfOut {
	float* logprobs = nullptr;
	int* greedy = nullptr;
	int k = 0;
	int* top_ids = nullptr;
	float* top_logprobs = nullptr;
	// the same outputs from slot `i` on
	PfOut at(size_t i) const {
		PfOut o = *this;
		if (logprobs) o.logprobs += i;
		if (greedy) o.greedy += i;
		if (k) o.top_ids += i * k, o.top_logprobs += i * k;
		return o;
	}
	// rows [s, s + m) of `src`, which holds the same outputs, to slots o .. o + m - 1: from the device on the stream, or
	// from the host
	void put(const PfOut& src, size_t s, size_t m, size_t o, bool from_device) const {
		auto cp = [&](void* dst, const void* from, size_t bytes) {
			if (from_device) CUDA_CHECK(cudaMemcpyAsync(dst, from, bytes, cudaMemcpyDeviceToHost, g.stream));
			else memcpy(dst, from, bytes);
		};
		cp(logprobs + o, src.logprobs + s, m * sizeof(float));
		if (greedy) cp(greedy + o, src.greedy + s, m * sizeof(int));
		if (k) cp(top_ids + o * k, src.top_ids + s * k, m * k * sizeof(int)), cp(top_logprobs + o * k, src.top_logprobs + s * k, m * k * sizeof(float));
	}
};

// Host rows for the outputs of `x`, where a block's or a lone pass's rows land before they go to the caller's slots
struct PfRowBuf {
	std::vector<float> lp, tl;
	std::vector<int> gr, ti;
	PfOut out; // x's outputs, in these rows
	PfRowBuf(const PfOut& x, size_t rows) : lp(rows), tl(rows * x.k), gr(x.greedy ? rows : 0), ti(rows * x.k), out(x) {
		out.logprobs = lp.data(), out.greedy = x.greedy ? gr.data() : nullptr, out.top_ids = ti.data(), out.top_logprobs = tl.data();
	}
	PfRowBuf(const PfRowBuf&) = delete;
};

// The scoring buffers for pf.cap rows, with `greedy` the argmax buffers and with `topk` the top-k buffers, which the
// plain scoring calls never allocate (freed and re-made with the pass's own buffers when a longer block needs more rows)
static void pf_score_reserve(bool greedy, bool topk) {
	const int nvt = cdiv(g.cfg.vocab_size, PF_BM);
	if (!pf.scoring) {
		pf.part = (float2*)dev_alloc((size_t)pf.cap * nvt * sizeof(float2));
		pf.tgt = (float*)dev_alloc((size_t)pf.cap * sizeof(float));
		pf.logprob = (float*)dev_alloc((size_t)pf.cap * sizeof(float));
		pf.targets = (int*)dev_alloc((size_t)pf.cap * sizeof(int));
		pf.scoring = true;
	}
	if (greedy && !pf.gidx) {
		pf.gidx = (int*)dev_alloc((size_t)pf.cap * nvt * sizeof(int));
		pf.greedy = (int*)dev_alloc((size_t)pf.cap * sizeof(int));
	}
	if (topk && !pf.topv) { // sized for the largest k: at Llama-3-8B's vocabulary, 2048 rows take 328 MB of tile lists
		pf.topv = (float*)dev_alloc((size_t)pf.cap * nvt * PF_TOPK_MAX * sizeof(float));
		pf.topi = (int*)dev_alloc((size_t)pf.cap * nvt * PF_TOPK_MAX * sizeof(int));
		pf.top_ids = (int*)dev_alloc((size_t)pf.cap * PF_TOPK_MAX * sizeof(int));
		pf.top_lp = (float*)dev_alloc((size_t)pf.cap * PF_TOPK_MAX * sizeof(float));
	}
}

// The merge of the classifier's tile records into each row's log-probability (pf.logprob), with `greedy` its argmax
// (pf.greedy), with k > 0 its k largest logits (pf.top_ids / pf.top_lp)
static void pf_merge(int n, bool greedy, int k) {
	const int nvt = cdiv(g.cfg.vocab_size, PF_BM);
	const auto merge = k ? k_pf_logprob<false, true> : greedy ? k_pf_logprob<true> : k_pf_logprob<false>;
	launch_pdl(merge, cdiv(n, 8), 256, k ? (size_t)8 * nvt : 0, (const float2*)pf.part, (const float*)pf.tgt, pf.logprob, n, nvt, (const int*)pf.gidx,
	           pf.greedy, (const float*)pf.topv, (const int*)pf.topi, k, pf.top_ids, pf.top_lp);
}

// After pf_run over n rows: the final norm, the classifier with its log-softmax epilogue, the merge of the tile records;
// with `greedy` the classifier and the merge also give each row's argmax in pf.greedy, with k > 0 its k largest logits'
// indices and log-probabilities in pf.top_ids / pf.top_lp [n][k].  A short block's greedy classifier runs on k_vf_gemm,
// VF_CLS_UNITS vocabulary tiles per launch; with `sample` (a short greedy block) it also writes the logit rows and tile
// maxima that vf_sample_rows samples, and the merge is left out.
template <int DBITS, typename KVT>
static void pf_score(Formats<DBITS, KVT>, int n, PfRows layout, bool greedy, int k, bool sample = false) {
	const Config& c = g.cfg;
	const Weights& w = g.w;
	const int nvt = cdiv(c.vocab_size, PF_BM);
	launch_pdl(k_pf_norm, n, 256, 0, (const float*)pf.X, (const float*)w.rms_final_weight, pf.Nhi, pf.Nlo, n, c.dim, c.norm_eps, (int)c.norm_ln);
	PfGemmArgs a = {};
	a.n_tokens = n, a.w[0] = w.wcls, a.K = c.dim;
	a.targets = pf.targets, a.part = pf.part, a.tgt = pf.tgt, a.vocab = c.vocab_size, a.gidx = pf.gidx;
	if (k) {
		a.topv = pf.topv, a.topi = pf.topi, a.topk = k;
		pf_gemm<PF_CLS_TOPK, DBITS, KVT>(pf.tmN, a, nvt * PF_BM, n);
	} else if (greedy && pf_short(layout)) {
		for (int t0 = 0; t0 < nvt; t0 += VF_CLS_UNITS) {
			if (sample) vf_gemm<PF_CLS_SAMPLE, DBITS, KVT>(pf.Nhi, pf.Nlo, a, imin(VF_CLS_UNITS, nvt - t0), t0);
			else vf_gemm<PF_CLS_GREEDY, DBITS, KVT>(pf.Nhi, pf.Nlo, a, imin(VF_CLS_UNITS, nvt - t0), t0);
		}
		if (sample) return;
	} else if (greedy) {
		pf_gemm<PF_CLS_GREEDY, DBITS, KVT>(pf.tmN, a, nvt * PF_BM, n);
	} else {
		pf_gemm<PF_CLS, DBITS, KVT>(pf.tmN, a, nvt * PF_BM, n);
	}
	pf_merge(n, greedy, k);
}

// One block of the pass: the n rows the caller reserved (pf_reserve) and uploaded to pf.tokens (and, packed, to pf.rowpos,
// pf.seg and pf.ctx) at cache slots pos0 + t, laid out as `layout` says.  With `x.logprobs`, the rows are scored against
// targets[0 .. n) as well, and `x` gets the outputs of row t at slot t.
static void pf_block(int n, int pos0, PfRows layout, const int* targets, const PfOut& x) {
	if (x.logprobs) {
		pf_score_reserve(x.greedy, x.k > 0);
		CUDA_CHECK(cudaMemcpyAsync(pf.targets, targets, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	}
	with_formats([&](auto f) { pf_run(f, n, pos0, layout); });
	if (x.logprobs) {
		with_formats([&](auto f) { pf_score(f, n, layout, x.greedy, x.k); });
		PfOut dev = x;
		dev.logprobs = pf.logprob, dev.greedy = pf.greedy, dev.top_ids = pf.top_ids, dev.top_logprobs = pf.top_lp;
		x.put(dev, 0, n, 0, true);
	}
	CUDA_CHECK(cudaStreamSynchronize(g.stream)); // the uploads read the caller's memory (pageable): they must have left it
	CUDA_CHECK(cudaGetLastError());
}

// The batched pass over tokens[0 .. n) at positions pos0 .., in blocks of at most 2048 rows.  With `x.logprobs`, every
// block is scored as well: logprobs[i] = ln softmax(logits after tokens[i])[tokens[i + 1]], so tokens[n] must exist, and
// `x` gets the outputs of position i at its slot i.
static void pf_pass(const int* tokens, int n, int pos0, const PfOut& x = PfOut()) {
	const int chunk_cap = 2048;
	for (int o = 0; o < n; o += chunk_cap) {
		const int m = n - o < chunk_cap ? n - o : chunk_cap;
		pf_reserve(m);
		CUDA_CHECK(cudaMemcpyAsync(pf.tokens, tokens + o, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		pf_block(m, pos0 + o, PF_ONE, tokens + o + 1, x.at(o));
	}
}

static void check_tokens(const int* tokens, int n) {
	for (int i = 0; i < n; ++i)
		if (tokens[i] < 0 || tokens[i] >= g.cfg.vocab_size) CALM_FATAL("token %d out of range", tokens[i]);
}

// Feed `n` prompt tokens at positions pos0 .. pos0 + n - 1: the KV cache afterwards is what n calls of
// forward_cuda(token, pos, FF_UPDATE_KV_ONLY) leave (within the stated tolerance); no logits, no synchronisation.
// Returns 1 when the tensor-core pass ran, 0 when the tokens were fed one by one (unsupported model shape, MoE, tensor
// parallelism, or a block that would roll the cache over).
extern "C" int forward_prefill_cuda(struct Transformer* transformer, const int* tokens, int n, int pos0) {
	if (n <= 0) return 1;
	check_call(transformer, tokens[0], pos0);
	check_tokens(tokens, n);
	if (!pf_supported() || pos0 + n > g.cfg.seq_len) {
		for (int i = 0; i < n; ++i) {
			set_params(tokens[i], pos0 + i, 0);
			launch_token(0);
		}
		return 0;
	}
	pf_pass(tokens, n, pos0);
	return 1;
}

// The decode path's log-softmax of one logit row l[0 .. vocab), in double: *logprob = l[target] - M - ln S, and with k > 0
// the k largest logits, equal logits by index ascending (the same order as the tensor-core pass), and theirs
static void host_logprobs(const float* l, int vocab, int target, int k, float* logprob, int* top_ids, float* top_logprobs) {
	double mx = l[0], s = 0.0;
	for (int v = 1; v < vocab; ++v) mx = l[v] > mx ? l[v] : mx;
	for (int v = 0; v < vocab; ++v) s += exp((double)l[v] - mx);
	*logprob = (float)((double)l[target] - mx - log(s));
	if (k) {
		std::vector<int> idx(vocab);
		for (int v = 0; v < vocab; ++v) idx[v] = v;
		std::partial_sort(idx.begin(), idx.begin() + k, idx.end(), [l](int a, int b) { return l[a] > l[b] || (l[a] == l[b] && a < b); });
		for (int r = 0; r < k; ++r) top_ids[r] = idx[r], top_logprobs[r] = (float)((double)l[idx[r]] - mx - log(s));
	}
}

// Score tokens[1 .. n) given what precedes each (the reference's study(), run.c:291-308): tokens[0 .. n - 1) go through
// the prompt pass and logprobs[i] = ln softmax(logits after tokens[i])[tokens[i + 1]].  The cache is left as
// forward_prefill_cuda(tokens, n - 1, pos0) leaves it.  Shapes the pass does not serve go one position at a time through
// the decode path with a log-softmax in double on the host (returns 0).
// calm_b200_score, and with the extra outputs of `x` its greedy and top-k siblings
static int pf_score_one(struct Transformer* transformer, const int* tokens, int n, int pos0, const PfOut& x) {
	if (n < 2) return 1;
	check_call(transformer, tokens[0], pos0);
	check_tokens(tokens, n);
	const int rows = n - 1, vocab = g.cfg.vocab_size;
	if (!pf_supported() || pos0 + rows > g.cfg.seq_len) {
		for (int i = 0; i < rows; ++i) {
			set_params(tokens[i], pos0 + i, 0);
			launch_token(1);
			sync_stream();
			const float* l = g.logits_host;
			host_logprobs(l, vocab, tokens[i + 1], x.k, &x.logprobs[i], x.top_ids + (size_t)i * x.k, x.top_logprobs + (size_t)i * x.k);
			if (x.greedy) { // first maximum (sampler.c:34-42), as calm_b200_forward_argmax
				int best = 0;
				for (int v = 1; v < vocab; ++v)
					if (l[v] > l[best]) best = v;
				x.greedy[i] = best;
			}
		}
		CUDA_CHECK(cudaGetLastError());
		return 0;
	}
	pf_pass(tokens, rows, pos0, x);
	return 1;
}

// The outputs of a greedy call `who`, checked before any device work
static PfOut greedy_out(const char* who, float* logprobs, int* greedy) {
	if (!greedy) CALM_FATAL("%s: greedy is NULL", who);
	return PfOut{logprobs, greedy};
}

// The outputs of a top-k call `who`, checked before any device work
static PfOut topk_out(const char* who, int k, float* logprobs, int* top_ids, float* top_logprobs) {
	if (!g.ready) CALM_FATAL("%s before prepare_cuda", who);
	const int kmax = imin(CALM_B200_TOPK_MAX, g.cfg.vocab_size);
	if (k < 1 || k > kmax) CALM_FATAL("%s: k %d outside [1, %d]", who, k, kmax);
	if (!top_ids || !top_logprobs) CALM_FATAL("%s: top_ids or top_logprobs is NULL", who);
	return PfOut{logprobs, nullptr, k, top_ids, top_logprobs};
}

extern "C" int calm_b200_score(struct Transformer* transformer, const int* tokens, int n, int pos0, float* logprobs) {
	return pf_score_one(transformer, tokens, n, pos0, PfOut{logprobs});
}

extern "C" int calm_b200_score_greedy(struct Transformer* transformer, const int* tokens, int n, int pos0, float* logprobs, int* greedy) {
	return pf_score_one(transformer, tokens, n, pos0, greedy_out("score_greedy", logprobs, greedy));
}

extern "C" int calm_b200_score_topk(struct Transformer* transformer, const int* tokens, int n, int pos0, int k, float* logprobs, int* top_ids,
                                    float* top_logprobs) {
	return pf_score_one(transformer, tokens, n, pos0, topk_out("score_topk", k, logprobs, top_ids, top_logprobs));
}

// A packed block being filled: per-row inputs, the sequences it scores with their first rows, and the contexts it holds
// by (ctx_off, ctx_len) with their first rows.  Row t of the block is cache slot t.
struct PfPackedBlock {
	std::vector<int> tok, tgt, pos, seg;
	std::vector<int2> ctx;
	std::vector<std::pair<int, int>> seqs;
	std::map<std::pair<int, int>, int> placed;
	int rows() const { return (int)tok.size(); }
	// Rows for the r inputs t[0 .. r) at RoPE positions p0 .., continuing context cx, rounded up to a multiple of 8 with
	// filler rows that repeat the last input, so that a k_pf_attn CTA never straddles two sequences; row j targets
	// t[min(j + 1, tl)].  Causal attention keeps filler rows out of every live row.  Returns the first row.
	int add(const int* t, int r, int tl, int p0, int2 cx) {
		const int s = rows();
		for (int j = 0; j < cdiv(r, 8) * 8; ++j)
			tok.push_back(t[imin(j, r - 1)]), tgt.push_back(t[imin(j + 1, tl)]), pos.push_back(p0 + j), seg.push_back(s), ctx.push_back(cx);
		return s;
	}
};

// Run a block and write its sequences' log-probabilities; the results of context and filler rows are dropped.  A block that
// holds no context runs the packed attention (k_pf_attn<.., SEG>); only one with a context uploads pf.ctx and runs the
// context walk (k_pf_attn<.., SEG, CTX>).
static void pf_score_packed_block(PfPackedBlock& b, const int* off, const int* len, const PfOut& x) {
	const int rows = b.rows();
	const bool contexts = !b.placed.empty();
	const PfRowBuf buf(x, rows);
	pf_reserve(rows);
	CUDA_CHECK(cudaMemcpyAsync(pf.tokens, b.tok.data(), (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaMemcpyAsync(pf.rowpos, b.pos.data(), (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaMemcpyAsync(pf.seg, b.seg.data(), (size_t)rows * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	if (contexts) CUDA_CHECK(cudaMemcpyAsync(pf.ctx, b.ctx.data(), (size_t)rows * sizeof(int2), cudaMemcpyHostToDevice, g.stream));
	pf_block(rows, 0, contexts ? PF_CONTEXTS : PF_PACKED, b.tgt.data(), buf.out);
	for (const auto& [i, s] : b.seqs) x.put(buf.out, s, len[i] - 1, off[i], false);
	b = PfPackedBlock();
}

// Score nseq sequences that continue contexts (include/calm_b200.h); `who` names the call in error messages.  Next-fit
// packing in input order into blocks of at most C = min(2048, seq_len rounded down to 8) rows: a context takes
// ceil8(ctx_len) rows at RoPE positions 0 ..; a sequence takes ceil8(len - 1) rows at positions ctx_len .., after its
// context's rows in the same block.  Sequences with the same (ctx_off, ctx_len) share one placement of the context per
// block; a sequence whose context is not yet in the block brings it along.  A context and sequence too long for any block,
// together, are scored alone by calm_b200_score.  With every ctx_len 0 no block holds a context: calm_b200_score_batch.
// With the extra outputs of `x`, the greedy and top-k calls.
static int pf_score_packed(const char* who, struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                           const int* off, const int* len, int nseq, const PfOut& x) {
	if (!g.ready) CALM_FATAL("%s before prepare_cuda", who);
	if (n < 0 || nseq < 0) CALM_FATAL("%s: negative count (n %d, nseq %d)", who, n, nseq);
	if (nseq == 0) return 1;
	check_tokens(tokens, n);
	std::vector<std::pair<long, long>> out; // [first, last + 1) of the logprobs each sequence writes
	for (int i = 0; i < nseq; ++i) {
		if (off[i] < 0 || len[i] < 0 || (long)off[i] + len[i] > n) CALM_FATAL("%s: sequence %d (off %d, len %d) outside the %d tokens", who, i, off[i], len[i], n);
		if (ctx_off[i] < 0 || ctx_len[i] < 0 || (long)ctx_off[i] + ctx_len[i] > n)
			CALM_FATAL("%s: context of sequence %d (off %d, len %d) outside the %d tokens", who, i, ctx_off[i], ctx_len[i], n);
		if (len[i] >= 2) out.push_back({off[i], (long)off[i] + len[i] - 1});
	}
	std::sort(out.begin(), out.end());
	for (size_t k = 1; k < out.size(); ++k)
		if (out[k].first < out[k - 1].second) CALM_FATAL("%s: output ranges [%ld, %ld) and [%ld, %ld) overlap", who, out[k - 1].first, out[k - 1].second, out[k].first, out[k].second);
	// calm_b200_score of ctx ++ sequence, by definition the result: for shapes the pass does not serve and units too big
	auto alone = [&](int i) {
		std::vector<int> cat(tokens + ctx_off[i], tokens + ctx_off[i] + ctx_len[i]);
		cat.insert(cat.end(), tokens + off[i], tokens + off[i] + len[i]);
		const PfRowBuf buf(x, cat.size() - 1); // the rows of ctx ++ sequence
		const int served = pf_score_one(transformer, cat.data(), (int)cat.size(), 0, buf.out);
		x.put(buf.out, ctx_len[i], len[i] - 1, off[i], false);
		return served;
	};
	if (!pf_supported()) {
		for (int i = 0; i < nseq; ++i)
			if (len[i] >= 2) alone(i);
		return 0;
	}
	const int cap = imin(2048, g.cfg.seq_len / 8 * 8); // a row is its cache slot: no row may reach seq_len
	PfPackedBlock b;
	std::vector<int> big;
	for (int i = 0; i < nseq; ++i) {
		if (len[i] < 2) continue;
		const int R = cdiv(len[i] - 1, 8) * 8, Rc = cdiv(ctx_len[i], 8) * 8;
		if (Rc + R > cap) {
			big.push_back(i);
			continue;
		}
		const std::pair<int, int> key(ctx_off[i], ctx_len[i]);
		if (b.rows() + (b.placed.count(key) ? 0 : Rc) + R > cap) pf_score_packed_block(b, off, len, x);
		int c0 = 0;
		if (ctx_len[i]) {
			const auto it = b.placed.find(key);
			c0 = it != b.placed.end() ? it->second : (b.placed[key] = b.add(tokens + ctx_off[i], ctx_len[i], ctx_len[i] - 1, 0, make_int2(0, 0)));
		}
		b.seqs.push_back({i, b.add(tokens + off[i], len[i] - 1, len[i] - 1, ctx_len[i], make_int2(c0, ctx_len[i]))});
	}
	if (b.rows()) pf_score_packed_block(b, off, len, x);
	int served = 1;
	for (int i : big) served &= alone(i);
	return served;
}

// calm_b200_score_batch and its greedy and top-k siblings: the context calls with every context empty
static int pf_score_batch(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq, const PfOut& x) {
	const std::vector<int> empty(nseq > 0 ? nseq : 0);
	return pf_score_packed("score_batch", transformer, tokens, n, empty.data(), empty.data(), off, len, nseq, x);
}

extern "C" int calm_b200_score_batch(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq, float* logprobs) {
	return pf_score_batch(transformer, tokens, n, off, len, nseq, PfOut{logprobs});
}

extern "C" int calm_b200_score_batch_greedy(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq,
                                            float* logprobs, int* greedy) {
	return pf_score_batch(transformer, tokens, n, off, len, nseq, greedy_out("score_batch_greedy", logprobs, greedy));
}

extern "C" int calm_b200_score_batch_topk(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq, int k,
                                          float* logprobs, int* top_ids, float* top_logprobs) {
	return pf_score_batch(transformer, tokens, n, off, len, nseq, topk_out("score_batch_topk", k, logprobs, top_ids, top_logprobs));
}

extern "C" int calm_b200_score_context(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                       const int* off, const int* len, int nseq, float* logprobs) {
	return pf_score_packed("score_context", transformer, tokens, n, ctx_off, ctx_len, off, len, nseq, PfOut{logprobs});
}

extern "C" int calm_b200_score_context_greedy(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                              const int* off, const int* len, int nseq, float* logprobs, int* greedy) {
	return pf_score_packed("score_context", transformer, tokens, n, ctx_off, ctx_len, off, len, nseq, greedy_out("score_context_greedy", logprobs, greedy));
}

extern "C" int calm_b200_score_context_topk(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                            const int* off, const int* len, int nseq, int k, float* logprobs, int* top_ids, float* top_logprobs) {
	return pf_score_packed("score_context", transformer, tokens, n, ctx_off, ctx_len, off, len, nseq, topk_out("score_context_topk", k, logprobs, top_ids, top_logprobs));
}

// ---------------------------------------------------------------------------------------------
// calm_b200_verify_greedy: a block of at most CALM_B200_VERIFY_MAX tokens (a decode token and its drafts) through the
// prompt pass as a short block, whose projections and classifier run on the short-block GEMM of verify.cuh.

extern "C" int calm_b200_verify_greedy(struct Transformer* transformer, const int* tokens, int n, int pos0, int* greedy) {
	if (!g.ready) CALM_FATAL("verify_greedy before prepare_cuda");
	if (n < 1 || n > CALM_B200_VERIFY_MAX) CALM_FATAL("verify_greedy: n %d outside [1, %d]", n, CALM_B200_VERIFY_MAX);
	if (!tokens || !greedy) CALM_FATAL("verify_greedy: tokens or greedy is NULL");
	check_call(transformer, tokens[0], pos0);
	check_tokens(tokens, n);
	if (!pf_supported() || pos0 + n > g.cfg.seq_len) {
		for (int i = 0; i < n; ++i) greedy[i] = calm_b200_forward_argmax(transformer, tokens[i], pos0 + i);
		return 0;
	}
	pf_reserve(n);
	pf_score_reserve(true, false);
	vf_reserve();
	CUDA_CHECK(cudaMemcpyAsync(pf.tokens, tokens, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	with_formats([&](auto f) {
		pf_run(f, n, pos0, PF_SHORT);
		pf_score(f, n, PF_SHORT, true, 0);
	});
	CUDA_CHECK(cudaMemcpyAsync(greedy, pf.greedy, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
	sync_stream();
	CUDA_CHECK(cudaGetLastError());
	return 1;
}

// ---------------------------------------------------------------------------------------------
// calm_b200_verify_sample: the short block with the classifier in PF_CLS_SAMPLE, whose logit rows the unchanged device
// sampler draws from, one row at a time.

// the logit rows and tile maxima, and each row's sampler lists, sums, counts, state and token (pf.vlogits ..)
static void vf_sample_reserve() {
	if (pf.vlogits) return;
	const size_t vocab = g.cfg.vocab_size, nvt = cdiv(g.cfg.vocab_size, PF_BM), nch = g.sample_chunks;
	pf.vlogits = (float*)dev_alloc(VF_TOK * vocab * sizeof(float));
	pf.vtmax = (float*)dev_alloc(VF_TOK * nvt * sizeof(float));
	pf.vsidx = (int*)dev_alloc(VF_TOK * nch * SAMPLE_CHUNK * sizeof(int));
	pf.vsprob = (float*)dev_alloc(VF_TOK * nch * SAMPLE_CHUNK * sizeof(float));
	pf.vcsum = (float*)dev_alloc(VF_TOK * nch * sizeof(float));
	pf.vcount = (int*)dev_alloc(VF_TOK * nch * sizeof(int));
	pf.vstate = (SampleState*)dev_alloc(VF_TOK * sizeof(SampleState));
	pf.vsampled = (int*)dev_alloc(VF_TOK * sizeof(int));
}

// The n rows of the last PF_CLS_SAMPLE classifier through the decode's sampler, side by side: row i is k_sample_scan +
// k_sample_pick on its own lists and its own SampleState pf.vstate[i] (k_sample_scan_rows / k_sample_pick_rows), and its
// token goes to out[i] (default pf.vsampled[i]).  `masked`: k_sample_scan_rows_masked, where -inf never survives.
// `trunc` (calm_b200_decode_sample_queue_truncated): its ntrunc rows first go through k_sample_trunc_rows, which writes
// -inf over their dropped entries, and the scan is the masked one.
static void vf_sample_rows(int n, int* out = nullptr, bool masked = false, const TruncRows* trunc = nullptr, int ntrunc = 0) {
	const int vocab = g.cfg.vocab_size, nvt = cdiv(vocab, PF_BM), nch = g.sample_chunks;
	SampleArgs sa;
	sa.logits = pf.vlogits, sa.cand_val = pf.vtmax, sa.ncand = nvt, sa.vocab = vocab, sa.nchunks = nch;
	sa.st = pf.vstate, sa.count = pf.vcount, sa.csum = pf.vcsum, sa.sidx = pf.vsidx, sa.sprob = pf.vsprob;
	if (trunc) trunc_launch(dim3(TRUNC_CTAS, ntrunc), g.stream, sa, *trunc, vocab), masked = true;
	if (masked) launch_pdl(k_sample_scan_rows_masked, dim3(nch, n), 256, 0, sa);
	else launch_pdl(k_sample_scan_rows, dim3(nch, n), 256, 0, sa);
	launch_pdl(k_sample_pick_rows, n, 256, 0, sa, pf.vstate, out ? out : pf.vsampled);
}

extern "C" int calm_b200_verify_sample(struct Transformer* transformer, const int* tokens, int n, int pos0, float temperature, float minp,
                                       unsigned long long* rng_state, int* sampled) {
	if (!g.ready) CALM_FATAL("verify_sample before prepare_cuda");
	if (n < 1 || n > CALM_B200_VERIFY_MAX) CALM_FATAL("verify_sample: n %d outside [1, %d]", n, CALM_B200_VERIFY_MAX);
	if (!tokens || !sampled || !rng_state) CALM_FATAL("verify_sample: tokens, rng_state or sampled is NULL");
	if (temperature == 0.0f || minp >= 1.0f) return calm_b200_verify_greedy(transformer, tokens, n, pos0, sampled); // sample() is greedy there
	check_call(transformer, tokens[0], pos0);
	check_tokens(tokens, n);
	int served = 0;
	if (!pf_supported() || pos0 + n > g.cfg.seq_len) {
		unsigned long long s = *rng_state; // a local copy: the caller's generator advances by the draws it keeps
		for (int i = 0; i < n; ++i) sampled[i] = calm_b200_forward_sample(transformer, tokens[i], pos0 + i, temperature, minp, &s);
	} else {
		pf_reserve(n);
		pf_score_reserve(true, false);
		vf_reserve();
		vf_sample_reserve();
		SampleState st[CALM_B200_VERIFY_MAX]; // row i draws the (i + 1)-th coin: the caller's state advanced i times
		unsigned long long s = *rng_state;
		for (int i = 0; i < n; ++i) st[i].rng = s, st[i].temperature = temperature, st[i].cut_delta = logf(minp) * temperature, s = xorshift_step(s);
		CUDA_CHECK(cudaMemcpyAsync(pf.tokens, tokens, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		CUDA_CHECK(cudaMemcpyAsync(pf.vstate, st, (size_t)n * sizeof(SampleState), cudaMemcpyHostToDevice, g.stream));
		with_formats([&](auto f) {
			pf_run(f, n, pos0, PF_SHORT);
			pf_score(f, n, PF_SHORT, true, 0, true);
		});
		vf_sample_rows(n);
		CUDA_CHECK(cudaMemcpyAsync(sampled, pf.vsampled, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
		sync_stream();
		CUDA_CHECK(cudaGetLastError());
		pf.vrows = n;
		served = 1;
	}
	int acc = 0; // accepted drafts: the caller emits sampled[0 .. acc], one draw each
	while (acc < n - 1 && sampled[acc] == tokens[acc + 1]) ++acc;
	for (int i = 0; i <= acc; ++i) *rng_state = xorshift_step(*rng_state);
	return served;
}

// The draft for `seq`: the key is its last gl tokens, for gl = 3, 2, 1 in turn, and the draft is the tokens that follow the
// key's rightmost occurrence in the corpus among those some token follows, at most `cap` of them.  The corpus is `source`,
// or with source == NULL `seq` itself, whose own final occurrence of the key is then passed over since nothing follows it.
static int vf_lookup(const std::vector<int>& seq, const int* source, int n_source, int cap, int* draft) {
	const int* corpus = source ? source : seq.data();
	const int nc = source ? n_source : (int)seq.size();
	for (int gl = 3; gl >= 1; --gl) {
		if ((int)seq.size() < gl) continue;
		const int* key = seq.data() + seq.size() - gl;
		for (int i = nc - gl - 1; i >= 0; --i)
			if (std::equal(key, key + gl, corpus + i)) {
				const int d = imin(cap, nc - i - gl);
				std::copy(corpus + i + gl, corpus + i + gl + d, draft);
				return d;
			}
	}
	return 0;
}

// The argument checks of the lookup calls (`who`), before any device work
static void lookup_checks(const char* who, const int* tokens, int n, int n_tokens, const int* source, int n_source, int max_draft, const int* out_tokens) {
	if (!g.ready) CALM_FATAL("%s before prepare_cuda", who);
	if (!tokens || n < 1) CALM_FATAL("%s: needs at least one token (n = %d)", who, n);
	if (n_tokens < 0 || (n_tokens > 0 && !out_tokens)) CALM_FATAL("%s: n_tokens %d or out_tokens NULL", who, n_tokens);
	if (max_draft < 1 || max_draft > CALM_B200_VERIFY_MAX - 1) CALM_FATAL("%s: max_draft %d outside [1, %d]", who, max_draft, CALM_B200_VERIFY_MAX - 1);
	if (source && n_source < 0) CALM_FATAL("%s: n_source %d", who, n_source);
}

// The loop of calm_b200_decode_lookup and calm_b200_decode_lookup_sample, after lookup_checks: step(cur, pos) is one
// decode step, which returns the token after `cur`; verify(block, m, pos, out) feeds block[0 .. m) at pos .. and writes
// the token after each to out[0 .. m).  The longest prefix of drafts that out confirms is accepted, and the token after it
// is emitted too.
template <typename Step, typename Verify>
static int lookup_loop(struct Transformer* transformer, const int* tokens, int n, int n_tokens, const int* source, int n_source, int max_draft,
                       int* out_tokens, Step step, Verify verify) {
	check_call(transformer, tokens[n - 1], n - 1);
	check_tokens(tokens, n);
	if (source) check_tokens(source, n_source);
	const bool served = pf_supported();
	std::vector<int> seq(tokens, tokens + n);
	seq.reserve(n + n_tokens);
	int block[CALM_B200_VERIFY_MAX], greedy[CALM_B200_VERIFY_MAX];
	int cur = tokens[n - 1], pos = n - 1, emitted = 0, steps = 0;
	while (emitted < n_tokens) {
		// drafts never run past the tokens still wanted or the end of the cache
		const int cap = served ? imin(imin(max_draft, n_tokens - emitted - 1), g.cfg.seq_len - 1 - pos) : 0;
		const int d = cap > 0 ? vf_lookup(seq, source, n_source, cap, block + 1) : 0;
		++steps;
		if (d == 0) { // no draft: one decode step
			cur = step(cur, pos++);
			out_tokens[emitted++] = cur;
			seq.push_back(cur);
			continue;
		}
		block[0] = cur;
		verify(block, d + 1, pos, greedy);
		int acc = 0; // accepted drafts; greedy[acc] is the correction, or the bonus token after d accepted drafts
		while (acc < d && block[1 + acc] == greedy[acc]) ++acc;
		for (int i = 0; i <= acc; ++i) out_tokens[emitted++] = greedy[i], seq.push_back(greedy[i]);
		cur = greedy[acc], pos += acc + 1;
	}
	return steps;
}

extern "C" int calm_b200_decode_lookup(struct Transformer* transformer, const int* tokens, int n, int n_tokens, const int* source, int n_source,
                                       int max_draft, int* out_tokens) {
	lookup_checks("decode_lookup", tokens, n, n_tokens, source, n_source, max_draft, out_tokens);
	return lookup_loop(
	    transformer, tokens, n, n_tokens, source, n_source, max_draft, out_tokens, [&](int cur, int pos) { return calm_b200_forward_argmax(transformer, cur, pos); },
	    [&](const int* block, int m, int pos, int* out) { calm_b200_verify_greedy(transformer, block, m, pos, out); });
}

// decode_lookup's loop with sampled tokens: a step is calm_b200_forward_sample, a verification calm_b200_verify_sample, and
// both advance the caller's generator by the tokens they emit
extern "C" int calm_b200_decode_lookup_sample(struct Transformer* transformer, const int* tokens, int n, int n_tokens, const int* source, int n_source,
                                              int max_draft, float temperature, float minp, unsigned long long* rng_state, int* out_tokens) {
	lookup_checks("decode_lookup_sample", tokens, n, n_tokens, source, n_source, max_draft, out_tokens);
	if (!rng_state) CALM_FATAL("decode_lookup_sample: rng_state is NULL");
	if (temperature == 0.0f || minp >= 1.0f) return calm_b200_decode_lookup(transformer, tokens, n, n_tokens, source, n_source, max_draft, out_tokens);
	return lookup_loop(
	    transformer, tokens, n, n_tokens, source, n_source, max_draft, out_tokens,
	    [&](int cur, int pos) { return calm_b200_forward_sample(transformer, cur, pos, temperature, minp, rng_state); },
	    [&](const int* block, int m, int pos, int* out) { calm_b200_verify_sample(transformer, block, m, pos, temperature, minp, rng_state, out); });
}

// ---------------------------------------------------------------------------------------------
// calm_b200_decode_sample_n: nseq continuations of one prompt, one short block per step whose rows are the sequences
// (PF_SAMPLES), with the prompt's keys read once per step for all of them (sample_n.cuh).

static_assert(CALM_B200_SAMPLE_N_MAX == VF_TOK, "the sequences of a step are one token tile of k_vf_gemm");

// the pass's buffers for `rows` rows, the short block's and its sampler's, then the chunk partials for `chunks` chunks per
// query (kept when large enough), the positions and the step tokens
static void sn_reserve(int rows, int chunks) {
	const Config& c = g.cfg;
	pf_reserve(rows);
	pf_score_reserve(true, false);
	vf_reserve();
	vf_sample_reserve();
	if (!pf.snpos) {
		pf.snpos = (int*)dev_alloc((size_t)c.seq_len * sizeof(int));
		pf.sntok = (int*)dev_alloc((size_t)c.seq_len * sizeof(int));
	}
	if (chunks <= pf.snchunks) return;
	if (pf.snpart) {
		CUDA_CHECK(cudaStreamSynchronize(g.stream));
		cudaFree(pf.snpart);
	}
	pf.snchunks = chunks;
	pf.snpart = (float*)dev_alloc((size_t)VF_TOK * c.n_heads * chunks * (c.head_dim + 2) * sizeof(float));
}

// The step loop of calm_b200_decode_sample_n and calm_b200_decode_sample_batch: n_tokens short blocks of nseq rows laid
// out as `layout`, step j at slot base s0.pos0 + j * nseq, row b fed tok0[b] at RoPE position p0[b] and then its own
// samples at p0[b] + 1, ...; the sampled tokens go back to the next step on the device, and the tokens and states are
// copied back once at the end.  The caller has reserved the buffers (sn_reserve).
static void sn_decode(PfRows layout, PfSampleStep s0, const int* tok0, const int* p0, int n_tokens, float temperature, float minp,
                      unsigned long long* rng_states, int* out_tokens) {
	const int nseq = s0.nseq;
	const bool greedy = temperature == 0.0f || minp >= 1.0f; // sample() is greedy there and leaves the generator alone
	const size_t rows = (size_t)n_tokens * nseq;
	std::vector<int> pos(rows);
	for (size_t r = 0; r < rows; ++r) pos[r] = p0[r % nseq] + (int)(r / nseq);
	CUDA_CHECK(cudaMemcpyAsync(pf.snpos, pos.data(), rows * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaMemcpyAsync(pf.tokens, tok0, nseq * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	SampleState st[CALM_B200_SAMPLE_N_MAX];
	if (!greedy) {
		for (int b = 0; b < nseq; ++b) st[b].rng = rng_states[b], st[b].temperature = temperature, st[b].cut_delta = logf(minp) * temperature;
		CUDA_CHECK(cudaMemcpyAsync(pf.vstate, st, nseq * sizeof(SampleState), cudaMemcpyHostToDevice, g.stream));
	}
	for (int j = 0; j < n_tokens; ++j) {
		PfSampleStep ss = s0;
		ss.step = j;
		int* out = pf.sntok + (size_t)j * nseq;
		with_formats([&](auto f) {
			pf_run(f, nseq, s0.pos0 + j * nseq, layout, &ss);
			pf_score(f, nseq, layout, true, 0, !greedy);
		});
		if (greedy) CUDA_CHECK(cudaMemcpyAsync(out, pf.greedy, nseq * sizeof(int), cudaMemcpyDeviceToDevice, g.stream));
		else vf_sample_rows(nseq, out);
		if (j + 1 < n_tokens) CUDA_CHECK(cudaMemcpyAsync(pf.tokens, out, nseq * sizeof(int), cudaMemcpyDeviceToDevice, g.stream));
	}
	std::vector<int> all(rows);
	CUDA_CHECK(cudaMemcpyAsync(all.data(), pf.sntok, rows * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
	if (!greedy) CUDA_CHECK(cudaMemcpyAsync(st, pf.vstate, nseq * sizeof(SampleState), cudaMemcpyDeviceToHost, g.stream));
	sync_stream();
	CUDA_CHECK(cudaGetLastError());
	for (int b = 0; b < nseq; ++b)
		for (int i = 0; i < n_tokens; ++i) out_tokens[(size_t)b * n_tokens + i] = all[(size_t)i * nseq + b];
	if (!greedy) {
		for (int b = 0; b < nseq; ++b) rng_states[b] = st[b].rng;
		pf.vrows = nseq;
	}
}

extern "C" int calm_b200_decode_sample_n(struct Transformer* transformer, int token0, int pos0, int n_tokens, int nseq, float temperature, float minp,
                                         unsigned long long* rng_states, int* out_tokens) {
	if (!g.ready) CALM_FATAL("decode_sample_n before prepare_cuda");
	if (nseq < 1 || nseq > CALM_B200_SAMPLE_N_MAX) CALM_FATAL("decode_sample_n: nseq %d outside [1, %d]", nseq, CALM_B200_SAMPLE_N_MAX);
	if (n_tokens < 0) CALM_FATAL("decode_sample_n: negative n_tokens %d", n_tokens);
	if (n_tokens > 0 && (!rng_states || !out_tokens)) CALM_FATAL("decode_sample_n: rng_states or out_tokens is NULL");
	check_call(transformer, token0, pos0);
	if (n_tokens == 0) return 1;
	if (!pf_supported() || (long long)pos0 + (long long)nseq * n_tokens > g.cfg.seq_len) {
		for (int b = 0; b < nseq; ++b) calm_b200_decode_sample(transformer, token0, pos0, n_tokens, temperature, minp, &rng_states[b], out_tokens + (size_t)b * n_tokens);
		return 0;
	}
	sn_reserve(nseq, cdiv(pos0 + n_tokens, SN_CHUNK));
	int tok[CALM_B200_SAMPLE_N_MAX], pos[CALM_B200_SAMPLE_N_MAX];
	for (int b = 0; b < nseq; ++b) tok[b] = token0, pos[b] = pos0;
	sn_decode(PF_SAMPLES, PfSampleStep{pos0, 0, nseq, 0}, tok, pos, n_tokens, temperature, minp, rng_states, out_tokens);
	return 1;
}

// ---------------------------------------------------------------------------------------------
// calm_b200_decode_sample_batch: nseq sequences, each with its own prompt.  The prompts go through the prompt pass packed
// from slot 0 (PfPackedBlock, k_pf_attn<.., SEG>), then every step is one short block whose rows are the sequences
// (PF_BATCH), each row attending over its own prompt and its own interleaved slots (sample_n.cuh, BATCH).

constexpr int SB_BLOCK = 2048; // rows of a block of packed prompts

// The packed prompts of `pb` at cache slots base .. base + pb.rows() - 1, in blocks of at most SB_BLOCK rows at slot base
// base + o: pf.seg holds absolute slots, so a prompt that straddles a block edge walks its keys from its first slot, which
// the earlier block wrote.  Rows that continue a context (calm_b200_decode_sample_queue_context) carry its absolute first
// slot in pb.ctx; a block that holds such a row uploads pf.ctx and runs the context walk (PF_CONTEXTS), which reads the
// context's slots wherever an earlier block or an earlier call of this function wrote them.  The caller has reserved the
// pass for min(pb.rows(), SB_BLOCK) rows.
static void sb_prefill(PfPackedBlock& pb, int base) {
	for (int& s : pb.seg) s += base;
	const int G = pb.rows();
	for (int o = 0; o < G; o += SB_BLOCK) {
		const int m = imin(G - o, SB_BLOCK);
		const bool contexts = std::any_of(pb.ctx.begin() + o, pb.ctx.begin() + o + m, [](int2 c) { return c.y > 0; });
		CUDA_CHECK(cudaMemcpyAsync(pf.tokens, pb.tok.data() + o, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		CUDA_CHECK(cudaMemcpyAsync(pf.rowpos, pb.pos.data() + o, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		CUDA_CHECK(cudaMemcpyAsync(pf.seg, pb.seg.data() + o, (size_t)m * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		if (contexts) CUDA_CHECK(cudaMemcpyAsync(pf.ctx, pb.ctx.data() + o, (size_t)m * sizeof(int2), cudaMemcpyHostToDevice, g.stream));
		pf_block(m, base + o, contexts ? PF_CONTEXTS : PF_PACKED, nullptr, PfOut());
	}
}

extern "C" int calm_b200_decode_sample_batch(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nseq,
                                             int n_tokens, float temperature, float minp, unsigned long long* rng_states, int* out_tokens) {
	if (!g.ready) CALM_FATAL("decode_sample_batch before prepare_cuda");
	if (nseq < 1 || nseq > CALM_B200_SAMPLE_N_MAX) CALM_FATAL("decode_sample_batch: nseq %d outside [1, %d]", nseq, CALM_B200_SAMPLE_N_MAX);
	if (n_tokens < 0) CALM_FATAL("decode_sample_batch: negative n_tokens %d", n_tokens);
	if (n_tokens == 0) return 1;
	if (!tokens || !off || !len || !rng_states || !out_tokens) CALM_FATAL("decode_sample_batch: an array is NULL");
	if (n < 0) CALM_FATAL("decode_sample_batch: negative n %d", n);
	for (int b = 0; b < nseq; ++b)
		if (len[b] < 1 || off[b] < 0 || (long)off[b] + len[b] > n) CALM_FATAL("decode_sample_batch: prompt %d (off %d, len %d) empty or outside the %d tokens", b, off[b], len[b], n);
	check_tokens(tokens, n);
	// prompt b's L_b = len[b] - 1 rows take ceil8(L_b) slots from s_b; the steps follow from G, nseq slots each
	long long G = 0;
	int lmax = 0;
	for (int b = 0; b < nseq; ++b) G += cdiv(len[b] - 1, 8) * 8, lmax = std::max(lmax, len[b] - 1);
	if (!pf_supported() || G + (long long)nseq * n_tokens > g.cfg.seq_len) {
		for (int b = 0; b < nseq; ++b) {
			const int* p = tokens + off[b];
			forward_prefill_cuda(transformer, p, len[b] - 1, 0);
			calm_b200_decode_sample(transformer, p[len[b] - 1], len[b] - 1, n_tokens, temperature, minp, &rng_states[b], out_tokens + (size_t)b * n_tokens);
		}
		return 0;
	}
	PfPackedBlock pb;
	int2 rows[CALM_B200_SAMPLE_N_MAX];
	int tok[CALM_B200_SAMPLE_N_MAX], pos[CALM_B200_SAMPLE_N_MAX];
	for (int b = 0; b < nseq; ++b) {
		const int* p = tokens + off[b];
		const int L = len[b] - 1;
		rows[b] = make_int2(pb.add(p, L, L, 0, make_int2(0, 0)), L), tok[b] = p[L], pos[b] = L;
	}
	sn_reserve(std::max(imin((int)G, SB_BLOCK), nseq), cdiv(lmax + n_tokens, SN_CHUNK));
	if (!pf.sbrows) pf.sbrows = (int2*)dev_alloc(VF_TOK * sizeof(int2));
	CUDA_CHECK(cudaMemcpyAsync(pf.sbrows, rows, nseq * sizeof(int2), cudaMemcpyHostToDevice, g.stream));
	sb_prefill(pb, 0);
	sn_decode(PF_BATCH, PfSampleStep{(int)G, 0, nseq, lmax}, tok, pos, n_tokens, temperature, minp, rng_states, out_tokens);
	return 1;
}

// ---------------------------------------------------------------------------------------------
// calm_b200_decode_sample_queue: a queue of requests, at most max_rows in flight.  Before every step the requests at the
// head of the queue that fit are admitted (a round): their prompts go through the packed prompt pass, then every step is
// one short block over the rows in flight (PF_QUEUE), and a row retires after max_new tokens or a stop token.  Cache slots
// are placed by SqSlots (include/calm_b200.h states the rule).

static_assert(SQ_ROWS == VF_TOK, "the rows of a queue step are one token tile of k_vf_gemm");

// First-fit allocation of cache slots in [0, seq_len), coalescing on release
struct SqSlots {
	std::map<int, int> free_; // start -> end of each free interval
	explicit SqSlots(int n) { free_[0] = n; }
	// the lowest start, a multiple of `align`, of n free slots, taken; -1 if there is none
	int take(int n, int align) {
		for (auto it = free_.begin(); it != free_.end(); ++it) {
			const int s = it->first, e = it->second, a = cdiv(s, align) * align;
			if (a + n > e) continue;
			free_.erase(it);
			if (s < a) free_[s] = a;
			if (a + n < e) free_[a + n] = e;
			return a;
		}
		return -1;
	}
	void give(int s, int n) {
		if (n == 0) return;
		int e = s + n;
		auto nx = free_.lower_bound(s);
		if (nx != free_.end() && nx->first == e) e = nx->second, nx = free_.erase(nx);
		if (nx != free_.begin() && std::prev(nx)->second == s) {
			std::prev(nx)->second = e;
			return;
		}
		free_[s] = e;
	}
};

// A request's place: its context's nc entries at slots c .. (nc = 0: none), its own prompt entries (L - nc of them) at
// slots s .., its generated entries at slots t ..
struct SqPlace {
	int s, L, t, c, nc;
};

using SqCtx = std::pair<int, int>; // a context by (ctx_off, ctx_len): requests share it exactly when these are equal

// The requests' contexts.  Both arrays NULL: no request has a context, except where `required` (the context call).
struct SqContexts {
	const int *ctx_off, *ctx_len;
	bool required;
	int off(int i) const { return ctx_off ? ctx_off[i] : 0; }
	int len(int i) const { return ctx_len ? ctx_len[i] : 0; }
	SqCtx key(int i) const { return SqCtx(off(i), len(i)); }
	bool missing() const { return !ctx_off != !ctx_len || (required && !ctx_off); }
};

// The placement of one round, the requests `rs` in input order, with the contexts `resident` holds at their first slots:
// one extent starting at a multiple of 8 that holds, request by request, the request's context (ceil8(ctx_len) slots) if
// it is neither resident nor placed by an earlier request of the round, then its own prompt (ceil8(len - 1) slots); then
// one extent of max_new slots per request.  False (and `a` spent) when one does not fit; `base` gets the first extent's
// first slot.
static bool sq_place(SqSlots& a, const std::vector<int>& rs, const SqContexts& ctx, const int* len, const int* max_new, const std::map<SqCtx, int>& resident,
                     std::vector<SqPlace>& out, int& base) {
	std::map<SqCtx, int> placed; // contexts of this round, by their offset in the extent
	int P = 0;
	for (int i : rs) {
		const SqCtx k = ctx.key(i);
		if (ctx.len(i) && !resident.count(k) && !placed.count(k)) placed[k] = P, P += cdiv(ctx.len(i), 8) * 8;
		P += cdiv(len[i] - 1, 8) * 8;
	}
	const int s0 = base = P ? a.take(P, 8) : 0;
	if (s0 < 0) return false;
	out.clear();
	std::set<SqCtx> seen;
	int s = s0;
	for (int i : rs) {
		const SqCtx k = ctx.key(i);
		int c = 0;
		if (ctx.len(i)) {
			const auto r = resident.find(k);
			c = r != resident.end() ? r->second : s0 + placed.at(k);
			if (r == resident.end() && seen.insert(k).second) s += cdiv(ctx.len(i), 8) * 8;
		}
		const int t = a.take(max_new[i], 1);
		if (t < 0) return false;
		out.push_back(SqPlace{s, ctx.len(i) + len[i] - 1, t, c, ctx.len(i)});
		s += cdiv(len[i] - 1, 8) * 8;
	}
	return true;
}

// The log-probability outputs of calm_b200_decode_sample_queue_logprobs: request i step j writes logprobs[O_i + j] and
// top_ids / top_logprobs[(O_i + j) * k ..] (off: none, and k is 0)
struct SqLogprobs {
	bool on;
	int k;
	float* logprobs;
	int* top_ids;
	float* top_logprobs;
};

// Queue buffers sharing capacity `cap` regrown to `need` elements, after the stream: no earlier call still reads them
template <typename... T>
static void sq_grow(size_t& cap, size_t need, T*&... bufs) {
	if (need <= cap) return;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	cap = need;
	((cudaFree(bufs), bufs = (T*)dev_alloc(need * sizeof(T))), ...);
}

// One launch of a queue step's classifier: MASK (with PEN, TOPK) if `mask`, else PEN (with TOPK) if `pen`, else TOPK if k > 0
template <int MODE, int DBITS, typename KVT>
static void sq_gemm(const PfGemmArgs& a, int units, int t0, int k, bool pen, bool mask) {
	if (mask) vf_gemm<MODE, DBITS, KVT, true, true, true>(pf.Nhi, pf.Nlo, a, units, t0);
	else if (pen) vf_gemm<MODE, DBITS, KVT, true, true>(pf.Nhi, pf.Nlo, a, units, t0);
	else if (k) vf_gemm<MODE, DBITS, KVT, true>(pf.Nhi, pf.Nlo, a, units, t0);
	else vf_gemm<MODE, DBITS, KVT>(pf.Nhi, pf.Nlo, a, units, t0);
}

// A queue step's final norm and short-block classifier: greedy (or, with `sample`, sampled) on the n rows, with k > 0
// writing each tile's top-k lists to pf.sqtopv / pf.sqtopi, with `pen` (a step with non-neutral rows) processing those
// rows' logits and with `mask` (a step with a constrained row) also masking them.  The merge is left to the caller.
template <int DBITS, typename KVT>
static void sq_classify(Formats<DBITS, KVT>, int n, int k, bool sample, bool pen, bool mask) {
	const Config& c = g.cfg;
	const int nvt = cdiv(c.vocab_size, PF_BM);
	launch_pdl(k_pf_norm, n, 256, 0, (const float*)pf.X, (const float*)g.w.rms_final_weight, pf.Nhi, pf.Nlo, n, c.dim, c.norm_eps, (int)c.norm_ln);
	PfGemmArgs a = {};
	a.n_tokens = n, a.w[0] = g.w.wcls, a.K = c.dim;
	a.targets = pf.targets, a.part = pf.part, a.tgt = pf.tgt, a.vocab = c.vocab_size, a.gidx = pf.gidx;
	a.topv = pf.sqtopv, a.topi = pf.sqtopi, a.topk = k;
	const auto gemm = sample ? sq_gemm<PF_CLS_SAMPLE, DBITS, KVT> : sq_gemm<PF_CLS_GREEDY, DBITS, KVT>;
	for (int t0 = 0; t0 < nvt; t0 += VF_CLS_UNITS) gemm(a, imin(VF_CLS_UNITS, nvt - t0), t0, k, pen, mask);
}

// The merge of a step with log-probabilities: pf_merge's greedy merge (k > 0: with the top-k lists of pf.sqtopv into
// pf.sqtid / pf.sqtlp), every row's log-probability that of its target
static void sq_merge(int n, int k) {
	const int nvt = cdiv(g.cfg.vocab_size, PF_BM);
	const auto merge = k ? k_pf_logprob<true, true> : k_pf_logprob<true>;
	launch_pdl(merge, cdiv(n, 8), 256, k ? (size_t)8 * nvt : 0, (const float2*)pf.part, (const float*)pf.tgt, pf.logprob, n, nvt, (const int*)pf.gidx,
	           pf.greedy, (const float*)pf.sqtopv, (const int*)pf.sqtopi, k, pf.sqtid, pf.sqtlp);
}

// The logit processing of calm_b200_decode_sample_queue_penalties (include/calm_b200.h): presence / frequency /
// repetition may each be NULL (0, 0, 1), bias_off / bias_len both NULL when n_bias == 0
// calm_b200_decode_sample_queue_truncated's per-request top_k / top_p (either array may be NULL: 0 / 1 for every request)
struct SqTrunc {
	const int* top_k;
	const float* top_p;
	int k(int i) const { return top_k ? top_k[i] : 0; }
	float p(int i) const { return top_p ? top_p[i] : 1.0f; }
};

struct SqPenalties {
	const float* presence;
	const float* frequency;
	const float* repetition;
	const int* bias_off;
	const int* bias_len;
	const int* bias_ids;
	const float* bias_val;
	int n_bias;
	float p(int i) const { return presence ? presence[i] : 0.0f; }
	float f(int i) const { return frequency ? frequency[i] : 0.0f; }
	float r(int i) const { return repetition ? repetition[i] : 1.0f; }
	int nb(int i) const { return bias_len ? bias_len[i] : 0; }
	bool neutral(int i) const { return p(i) == 0.0f && f(i) == 0.0f && r(i) == 1.0f && nb(i) == 0; }
};

// sq_pen_logit on the host, for the fallback: the same IEEE operations, one per statement (no contraction)
static float sq_pen_logit_host(float l, int c, bool seen, float b, float p, float f, float r) {
	float l1 = l;
	if (seen && r != 1.0f) l1 = l > 0.0f ? l / r : l * r;
	const float fc = f * (float)c;
	const float bf = b - fc;
	const float a = bf - (c > 0 ? p : 0.0f);
	return a == 0.0f ? l1 : l1 + a;
}

// The token automaton of calm_b200_decode_sample_queue_constrained (include/calm_b200.h) and each request's start state
// (start NULL: no request is constrained).  sq_check checks it and fills `fin`, which states are final.
struct SqAutomaton {
	int n_states;
	const uint32_t* allow;
	const int* next_default;
	const int* exc_off;
	const int* exc_tok;
	const int* exc_next;
	const int* start;
	int* out_state;
	int words;             // ceil(vocab / 32): one state's bitmask
	std::vector<char> fin; // [n_states] no token allowed
	int s0(int i) const { return start ? start[i] : -1; }
	bool ends(int s) const { return s >= 0 && fin[s]; } // a token that led to state s ends its request
	bool allowed(int s, int v) const { return (allow[(size_t)s * words + (v >> 5)] >> (v & 31)) & 1u; }
	// the state after allowed token v in state s: its exception, else the default.  v comes from the device (or the
	// fallback's sampler), which never draws a masked token; one that did would be a bug, so it aborts here rather than
	// taking a default that may be -1 and leaving the request unconstrained.
	int next(int s, int v) const {
		if (v < 0 || v >= words * 32 || !allowed(s, v)) CALM_FATAL("constrained queue: token %d is not allowed in state %d", v, s);
		const int* b = exc_tok + exc_off[s];
		const int* e = exc_tok + exc_off[s + 1];
		const int* x = std::lower_bound(b, e, v);
		return x != e && *x == v ? exc_next[x - exc_tok] : next_default[s];
	}
};

// Abort unless `a` is a well-formed automaton for a vocabulary of `vocab` tokens with valid start states (the automaton
// itself is read only when some request is constrained); fills a.words and a.fin
static void sq_check_automaton(const char* who, SqAutomaton& a, int nreq, const int* max_new, int vocab) {
	if (a.n_states < 0) CALM_FATAL("%s: negative n_states %d", who, a.n_states);
	a.words = cdiv(vocab, 32);
	bool any = false;
	for (int i = 0; i < nreq; ++i) {
		if (a.s0(i) < -1 || a.s0(i) >= a.n_states) CALM_FATAL("%s: request %d's start state %d outside [-1, %d)", who, i, a.s0(i), a.n_states);
		any = any || a.s0(i) >= 0;
	}
	if (!any) return;
	if (!a.allow || !a.next_default || !a.exc_off || !a.exc_tok || !a.exc_next) CALM_FATAL("%s: an automaton array is NULL", who);
	if (a.exc_off[0] != 0) CALM_FATAL("%s: exc_off[0] is %d, not 0", who, a.exc_off[0]);
	const uint32_t tail = vocab % 32 ? ~0u << (vocab % 32) : 0u; // the last word's bits past the vocabulary
	a.fin.assign(a.n_states, 0);
	for (int s = 0; s < a.n_states; ++s) {
		const uint32_t* w = a.allow + (size_t)s * a.words;
		if (w[a.words - 1] & tail) CALM_FATAL("%s: state %d allows a token past the %d-token vocabulary", who, s, vocab);
		long allowed = 0;
		for (int j = 0; j < a.words; ++j) allowed += __builtin_popcount(w[j]);
		a.fin[s] = allowed == 0;
		const int e0 = a.exc_off[s], e1 = a.exc_off[s + 1];
		if (e1 < e0) CALM_FATAL("%s: exc_off decreases at state %d (%d, %d)", who, s, e0, e1);
		for (int e = e0; e < e1; ++e) {
			const int v = a.exc_tok[e];
			if (v < 0 || v >= vocab || !a.allowed(s, v)) CALM_FATAL("%s: state %d's exception token %d is not allowed in it", who, s, v);
			if (e > e0 && v <= a.exc_tok[e - 1]) CALM_FATAL("%s: state %d's exception tokens are not strictly ascending at %d", who, s, v);
			if (a.exc_next[e] < 0 || a.exc_next[e] >= a.n_states) CALM_FATAL("%s: state %d's exception next state %d outside [0, %d)", who, s, a.exc_next[e], a.n_states);
		}
		const int d = a.next_default[s];
		if (d < -1 || d >= a.n_states) CALM_FATAL("%s: state %d's default next state %d outside [-1, %d)", who, s, d, a.n_states);
		if (d == -1 && allowed > e1 - e0) CALM_FATAL("%s: state %d allows a token outside its exception list and has no default next state", who, s);
	}
	for (int i = 0; i < nreq; ++i)
		if (max_new[i] > 0 && a.s0(i) >= 0 && a.fin[a.s0(i)]) CALM_FATAL("%s: request %d starts in final state %d", who, i, a.s0(i));
}

// The prompt-lookup drafts of calm_b200_decode_sample_queue_lookup: up to max_draft draft rows per request and step, and
// where the call counts the draft rows it ran and the drafts it accepted (either may be NULL)
struct SqLookup {
	int max_draft;
	int* drafted;
	int* accepted;
};

// One queue call: its requests and every option, each option neutral (all-zero) where the entry point has none of it
struct SqCall {
	const char* who; // the entry point, in error messages
	struct Transformer* transformer;
	const int* tokens;
	int n;
	SqContexts ctx;
	const int *off, *len;
	int nreq;
	const int* max_new;
	const float *temperature, *minp;
	const int* stop;
	int n_stop, max_rows;
	unsigned long long* rng_states;
	int *out_tokens, *out_len, *steps, *prompt_rows;
	SqLogprobs lp = {};
	SqPenalties pen = {};
	SqAutomaton aut = {};
	SqTrunc tr = {};
	SqLookup lk = {};
	bool greedy(int i) const { return temperature[i] == 0.0f || minp[i] >= 1.0f; } // sample() is greedy there
	bool truncated(int i) const { return !greedy(i) && (tr.k(i) > 0 || tr.p(i) < 1.0f); } // a sampled request with top-k or top-p
};

// Abort on a bad argument, before any device work; fills c.aut's words and final states, returns the sum of max_new
static size_t sq_check(SqCall& c) {
	const char* who = c.who;
	const int nreq = c.nreq, n = c.n;
	if (!g.ready) CALM_FATAL("%s before prepare_cuda", who);
	if (c.max_rows < 1 || c.max_rows > CALM_B200_SAMPLE_N_MAX) CALM_FATAL("%s: max_rows %d outside [1, %d]", who, c.max_rows, CALM_B200_SAMPLE_N_MAX);
	if (nreq < 0 || n < 0 || c.n_stop < 0) CALM_FATAL("%s: negative nreq %d, n %d or n_stop %d", who, nreq, n, c.n_stop);
	if (c.n_stop > 0 && !c.stop) CALM_FATAL("%s: stop is NULL", who);
	if (nreq > 0 && (!c.tokens || c.ctx.missing() || !c.off || !c.len || !c.max_new || !c.temperature || !c.minp || !c.rng_states || !c.out_tokens ||
	                 !c.out_len))
		CALM_FATAL("%s: an array is NULL", who);
	size_t total = 0; // sum of max_new: the output's extent
	for (int i = 0; i < nreq; ++i) {
		const int mn = c.max_new[i], o = c.off[i], l = c.len[i], co = c.ctx.off(i), cl = c.ctx.len(i);
		if (mn < 0) CALM_FATAL("%s: request %d has a negative max_new %d", who, i, mn);
		if (l < 1 || o < 0 || (long)o + l > n) CALM_FATAL("%s: prompt %d (off %d, len %d) empty or outside the %d tokens", who, i, o, l, n);
		if (co < 0 || cl < 0 || (long)co + cl > n) CALM_FATAL("%s: context of request %d (off %d, len %d) outside the %d tokens", who, i, co, cl, n);
		total += mn;
	}
	if (total > 0x7fffffff) CALM_FATAL("%s: %zu output tokens do not fit an int index", who, total);
	const SqPenalties& pen = c.pen;
	const int vocab = g.cfg.vocab_size;
	if (c.lp.on) {
		const int kmax = imin(CALM_B200_TOPK_MAX, vocab);
		if (c.lp.k < 0 || c.lp.k > kmax) CALM_FATAL("%s: k %d outside [0, %d]", who, c.lp.k, kmax);
		if (total > 0 && !c.lp.logprobs) CALM_FATAL("%s: logprobs is NULL", who);
		if (total > 0 && c.lp.k > 0 && (!c.lp.top_ids || !c.lp.top_logprobs)) CALM_FATAL("%s: top_ids or top_logprobs is NULL", who);
	}
	const float big = 1e6f; // bounds that keep every processed logit finite
	if (pen.n_bias < 0) CALM_FATAL("%s: negative n_bias %d", who, pen.n_bias);
	if (!pen.bias_off != !pen.bias_len || (!pen.bias_off && pen.n_bias > 0)) CALM_FATAL("%s: bias_off or bias_len is NULL", who);
	if (pen.n_bias > 0 && (!pen.bias_ids || !pen.bias_val)) CALM_FATAL("%s: bias_ids or bias_val is NULL", who);
	std::vector<int> listed(pen.bias_off ? vocab : 0, -1); // the request whose list last named the id
	for (int i = 0; i < nreq; ++i) {
		const float p = pen.p(i), f = pen.f(i), r = pen.r(i);
		if (!std::isfinite(p) || !std::isfinite(f) || !std::isfinite(r) || fabsf(p) > big || fabsf(f) > big || !(r >= 1e-6f && r <= big))
			CALM_FATAL("%s: request %d's presence %g, frequency %g or repetition %g is not finite or out of bounds", who, i, p, f, r);
		if (!pen.bias_off) continue;
		const int bo = pen.bias_off[i], bl = pen.bias_len[i];
		if (bo < 0 || bl < 0 || (long)bo + bl > pen.n_bias) CALM_FATAL("%s: bias list %d (off %d, len %d) outside the %d entries", who, i, bo, bl, pen.n_bias);
		for (int e = bo; e < bo + bl; ++e) {
			const int id = pen.bias_ids[e];
			const float b = pen.bias_val[e];
			if (id < 0 || id >= vocab) CALM_FATAL("%s: request %d's bias id %d outside [0, %d)", who, i, id, vocab);
			if (listed[id] == i) CALM_FATAL("%s: request %d's bias list repeats id %d", who, i, id);
			if (!std::isfinite(b) || fabsf(b) > big) CALM_FATAL("%s: request %d's bias %g for id %d is not finite or out of bounds", who, i, b, id);
			listed[id] = i;
		}
	}
	sq_check_automaton(who, c.aut, nreq, c.max_new, vocab);
	for (int i = 0; i < nreq; ++i) {
		trunc_check(who, i, c.tr.k(i), c.tr.p(i));
		if (c.max_new[i] > 0 && c.truncated(i) && vocab > TRUNC_VOCAB_MAX)
			CALM_FATAL("%s: request %d is truncated, and truncation serves vocabularies up to %d tokens, not %d", who, i, TRUNC_VOCAB_MAX, vocab);
	}
	if (c.lk.max_draft < 0 || c.lk.max_draft > SQ_ROWS - 1) CALM_FATAL("%s: max_draft %d outside [0, %d]", who, c.lk.max_draft, SQ_ROWS - 1);
	check_tokens(c.tokens, n);
	check_tokens(c.stop, c.n_stop);
	return total;
}

// The host path (MoE, tensor parallelism, a request past seq_len): each request alone, decode_sample's stream cut at a stop
static int sq_fallback(const SqCall& c, std::vector<int>& cur, const std::vector<char>& is_stop, const std::vector<size_t>& O) {
	for (int i = 0; i < c.nreq; ++i) {
		std::vector<int> p(c.tokens + c.ctx.off(i), c.tokens + c.ctx.off(i) + c.ctx.len(i));
		p.insert(p.end(), c.tokens + c.off[i], c.tokens + c.off[i] + c.len[i]);
		const int L = (int)p.size() - 1;
		int tok = p[L], k = 0;
		if (c.max_new[i] > 0) forward_prefill_cuda(c.transformer, p.data(), L, 0);
		const bool processed = !c.pen.neutral(i), masked = cur[i] >= 0, cut = c.truncated(i);
		std::vector<float> logits(c.lp.on || processed || masked || cut ? g.cfg.vocab_size : 0);
		std::vector<int> cnt(processed ? g.cfg.vocab_size : 0);
		std::vector<float> bias(processed ? g.cfg.vocab_size : 0);
		std::vector<char> seen(processed ? g.cfg.vocab_size : 0);
		if (processed) {
			for (int t : p) seen[t] = 1;
			for (int e = 0; e < c.pen.nb(i); ++e) bias[c.pen.bias_ids[c.pen.bias_off[i] + e]] = c.pen.bias_val[c.pen.bias_off[i] + e];
		}
		while (k < c.max_new[i]) {
			if (processed || masked || cut) { // the decode path's device logits (its argmax discarded), processed, masked and sampled on the host
				unsigned long long unused = 1;
				calm_b200_forward_sample(c.transformer, tok, L + k, 0.0f, 0.0f, &unused);
				calm_b200_read_device_logits(logits.data());
				for (int v = 0; processed && v < g.cfg.vocab_size; ++v)
					logits[v] = sq_pen_logit_host(logits[v], cnt[v], seen[v] || cnt[v] > 0, bias[v], c.pen.p(i), c.pen.f(i), c.pen.r(i));
				for (int v = 0; masked && v < g.cfg.vocab_size; ++v)
					if (!c.aut.allowed(cur[i], v)) logits[v] = -INFINITY;
				// (greedy: the first maximum; sampled: through k_sample_scan_rows_masked where the row is masked, after
				// k_sample_trunc_rows where it is truncated)
				tok = sample_logits(logits.data(), g.cfg.vocab_size, c.temperature[i], c.minp[i], &c.rng_states[i], nullptr, masked, cut ? c.tr.k(i) : 0,
				                    cut ? c.tr.p(i) : 1.0f);
				if (processed) ++cnt[tok];
				if (c.lp.on) {
					const size_t o = O[i] + k;
					host_logprobs(logits.data(), g.cfg.vocab_size, tok, c.lp.k, c.lp.logprobs + o, c.lp.top_ids + o * c.lp.k, c.lp.top_logprobs + o * c.lp.k);
					for (size_t e = o * c.lp.k; masked && e < (o + 1) * c.lp.k; ++e) // ranks past the allowed tokens
						if (c.lp.top_logprobs[e] == -INFINITY) c.lp.top_ids[e] = -1;
				}
				c.out_tokens[O[i] + k++] = tok;
				if (masked) cur[i] = c.aut.next(cur[i], tok);
				if (is_stop[tok] || c.aut.ends(cur[i])) break;
				continue;
			}
			tok = calm_b200_forward_sample(c.transformer, tok, L + k, c.temperature[i], c.minp[i], &c.rng_states[i]);
			if (c.lp.on) { // the step's device logits, through pf_score_one's decode-path log-softmax
				const size_t o = O[i] + k;
				calm_b200_read_device_logits(logits.data());
				host_logprobs(logits.data(), g.cfg.vocab_size, tok, c.lp.k, c.lp.logprobs + o, c.lp.top_ids + o * c.lp.k, c.lp.top_logprobs + o * c.lp.k);
			}
			c.out_tokens[O[i] + k++] = tok;
			if (is_stop[tok]) break;
		}
		c.out_len[i] = k;
		if (c.aut.out_state) c.aut.out_state[i] = cur[i];
	}
	return 0;
}

// A step's top-k tile lists and merged lists for VF_TOK rows and the largest k (sq_classify / sq_merge with k > 0)
static void sq_topk_reserve() {
	if (pf.sqtopv) return;
	const size_t nvt = cdiv(g.cfg.vocab_size, PF_BM);
	pf.sqtopv = (float*)dev_alloc(VF_TOK * nvt * PF_TOPK_MAX * sizeof(float));
	pf.sqtopi = (int*)dev_alloc(VF_TOK * nvt * PF_TOPK_MAX * sizeof(int));
	pf.sqtid = (int*)dev_alloc(VF_TOK * PF_TOPK_MAX * sizeof(int));
	pf.sqtlp = (float*)dev_alloc(VF_TOK * PF_TOPK_MAX * sizeof(float));
}

// The device buffers of a call of `total` tokens and its uploads, once per call: the lanes' rows, tokens and bias lists
// when a request is not neutral, the automaton's bitmasks when one is constrained (cur: each request's start state)
static void sq_reserve(const SqCall& c, size_t total, const std::vector<int>& cur) {
	const size_t vocab = g.cfg.vocab_size;
	if (!pf.sqrows) {
		pf.sqrows = (SqRows*)dev_alloc(sizeof(SqRows));
		pf.sqgroups = (SqGroups*)dev_alloc(sizeof(SqGroups));
		pf.sqtok = (int*)dev_alloc(2 * VF_TOK * sizeof(int));
		pf.sqlanes = (int*)dev_alloc(2 * SQ_ROWS * sizeof(int));
	}
	sq_grow(pf.sqout_cap, total, pf.sqout);
	sq_grow(pf.sqst_cap, c.nreq, pf.sqst);
	if (c.lp.on) sq_topk_reserve();
	if (c.lp.on) sq_grow(pf.sqlp_cap, total, pf.sqlp), sq_grow(pf.sqtop_cap, total * c.lp.k, pf.sqoid, pf.sqolp);
	bool any_pen = false, any_aut = false; // a request with max_new > 0 is not neutral / is constrained
	for (int i = 0; i < c.nreq; ++i) any_pen = any_pen || (c.max_new[i] > 0 && !c.pen.neutral(i));
	for (int i = 0; i < c.nreq; ++i) any_aut = any_aut || (c.max_new[i] > 0 && cur[i] >= 0);
	if (any_pen) {
		if (!pf.sqpcnt) {
			pf.sqpcnt = (int*)dev_alloc(SQ_ROWS * vocab * sizeof(int));
			pf.sqpbias = (float*)dev_alloc(SQ_ROWS * vocab * sizeof(float));
			pf.sqppar = (float4*)dev_alloc(SQ_ROWS * sizeof(float4));
		}
		sq_grow(pf.sqptok_cap, c.n, pf.sqptok);
		sq_grow(pf.sqpb_cap, c.pen.n_bias, pf.sqpbid, pf.sqpbval);
		CUDA_CHECK(cudaMemcpyAsync(pf.sqptok, c.tokens, (size_t)c.n * sizeof(int), cudaMemcpyHostToDevice, g.stream));
		if (c.pen.n_bias) {
			CUDA_CHECK(cudaMemcpyAsync(pf.sqpbid, c.pen.bias_ids, (size_t)c.pen.n_bias * sizeof(int), cudaMemcpyHostToDevice, g.stream));
			CUDA_CHECK(cudaMemcpyAsync(pf.sqpbval, c.pen.bias_val, (size_t)c.pen.n_bias * sizeof(float), cudaMemcpyHostToDevice, g.stream));
		}
	}
	if (any_aut) {
		const size_t words = (size_t)c.aut.n_states * c.aut.words;
		sq_grow(pf.sqallow_cap, words, pf.sqallow);
		CUDA_CHECK(cudaMemcpyAsync(pf.sqallow, c.aut.allow, words * sizeof(uint32_t), cudaMemcpyHostToDevice, g.stream));
	}
}

// One step's tables, as SqLoop::build leaves them for launch and retire
struct SqStep {
	SqRows r = {};
	SqGroups grp = {};
	SqLanes lanes;          // each row's penalty lane and automaton state
	TruncRows trows = {};   // the step's truncated rows
	SqNext nx = {};         // the draft each row's successor is fed, -1 after a request's last row
	int first[SQ_ROWS + 1]; // live request k's rows are first[k] .. first[k + 1] - 1
	int ntrunc = 0, nsampled = 0, lmax = 0, nsuf = 0;
	bool pen = false, mask = false, mask_sampled = false; // a row is a non-neutral request's; a constrained one's; .. that samples
};

// The step loop of a call that the batched path serves, and what it keeps across steps
struct SqLoop {
	const SqCall& c;
	std::vector<int>& cur; // a constrained request's automaton state after its tokens so far
	const std::vector<char>& is_stop;
	const std::vector<size_t>& O;
	const bool drafting;
	std::vector<int> lane_of;                 // a non-neutral request's lane while it is in flight
	std::vector<std::vector<int>> corpus;     // (drafting) ctx ++ prompt ++ tokens so far: the lookup's sequence
	std::vector<unsigned long long> hst;      // a sampled request's state after its tokens so far
	unsigned lanes_free = (1u << SQ_ROWS) - 1;
	SqSlots slots;
	std::map<SqCtx, int> resident; // contexts in the cache, at their first slot
	std::vector<int> done, row_of, live; // tokens so far; row in the last step; requests in flight, in admission order
	std::vector<int> round;              // the requests admitted before this step, their placement rp and its first slot rbase
	std::vector<SqPlace> place, rp;      // (place: every admitted request's)
	int rbase = 0, head = 0, nsteps = 0, rows_computed = 0, ndrafted = 0, naccepted = 0;
	int last_sampled = 0, tok_host[2 * VF_TOK]; // the last step's rows if it sampled; its tokens, read back

	SqLoop(const SqCall& c, std::vector<int>& cur, const std::vector<char>& is_stop, const std::vector<size_t>& O)
	    : c(c), cur(cur), is_stop(is_stop), O(O), drafting(c.lk.max_draft > 0), lane_of(c.nreq, -1), corpus(drafting ? c.nreq : 0),
	      hst(c.rng_states, c.rng_states + c.nreq), slots(g.cfg.seq_len), done(c.nreq, 0), row_of(c.nreq, -1), place(c.nreq) {}

	// A round: the requests at the head of the queue, in input order, while a row is free and their placement fits
	void take_round() {
		round.clear(), rp.clear();
		SqSlots after = slots;
		while (head < c.nreq && (int)(live.size() + round.size()) < c.max_rows) {
			if (c.max_new[head] == 0) {
				++head;
				continue;
			}
			std::vector<int> trial = round;
			trial.push_back(head);
			SqSlots a = slots;
			std::vector<SqPlace> tp;
			int tb;
			if (!sq_place(a, trial, c.ctx, c.len, c.max_new, resident, tp, tb)) break;
			round.swap(trial), rp.swap(tp), after = a, rbase = tb, ++head;
		}
		slots = after;
	}

	// Admission before a step: a round, the resident contexts no request in flight or of the round names released, the
	// round's prompts through the packed prompt pass and a lane for each non-neutral request of it; false when none is left
	bool admit() {
		take_round();
		std::set<SqCtx> named;
		for (int i : live) named.insert(c.ctx.key(i));
		for (int i : round) named.insert(c.ctx.key(i));
		for (auto it = resident.begin(); it != resident.end();) {
			if (named.count(it->first)) {
				++it;
				continue;
			}
			slots.give(it->second, cdiv(it->first.second, 8) * 8);
			it = resident.erase(it);
		}
		if (live.empty() && round.empty()) { // the cache is empty now: the head fits
			take_round();
			if (round.empty()) return false;
		}
		if (round.empty()) return true;
		PfPackedBlock pb;
		for (size_t k = 0; k < round.size(); ++k) {
			const int i = round[k];
			const SqPlace& q = rp[k];
			place[i] = q;
			const SqCtx key = c.ctx.key(i);
			if (q.nc && !resident.count(key)) { // placed by this round, at the extent's next rows
				resident[key] = q.c;
				pb.add(c.tokens + c.ctx.off(i), q.nc, q.nc - 1, 0, make_int2(0, 0));
			}
			pb.add(c.tokens + c.off[i], c.len[i] - 1, c.len[i] - 1, q.nc, make_int2(q.c, q.nc));
			if (drafting) {
				corpus[i].assign(c.tokens + c.ctx.off(i), c.tokens + c.ctx.off(i) + c.ctx.len(i));
				corpus[i].insert(corpus[i].end(), c.tokens + c.off[i], c.tokens + c.off[i] + c.len[i]);
			}
			if (!c.pen.neutral(i)) { // the lowest free lane
				const int ln = __builtin_ctz(lanes_free);
				lanes_free &= ~(1u << ln), lane_of[i] = ln;
				const SqPenAdmit qa = {ln, c.ctx.off(i), c.ctx.len(i), c.off[i], c.len[i], c.pen.bias_off ? c.pen.bias_off[i] : 0,
				                       c.pen.nb(i), make_float4(c.pen.p(i), c.pen.f(i), c.pen.r(i), 0.0f)};
				launch_pdl(k_sq_pen_admit, cdiv(g.cfg.vocab_size, SQ_PEN_SPAN), 256, 0, qa, (const int*)pf.sqptok, (const int*)pf.sqpbid,
				           (const float*)pf.sqpbval, g.cfg.vocab_size, pf.sqpcnt, pf.sqpbias, pf.sqppar);
			}
		}
		if (pb.rows()) sb_prefill(pb, rbase);
		rows_computed += pb.rows();
		live.insert(live.end(), round.begin(), round.end());
		return true;
	}

	// The step's rows in flight in admission order, each request's draft rows after its row in the rows left free: draft row
	// d at step j + d, fed the draft's d-th token, the generator advanced d times and the state advanced through the draft
	SqStep build() {
		SqStep s;
		SqRows& r = s.r;
		const int nlive = (int)live.size();
		int nfree = SQ_ROWS - nlive;            // rows left for drafts
		std::map<int, std::vector<int>> groups; // rows by their context's first slot
		std::vector<int> gorder;                // group slots in order of their first row
		for (int k = 0; k < nlive; ++k) {
			const int i = live[k], j = done[i];
			const SqPlace& q = place[i];
			const bool gr = c.greedy(i);
			int draft[SQ_ROWS], sd[SQ_ROWS]; // the draft, and a constrained request's state before each of its rows
			int nd = 0;
			sd[0] = cur[i];
			if (drafting && c.pen.neutral(i)) {
				nd = vf_lookup(corpus[i], nullptr, 0, imin(imin(c.lk.max_draft, c.max_new[i] - j - 1), nfree), draft);
				// no draft row follows its request's end: the draft stops before a stop token, a token the state disallows
				// and a token that leads to a final state
				for (int d = 0; d < nd; ++d) {
					const int v = draft[d];
					if (is_stop[v] || (sd[d] >= 0 && (!c.aut.allowed(sd[d], v) || c.aut.fin[c.aut.next(sd[d], v)]))) {
						nd = d;
						break;
					}
					sd[d + 1] = sd[d] >= 0 ? c.aut.next(sd[d], v) : -1;
				}
				nfree -= nd;
			}
			s.first[k] = r.n;
			unsigned long long st = hst[i]; // row d draws the coin after the d coins before it
			for (int d = 0; d <= nd; ++d, st = xorshift_step(st)) {
				const int b = r.n++;
				r.q[b] = make_int4(q.s, q.L, q.t, j + d), r.pos[b] = q.L + j + d, r.slot[b] = q.t + j + d;
				r.src[b] = d ? -1 : row_of[i], r.tok0[b] = d ? draft[d - 1] : c.tokens[c.off[i] + c.len[i] - 1];
				// (a greedy row's sampler state is never read back: any valid one will do)
				r.st0[b].rng = gr ? 1 : d ? st : c.rng_states[i], r.st0[b].temperature = gr ? 1.0f : c.temperature[i];
				r.st0[b].cut_delta = gr ? 0.0f : logf(c.minp[i]) * c.temperature[i];
				r.out[b] = (int)(O[i] + j + d), r.req[b] = i, r.greedy[b] = gr;
				s.lanes.lane[b] = lane_of[i], s.lanes.state[b] = sd[d];
				s.pen = s.pen || lane_of[i] >= 0, s.mask = s.mask || sd[d] >= 0, s.mask_sampled = s.mask_sampled || (sd[d] >= 0 && !gr);
				if (c.truncated(i)) s.trows.row[s.ntrunc] = b, s.trows.top_k[s.ntrunc] = c.tr.k(i), s.trows.top_p[s.ntrunc++] = c.tr.p(i);
				s.nsampled += !gr, s.lmax = std::max(s.lmax, q.L + j + d);
				s.grp.ctx[b] = make_int2(q.c, q.nc);
				s.nsuf = std::max(s.nsuf, cdiv(q.L + j + d + 1, SN_CHUNK) - q.nc / SN_CHUNK);
				if (q.nc) {
					if (!groups.count(q.c)) gorder.push_back(q.c);
					groups[q.c].push_back(b);
				}
				s.nx.tok[b] = d < nd ? draft[d] : -1;
			}
		}
		s.first[nlive] = r.n;
		std::fill(s.lanes.lane + r.n, s.lanes.lane + SQ_ROWS, -1), std::fill(s.lanes.state + r.n, s.lanes.state + SQ_ROWS, -1);
		SqGroups& grp = s.grp; // rows with contexts: the groups table of the GROUPS attention
		for (int cs : gorder) {
			const std::vector<int>& rows = groups[cs];
			grp.first[grp.ng + 1] = grp.first[grp.ng] + (int)rows.size();
			grp.chunk0[grp.ng + 1] = grp.chunk0[grp.ng] + grp.ctx[rows[0]].y / SN_CHUNK;
			std::copy(rows.begin(), rows.end(), grp.rows + grp.first[grp.ng]);
			++grp.ng;
		}
		return s;
	}

	// The step's kernels: its tables, the pass over its rows, the classifier and the sampler, and its tokens' stores
	void launch(const SqStep& s) {
		launch_pdl(k_sq_begin, 1, 32, 0, s.r, pf.sqrows, (const int*)pf.sqtok, pf.tokens, pf.vstate);
		if (s.pen || s.mask) launch_pdl(k_sq_lanes, 1, 32, 0, s.lanes, pf.sqlanes);
		PfSampleStep ss = {0, 0, s.r.n, s.lmax};
		if (s.grp.ng) {
			launch_pdl(k_sq_groups, 1, 32, 0, s.grp, pf.sqgroups);
			ss.nshared = s.grp.chunk0[s.grp.ng], ss.nsuf = s.nsuf;
		}
		with_formats([&](auto f) {
			pf_run(f, s.r.n, 0, PF_QUEUE, &ss);
			sq_classify(f, s.r.n, c.lp.k, s.nsampled > 0, s.pen || s.mask, s.mask);
		});
		if (c.lp.on) { // the sampler, then every row's target and the merge, whose argmax is the greedy rows' token
			if (s.nsampled > 0) vf_sample_rows(s.r.n, nullptr, s.mask_sampled, s.ntrunc ? &s.trows : nullptr, s.ntrunc);
			launch_pdl(k_sq_tgt, s.r.n, 32, 0, (const SqRows*)pf.sqrows, (const float2*)pf.part, cdiv(g.cfg.vocab_size, PF_BM), (const float*)pf.vlogits,
			           g.cfg.vocab_size, (const int*)pf.vsampled, pf.tgt);
			sq_merge(s.r.n, c.lp.k);
		} else {
			if (s.nsampled < s.r.n) pf_merge(s.r.n, true, 0); // the greedy rows' argmax
			if (s.nsampled > 0) vf_sample_rows(s.r.n, nullptr, s.mask_sampled, s.ntrunc ? &s.trows : nullptr, s.ntrunc);
		}
		if (s.r.n > (int)live.size()) // a step with draft rows
			launch_pdl(k_sq_accept, 1, 32, 0, (const SqRows*)pf.sqrows, s.nx, (const int*)pf.greedy, (const int*)pf.vsampled, (const SampleState*)pf.vstate,
			           pf.sqtok, pf.sqtok + VF_TOK, pf.sqout, pf.sqst);
		else
			launch_pdl(k_sq_end, 1, 32, 0, (const SqRows*)pf.sqrows, (const int*)pf.greedy, (const int*)pf.vsampled, (const SampleState*)pf.vstate, pf.sqtok, pf.sqout, pf.sqst);
		if (c.lp.on)
			launch_pdl(k_sq_lp, 1, 32, 0, (const SqRows*)pf.sqrows, (const float*)pf.logprob, (const int*)pf.sqtid, (const float*)pf.sqtlp, c.lp.k, pf.sqlp,
			           pf.sqoid, pf.sqolp);
		if (s.pen) launch_pdl(k_sq_pen_step, 1, 32, 0, (const int*)pf.sqlanes, (const int*)pf.sqtok, g.cfg.vocab_size, pf.sqpcnt);
		++nsteps, last_sampled = s.nsampled > 0 ? s.r.n : 0;
	}

	// The step's tokens, read back where they decide stops, the constrained rows' states or the next drafts (with drafts, the
	// emitted flags too), advance each request; one that ends frees its own slots and lane, the others keep their order
	void retire(const SqStep& s) {
		if (c.n_stop || s.mask || drafting) {
			CUDA_CHECK(cudaMemcpyAsync(tok_host, pf.sqtok, (drafting ? 2 * VF_TOK : s.r.n) * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
			sync_stream();
		}
		std::vector<int> keep;
		for (int k = 0; k < (int)live.size(); ++k) {
			const int i = live[k], f = s.first[k], nr = s.first[k + 1] - f;
			int a = 0; // accepted drafts: the request emits its rows 0 .. a
			while (a < nr - 1 && tok_host[f + a] == s.nx.tok[f + a]) ++a;
			for (int d = 1; d < nr; ++d)
				if (tok_host[VF_TOK + f + d] != (d <= a)) CALM_FATAL("%s: row %d's emitted flag disagrees with the step's tokens", c.who, f + d);
			ndrafted += nr - 1, naccepted += a;
			for (int d = 0; d <= a; ++d) {
				++done[i];
				if (cur[i] >= 0) cur[i] = c.aut.next(cur[i], tok_host[f + d]);
				if (drafting) corpus[i].push_back(tok_host[f + d]);
				if (!c.greedy(i)) hst[i] = xorshift_step(hst[i]);
			}
			row_of[i] = f + a;
			if (done[i] < c.max_new[i] && !(c.n_stop && is_stop[tok_host[f + a]]) && !c.aut.ends(cur[i])) {
				keep.push_back(i);
				continue;
			}
			c.out_len[i] = done[i];
			slots.give(place[i].s, cdiv(c.len[i] - 1, 8) * 8), slots.give(place[i].t, c.max_new[i]);
			if (lane_of[i] >= 0) lanes_free |= 1u << lane_of[i], lane_of[i] = -1;
			if (c.aut.out_state) c.aut.out_state[i] = cur[i];
		}
		live.swap(keep);
	}

	// Every request's tokens, final generator state and log-probabilities, copied out, and the call's counts
	void finish(size_t total) {
		std::vector<int> all(total);
		std::vector<unsigned long long> st(c.nreq);
		CUDA_CHECK(cudaMemcpyAsync(all.data(), pf.sqout, total * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
		CUDA_CHECK(cudaMemcpyAsync(st.data(), pf.sqst, c.nreq * sizeof(unsigned long long), cudaMemcpyDeviceToHost, g.stream));
		const size_t k = c.lp.k;
		std::vector<float> lps(c.lp.on ? total : 0), tlp(total * k);
		std::vector<int> tid(total * k);
		if (c.lp.on) {
			CUDA_CHECK(cudaMemcpyAsync(lps.data(), pf.sqlp, total * sizeof(float), cudaMemcpyDeviceToHost, g.stream));
			if (k) {
				CUDA_CHECK(cudaMemcpyAsync(tid.data(), pf.sqoid, total * k * sizeof(int), cudaMemcpyDeviceToHost, g.stream));
				CUDA_CHECK(cudaMemcpyAsync(tlp.data(), pf.sqolp, total * k * sizeof(float), cudaMemcpyDeviceToHost, g.stream));
			}
		}
		sync_stream();
		CUDA_CHECK(cudaGetLastError());
		for (int i = 0; i < c.nreq; ++i) {
			const size_t o = O[i], e = O[i] + c.out_len[i];
			std::copy(all.begin() + o, all.begin() + e, c.out_tokens + o);
			if (c.out_len[i] > 0 && !c.greedy(i)) c.rng_states[i] = st[i];
			if (c.lp.on) { // (slots past out_len[i] are left untouched)
				std::copy(lps.begin() + o, lps.begin() + e, c.lp.logprobs + o);
				std::copy(tid.begin() + o * k, tid.begin() + e * k, c.lp.top_ids + o * k);
				std::copy(tlp.begin() + o * k, tlp.begin() + e * k, c.lp.top_logprobs + o * k);
				if (c.aut.s0(i) >= 0) // the merge's entry past a list's allowed tokens is (-inf, INT_MAX): id -1 there
					for (size_t x = o * k; x < e * k; ++x)
						if (c.lp.top_ids[x] == INT_MAX) c.lp.top_ids[x] = -1;
			}
		}
		if (last_sampled) pf.vrows = last_sampled;
		if (c.steps) *c.steps = nsteps;
		if (c.prompt_rows) *c.prompt_rows = rows_computed;
		if (c.lk.drafted) *c.lk.drafted = ndrafted;
		if (c.lk.accepted) *c.lk.accepted = naccepted;
	}
};

// Every queue call, after its checks, either on the per-request fallback or as a loop of admit -> build -> launch ->
// retire.  Admission runs each round's extent through the packed prompt pass (sb_prefill), each request's own rows
// continuing its context at positions ctx_len ...  A step is one short block over the rows in flight (PF_QUEUE), with
// k_sn_attn's GROUPS variant where rows have contexts; with log-probabilities the TOPK epilogue (k > 0), and the merge
// after the sampler with each row's target set to its token (k_sq_tgt); the PEN classifier where a row is not neutral
// (its lane held from k_sq_pen_admit to retirement, counted by k_sq_pen_step) and MASK where one is constrained, their
// lanes and states kept by k_sq_lanes; the masked and truncating samplers where such rows sample; and k_sq_accept in
// place of k_sq_end where draft rows run.  A step without such rows launches what it would without those options.
static int sq_run(SqCall c) {
	const size_t total = sq_check(c);
	if (c.steps) *c.steps = 0;
	if (c.prompt_rows) *c.prompt_rows = 0;
	if (c.lk.drafted) *c.lk.drafted = 0;
	if (c.lk.accepted) *c.lk.accepted = 0;
	std::vector<int> cur(c.nreq); // a constrained request's automaton state after its tokens so far (-1: unconstrained)
	for (int i = 0; i < c.nreq; ++i) cur[i] = c.aut.s0(i);
	std::vector<char> is_stop(g.cfg.vocab_size, 0);
	for (int k = 0; k < c.n_stop; ++k) is_stop[c.stop[k]] = 1;
	std::vector<size_t> O(c.nreq + 1, 0); // request i's tokens go to out_tokens[O[i] ..]
	for (int i = 0; i < c.nreq; ++i) O[i + 1] = O[i] + c.max_new[i];
	for (int i = 0; i < c.nreq; ++i)
		if (c.max_new[i] == 0) c.out_len[i] = 0; // never admitted
	if (c.aut.out_state) std::copy(cur.begin(), cur.end(), c.aut.out_state); // (each request's final value below)
	if (total == 0) return 1;
	bool fits = true;
	int P = 0, chunks = 0;
	for (int i = 0; i < c.nreq; ++i) {
		if (c.max_new[i] == 0) continue;
		const int Rc = cdiv(c.ctx.len(i), 8) * 8, L = c.ctx.len(i) + c.len[i] - 1;
		fits = fits && (long long)Rc + cdiv(c.len[i] - 1, 8) * 8 + c.max_new[i] <= g.cfg.seq_len;
		P = imin(P + Rc + cdiv(c.len[i] - 1, 8) * 8, SB_BLOCK), chunks = std::max(chunks, cdiv(L + c.max_new[i], SN_CHUNK));
	}
	if (!pf_supported() || !fits) return sq_fallback(c, cur, is_stop, O);
	sn_reserve(std::max(P, VF_TOK), chunks);
	sq_reserve(c, total, cur);
	SqLoop q(c, cur, is_stop, O);
	while (q.admit()) {
		const SqStep s = q.build();
		q.launch(s), q.retire(s);
	}
	q.finish(total);
	return 1;
}

extern "C" int calm_b200_decode_sample_queue(struct Transformer* transformer, const int* tokens, int n, const int* off, const int* len, int nreq,
                                             const int* max_new, const float* temperature, const float* minp, const int* stop, int n_stop,
                                             int max_rows, unsigned long long* rng_states, int* out_tokens, int* out_len, int* steps) {
	return sq_run({"decode_sample_queue", transformer, tokens, n, {nullptr, nullptr}, off, len, nreq, max_new, temperature, minp, stop, n_stop, max_rows,
	                rng_states, out_tokens, out_len, steps, nullptr});
}

extern "C" int calm_b200_decode_sample_queue_context(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                     const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                     const float* minp, const int* stop, int n_stop, int max_rows, unsigned long long* rng_states,
                                                     int* out_tokens, int* out_len, int* steps, int* prompt_rows) {
	return sq_run({"decode_sample_queue_context", transformer, tokens, n, {ctx_off, ctx_len, true}, off, len, nreq, max_new, temperature, minp, stop,
	                n_stop, max_rows, rng_states, out_tokens, out_len, steps, prompt_rows});
}

extern "C" int calm_b200_decode_sample_queue_logprobs(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                      const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                      const float* minp, const int* stop, int n_stop, int max_rows, unsigned long long* rng_states,
                                                      int* out_tokens, int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                                      float* top_logprobs) {
	return sq_run({"decode_sample_queue_logprobs", transformer, tokens, n, {ctx_off, ctx_len}, off, len, nreq, max_new, temperature, minp, stop, n_stop,
	                max_rows, rng_states, out_tokens, out_len, steps, prompt_rows, {true, k, logprobs, top_ids, top_logprobs}});
}

extern "C" int calm_b200_decode_sample_queue_penalties(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                       const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                       const float* minp, const float* presence, const float* frequency, const float* repetition,
                                                       const int* bias_off, const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias,
                                                       const int* stop, int n_stop, int max_rows, unsigned long long* rng_states, int* out_tokens,
                                                       int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                                       float* top_logprobs) {
	return sq_run({"decode_sample_queue_penalties", transformer, tokens, n, {ctx_off, ctx_len}, off, len, nreq, max_new, temperature, minp, stop, n_stop,
	                max_rows, rng_states, out_tokens, out_len, steps, prompt_rows, {logprobs || k, k, logprobs, top_ids, top_logprobs},
	                {presence, frequency, repetition, bias_off, bias_len, bias_ids, bias_val, n_bias}});
}

extern "C" int calm_b200_decode_sample_queue_constrained(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                         const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                         const float* minp, const float* presence, const float* frequency, const float* repetition,
                                                         const int* bias_off, const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias,
                                                         const int* stop, int n_stop, int max_rows, unsigned long long* rng_states, int* out_tokens,
                                                         int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                                         float* top_logprobs, int n_states, const uint32_t* allow, const int* next_default,
                                                         const int* exc_off, const int* exc_tok, const int* exc_next, const int* start, int* out_state) {
	return sq_run({"decode_sample_queue_constrained", transformer, tokens, n, {ctx_off, ctx_len}, off, len, nreq, max_new, temperature, minp, stop, n_stop,
	                max_rows, rng_states, out_tokens, out_len, steps, prompt_rows, {logprobs || k, k, logprobs, top_ids, top_logprobs},
	                {presence, frequency, repetition, bias_off, bias_len, bias_ids, bias_val, n_bias},
	                {n_states, allow, next_default, exc_off, exc_tok, exc_next, start, out_state}});
}

extern "C" int calm_b200_decode_sample_queue_truncated(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                       const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                       const float* minp, const float* presence, const float* frequency, const float* repetition,
                                                       const int* bias_off, const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias,
                                                       const int* stop, int n_stop, int max_rows, unsigned long long* rng_states, int* out_tokens,
                                                       int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                                       float* top_logprobs, int n_states, const uint32_t* allow, const int* next_default,
                                                       const int* exc_off, const int* exc_tok, const int* exc_next, const int* start, int* out_state,
                                                       const int* top_k, const float* top_p) {
	return sq_run({"decode_sample_queue_truncated", transformer, tokens, n, {ctx_off, ctx_len}, off, len, nreq, max_new, temperature, minp, stop, n_stop,
	                max_rows, rng_states, out_tokens, out_len, steps, prompt_rows, {logprobs || k, k, logprobs, top_ids, top_logprobs},
	                {presence, frequency, repetition, bias_off, bias_len, bias_ids, bias_val, n_bias},
	                {n_states, allow, next_default, exc_off, exc_tok, exc_next, start, out_state}, {top_k, top_p}});
}

extern "C" int calm_b200_decode_sample_queue_lookup(struct Transformer* transformer, const int* tokens, int n, const int* ctx_off, const int* ctx_len,
                                                    const int* off, const int* len, int nreq, const int* max_new, const float* temperature,
                                                    const float* minp, const float* presence, const float* frequency, const float* repetition,
                                                    const int* bias_off, const int* bias_len, const int* bias_ids, const float* bias_val, int n_bias,
                                                    const int* stop, int n_stop, int max_rows, unsigned long long* rng_states, int* out_tokens,
                                                    int* out_len, int* steps, int* prompt_rows, int k, float* logprobs, int* top_ids,
                                                    float* top_logprobs, int n_states, const uint32_t* allow, const int* next_default,
                                                    const int* exc_off, const int* exc_tok, const int* exc_next, const int* start, int* out_state,
                                                    const int* top_k, const float* top_p, int max_draft, int* drafted, int* accepted) {
	return sq_run({"decode_sample_queue_lookup", transformer, tokens, n, {ctx_off, ctx_len}, off, len, nreq, max_new, temperature, minp, stop, n_stop,
	                max_rows, rng_states, out_tokens, out_len, steps, prompt_rows, {logprobs || k, k, logprobs, top_ids, top_logprobs},
	                {presence, frequency, repetition, bias_off, bias_len, bias_ids, bias_val, n_bias},
	                {n_states, allow, next_default, exc_off, exc_tok, exc_next, start, out_state}, {top_k, top_p}, {max_draft, drafted, accepted}});
}

// the logits of the last device-resident step (decode_greedy / decode_sample keep them in HBM): copy for tests
// ---------------------------------------------------------------------------------------------
// calm_b200_decode_beam: num_beams beams of one prompt, one short block per step whose rows are the live beams (PF_BEAM),
// the prompt's keys read once per step for all of them and each beam's generated keys through its ancestry
// (sample_n.cuh, BEAM); the classifier's top-K epilogue and merge give each row its K best tokens, and k_bm_select walks
// them into the next beams, the pool and the next ancestry.  Nothing is copied back before the end but, with a stop list,
// the 4-byte done flag after each step.

static_assert(BM_MAX == CALM_B200_BEAM_MAX, "the pool and the sums hold the most beams a call takes");

// a finished hypothesis's tokens and log-probabilities: row `row` of step `step`'s history through the backpointers, then
// its own token if it has one
static void bm_tokens(const std::vector<BmBack>& back, int B, const BmHyp& h, std::vector<int>& tok, std::vector<float>& lp) {
	tok.assign(h.step + (h.token >= 0), 0), lp.assign(tok.size(), 0.0f);
	if (h.token >= 0) tok[h.step] = h.token, lp[h.step] = h.lp;
	for (int s = h.step - 1, r = h.row; s >= 0; --s) {
		const BmBack& b = back[(size_t)s * B + r];
		tok[s] = b.token, lp[s] = b.lp, r = b.parent;
	}
}

extern "C" int calm_b200_decode_beam(struct Transformer* transformer, int token0, int pos0, int max_new, int num_beams, const int* stop, int n_stop,
                                     float length_penalty, int early_stopping, int num_return, int* out_tokens, int* out_len, float* out_logprobs,
                                     float* out_scores, int* steps) {
	if (!g.ready) CALM_FATAL("decode_beam before prepare_cuda");
	const int B = num_beams;
	if (B < 1 || B > CALM_B200_BEAM_MAX) CALM_FATAL("decode_beam: num_beams %d outside [1, %d]", B, CALM_B200_BEAM_MAX);
	if (max_new < 0 || n_stop < 0) CALM_FATAL("decode_beam: negative max_new %d or n_stop %d", max_new, n_stop);
	const long long K = (long long)std::max(2, 1 + n_stop) * B;
	if (K > CALM_B200_TOPK_MAX) CALM_FATAL("decode_beam: %lld candidates per beam (max(2, 1 + n_stop) x num_beams) exceed %d", K, CALM_B200_TOPK_MAX);
	if (num_return < 1 || num_return > B) CALM_FATAL("decode_beam: num_return %d outside [1, %d]", num_return, B);
	if (n_stop > 0 && !stop) CALM_FATAL("decode_beam: stop is NULL");
	for (int i = 0; i < n_stop; ++i)
		if (stop[i] < 0 || stop[i] >= g.cfg.vocab_size) CALM_FATAL("decode_beam: stop token %d out of range", stop[i]);
	if (!std::isfinite(length_penalty)) CALM_FATAL("decode_beam: length_penalty is not finite");
	if (early_stopping != 0 && early_stopping != 1) CALM_FATAL("decode_beam: early_stopping %d is not 0 or 1", early_stopping);
	if (!out_tokens || !out_len || !out_scores || !steps) CALM_FATAL("decode_beam: out_tokens, out_len, out_scores or steps is NULL");
	check_call(transformer, token0, pos0);
	if (max_new == 0) return 1;
	if (!pf_supported() || (long long)pos0 + (long long)B * max_new > g.cfg.seq_len) {
		*steps = 0;
		return 0;
	}
	sn_reserve(B, cdiv(pos0 + max_new, SN_CHUNK));
	sq_topk_reserve();
	const size_t nanc = (size_t)B * max_new, nback = (size_t)max_new * B, ntrace = nback * K;
	if (!pf.bmst) pf.bmst = (BmState*)dev_alloc(sizeof(BmState));
	sq_grow(pf.bmanc_cap, nanc, pf.bmanc[0], pf.bmanc[1]);
	sq_grow(pf.bmback_cap, nback, pf.bmback);
	sq_grow(pf.bmtrace_cap, ntrace, pf.bmtid, pf.bmtlp);
	std::vector<float> norm(max_new + 1); // norm[L] = L^length_penalty, in double, rounded once
	for (int L = 1; L <= max_new; ++L) norm[L] = (float)pow((double)L, (double)length_penalty);
	std::vector<int> pos(nanc);
	for (size_t r = 0; r < nanc; ++r) pos[r] = pos0 + (int)(r / B); // step j's rows at [j B, j B + rows)
	CUDA_CHECK(cudaMemcpyAsync(pf.snpos, pos.data(), nanc * sizeof(int), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaMemcpyAsync(pf.tokens, &token0, sizeof(int), cudaMemcpyHostToDevice, g.stream));
	CUDA_CHECK(cudaMemsetAsync(pf.bmanc[0], 0, nanc * sizeof(int), g.stream)); // step 0's one row reads its own key
	CUDA_CHECK(cudaMemsetAsync(pf.bmst, 0, sizeof(BmState), g.stream));
	BmArgs ba = {};
	ba.tid = pf.sqtid, ba.tlp = pf.sqtlp, ba.st = pf.bmst, ba.back = pf.bmback, ba.trace_id = pf.bmtid, ba.trace_lp = pf.bmtlp, ba.tokens = pf.tokens;
	std::copy(stop, stop + n_stop, ba.stop);
	ba.n_stop = n_stop, ba.B = B, ba.K = (int)K, ba.max_new = max_new, ba.early = early_stopping;
	int done = 0, j = 0, cur = 0;
	for (; j < max_new && !done; ++j, cur ^= 1) {
		const int rows = j ? B : 1;
		PfSampleStep ss = {pos0, j, rows, 0};
		ss.anc = pf.bmanc[cur], ss.nbeam = B, ss.anc_stride = max_new;
		with_formats([&](auto f) {
			pf_run(f, rows, pos0 + j * B, PF_BEAM, &ss);
			sq_classify(f, rows, (int)K, false, false, false);
		});
		sq_merge(rows, (int)K);
		ba.anc = pf.bmanc[cur], ba.anc_next = pf.bmanc[cur ^ 1], ba.j = j, ba.rows = rows;
		ba.norm_j = norm[std::max(1, j)], ba.norm_next = norm[j + 1];
		launch_pdl(k_bm_select, 1, BM_THREADS, 0, ba);
		if (n_stop) {
			CUDA_CHECK(cudaMemcpyAsync(&done, &pf.bmst->done, sizeof(int), cudaMemcpyDeviceToHost, g.stream));
			sync_stream();
		}
	}
	pf.bm_steps = j, pf.bm_beams = B, pf.bm_k = (int)K, pf.bm_max_new = max_new, pf.bm_last = cur ^ 1;
	BmState st;
	std::vector<BmBack> back((size_t)j * B);
	CUDA_CHECK(cudaMemcpyAsync(&st, pf.bmst, sizeof(BmState), cudaMemcpyDeviceToHost, g.stream));
	CUDA_CHECK(cudaMemcpyAsync(back.data(), pf.bmback, back.size() * sizeof(BmBack), cudaMemcpyDeviceToHost, g.stream));
	sync_stream();
	CUDA_CHECK(cudaGetLastError());
	if (!st.done) // the live beams, in beam order, after the last step
		for (int b = 0; b < B; ++b) bm_add(st, B, BmHyp{st.sum[b] / norm[max_new], st.sum[b], 0.0f, max_new, b, -1, 0});
	std::sort(st.pool, st.pool + st.npool, [](const BmHyp& x, const BmHyp& y) { return x.score > y.score || (x.score == y.score && x.order < y.order); });
	std::vector<int> tok;
	std::vector<float> lp;
	for (int r = 0; r < num_return && r < st.npool; ++r) {
		bm_tokens(back, B, st.pool[r], tok, lp);
		std::copy(tok.begin(), tok.end(), out_tokens + (size_t)r * max_new);
		if (out_logprobs) std::copy(lp.begin(), lp.end(), out_logprobs + (size_t)r * max_new);
		out_len[r] = (int)tok.size(), out_scores[r] = st.pool[r].score;
	}
	*steps = j;
	return 1;
}

extern "C" void calm_b200_read_device_logits(float* out) {
	CUDA_CHECK(cudaMemcpy(out, g.logits_dev, (size_t)g.cfg.vocab_size * sizeof(float), cudaMemcpyDeviceToHost));
}

extern "C" void calm_b200_timer_start(void) {
	CUDA_CHECK(cudaEventRecord(g.timer[0], g.stream));
}

extern "C" float calm_b200_timer_stop(void) {
	CUDA_CHECK(cudaEventRecord(g.timer[1], g.stream));
	CUDA_CHECK(cudaEventSynchronize(g.timer[1]));
	float ms = 0;
	CUDA_CHECK(cudaEventElapsedTime(&ms, g.timer[0], g.timer[1]));
	return ms;
}

extern "C" void* calm_b200_stream(void) {
	return (void*)g.stream;
}

extern "C" uint64_t calm_b200_launch_count(void) {
	return g_launches;
}

extern "C" void calm_b200_read_kv(struct Transformer* transformer, int layer, int kv_pos, float* k_out, float* v_out) {
	(void)transformer;
	const Config& c = g.cfg;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	size_t es = g.kvbits / 8;
	std::vector<unsigned char> kb(c.head_dim * es), vb(c.head_dim * es);
	for (int h = 0; h < c.n_kv_heads; ++h) {
		size_t off = (((size_t)layer * c.n_kv_heads + h) * c.seq_len + kv_pos) * c.head_dim * es;
		CUDA_CHECK(cudaMemcpy(kb.data(), (char*)g.kc + off, kb.size(), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(vb.data(), (char*)g.vc + off, vb.size(), cudaMemcpyDeviceToHost));
		for (int d = 0; d < c.head_dim; ++d) {
			float kf, vf;
			if (es == 2) {
				kf = __half2float(((__half*)kb.data())[d]);
				vf = __half2float(((__half*)vb.data())[d]);
			} else {
				kf = __half2float(__ushort_as_half((unsigned short)(kb[d] << 8)));
				vf = __half2float(__ushort_as_half((unsigned short)(vb[d] << 8)));
			}
			k_out[h * c.head_dim + d] = kf;
			v_out[h * c.head_dim + d] = vf;
		}
	}
}

// (test aid) One engine buffer as floats, after the stream has drained; see include/calm_b200.h for the selectors.
extern "C" int calm_b200_read_state(int which, int layer, float* out, int cap) {
	if (!g.ready) CALM_FATAL("read_state before prepare_cuda");
	const Config& c = g.cfg;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	const float* f32 = nullptr;           // a float buffer, copied as it is
	const __half *hi = nullptr, *lo = nullptr; // a prompt-pass activation pair, summed in float
	const int* i32 = nullptr;                 // an int buffer, converted to float
	size_t count = 0;
	switch (which) {
	case CALM_B200_STATE_X: f32 = g.x, count = c.dim; break;
	case CALM_B200_STATE_XB: f32 = g.xb, count = c.dim; break;
	case CALM_B200_STATE_Q: f32 = g.q, count = g.q_dim; break;
	case CALM_B200_STATE_ATT: f32 = g.att, count = g.q_dim; break;
	case CALM_B200_STATE_HB: f32 = g.hb, count = (size_t)g.nact * c.hidden_dim; break;
	case CALM_B200_STATE_MOE_SEL: count = 2 * (size_t)g.nact; break;
	case CALM_B200_STATE_KEYS:
	case CALM_B200_STATE_VALUES:
		if (layer < 0 || layer >= c.n_layers) CALM_FATAL("read_state: layer %d out of range", layer);
		count = (size_t)c.n_kv_heads * c.seq_len * c.head_dim;
		break;
	case CALM_B200_STATE_PF_X: f32 = pf.X, count = (size_t)pf.cap * c.dim; break;
	case CALM_B200_STATE_PF_Q: f32 = pf.Q, count = (size_t)pf.cap * g.q_dim; break;
	case CALM_B200_STATE_PF_ATT: hi = pf.Ahi, lo = pf.Alo, count = (size_t)pf.cap * g.q_dim; break;
	case CALM_B200_STATE_PF_HB: hi = pf.Hhi, lo = pf.Hlo, count = (size_t)pf.cap * c.hidden_dim; break;
	case CALM_B200_STATE_PF_LOGITS: f32 = pf.vlogits, count = (size_t)pf.vrows * c.vocab_size; break;
	case CALM_B200_STATE_BEAM_IDS: i32 = pf.bmtid, count = (size_t)pf.bm_steps * pf.bm_beams * pf.bm_k; break;
	case CALM_B200_STATE_BEAM_LOGPROBS: f32 = pf.bmtlp, count = (size_t)pf.bm_steps * pf.bm_beams * pf.bm_k; break;
	case CALM_B200_STATE_BEAM_ANC: i32 = pf.bmanc[pf.bm_last], count = (size_t)pf.bm_beams * pf.bm_max_new; break;
	default: CALM_FATAL("read_state: unknown selector %d", which);
	}
	if (count > 0x7fffffff) CALM_FATAL("read_state: %zu values do not fit the int the call returns", count);
	if (!out || (size_t)cap < count || count == 0) return (int)count; // (no prompt pass yet: its matrices are empty)
	if (f32) {
		CUDA_CHECK(cudaMemcpy(out, f32, count * sizeof(float), cudaMemcpyDeviceToHost));
	} else if (i32) {
		std::vector<int> v(count);
		CUDA_CHECK(cudaMemcpy(v.data(), i32, count * sizeof(int), cudaMemcpyDeviceToHost));
		for (size_t i = 0; i < count; ++i) out[i] = (float)v[i];
	} else if (hi) {
		std::vector<__half> h(count), l(count);
		CUDA_CHECK(cudaMemcpy(h.data(), hi, count * sizeof(__half), cudaMemcpyDeviceToHost));
		CUDA_CHECK(cudaMemcpy(l.data(), lo, count * sizeof(__half), cudaMemcpyDeviceToHost));
		for (size_t i = 0; i < count; ++i) out[i] = __half2float(h[i]) + __half2float(l[i]);
	} else if (which == CALM_B200_STATE_MOE_SEL) {
		MoeSel sel;
		CUDA_CHECK(cudaMemcpy(&sel, g.moe_sel, sizeof(sel), cudaMemcpyDeviceToHost));
		for (int k = 0; k < g.nact; ++k) out[k] = (float)sel.expert[k], out[g.nact + k] = sel.weight[k];
	} else { // one layer of the cache, [n_kv_heads][seq_len][head_dim]: halves, or e5m2 bytes (the high byte of a half)
		const size_t es = g.kvbits / 8;
		std::vector<unsigned char> raw(count * es);
		const char* base = (const char*)(which == CALM_B200_STATE_KEYS ? g.kc : g.vc) + (size_t)layer * count * es;
		CUDA_CHECK(cudaMemcpy(raw.data(), base, raw.size(), cudaMemcpyDeviceToHost));
		for (size_t i = 0; i < count; ++i)
			out[i] = es == 2 ? __half2float(((const __half*)raw.data())[i]) : __half2float(__ushort_as_half((unsigned short)(raw[i] << 8)));
	}
	return (int)count;
}

extern "C" void calm_b200_fill_kv(struct Transformer* transformer, int n_pos, uint64_t seed) {
	(void)transformer;
	const Config& c = g.cfg;
	size_t lh = (size_t)c.n_layers * c.n_kv_heads;
	if (n_pos > c.seq_len) n_pos = c.seq_len;
	if (g.kvbits == 8)
		k_fill_kv<uint8_t><<<g.sms * 4, 256, 0, g.stream>>>((uint8_t*)g.kc, (uint8_t*)g.vc, lh, c.seq_len, c.head_dim, n_pos, seed);
	else
		k_fill_kv<__half><<<g.sms * 4, 256, 0, g.stream>>>((__half*)g.kc, (__half*)g.vc, lh, c.seq_len, c.head_dim, n_pos, seed);
	++g_launches;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
}

// (test aid) 0xFF bytes (NaN as f32, f16 and e5m2) into every buffer whose previous contents no later call may depend on,
// and into the cache slots [kv_from_pos, seq_len) of every layer and kv head.  Only data is touched: TokenParams, the
// attention's {value, epoch} cells and counter, k_vf_gemm's arrival counters, the tensor-parallel exchange area, moe_sel, the sampler's state and survivor
// counts (the decode's and the sampled short block's), stamps, the watchdog words, the weights and rope_freq steer control flow, waits or addresses and stay as they are,
// as do the index buffers (cand_idx, sample_idx, pf.vsidx, out_tokens, pf.tokens, pf.targets, pf.rowpos, pf.seg and pf.ctx, read
// as a RoPE position and as key slots of the packed attention's loop, pf.sbrows, decode_sample_batch's key slots and
// chunk counts, pf.sqrows, decode_sample_queue's row table, and pf.sqgroups, its context groups): a stale index that is read is in range,
// as after any earlier call, while 0xFFFFFFFF would send the read out of bounds.  DESIGN.md s.3 lists both groups.
extern "C" void calm_b200_poison_state(struct Transformer* transformer, int kv_from_pos) {
	(void)transformer;
	if (!g.ready) CALM_FATAL("poison_state before prepare_cuda");
	if (kv_from_pos < 0) CALM_FATAL("poison_state: negative position");
	const Config& c = g.cfg;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	auto nan = [](void* p, size_t bytes) {
		if (p) CUDA_CHECK(cudaMemsetAsync(p, 0xFF, bytes, g.stream));
	};
	nan(g.x, c.dim * sizeof(float)), nan(g.xb, c.dim * sizeof(float)), nan(g.xpart, c.dim * sizeof(float));
	nan(g.q, g.q_dim * sizeof(float)), nan(g.att, g.q_dim * sizeof(float));
	nan(g.hb, (size_t)g.nact * c.hidden_dim * sizeof(float));
	nan(g.logits_dev, (size_t)c.vocab_size * sizeof(float));
	nan(g.attn_partial, (size_t)c.n_kv_heads * g.attn_qgroups * g.attn_nsplit * g.attn_hg * (c.head_dim + 2) * sizeof(float));
	nan(g.cand_val, g.ncand * sizeof(float));
	nan(g.rope_cs, (size_t)(c.head_dim / 2) * sizeof(float2));
	nan(g.sample_prob, (size_t)g.sample_chunks * SAMPLE_CHUNK * sizeof(float)), nan(g.sample_csum, g.sample_chunks * sizeof(float));
	if (pf.cap) { // every row of the prompt pass's matrices, the padding rows of a partial token tile included
		const size_t cap = pf.cap;
		nan(pf.X, cap * c.dim * sizeof(float)), nan(pf.Q, cap * g.q_dim * sizeof(float));
		nan(pf.Nhi, cap * c.dim * sizeof(__half)), nan(pf.Nlo, cap * c.dim * sizeof(__half));
		nan(pf.Ahi, cap * g.q_dim * sizeof(__half)), nan(pf.Alo, cap * g.q_dim * sizeof(__half));
		nan(pf.Hhi, cap * c.hidden_dim * sizeof(__half)), nan(pf.Hlo, cap * c.hidden_dim * sizeof(__half));
		nan(pf.rope, cap * (c.head_dim / 2) * sizeof(float2));
		if (pf.scoring) nan(pf.part, cap * cdiv(c.vocab_size, PF_BM) * sizeof(float2)), nan(pf.tgt, cap * sizeof(float)), nan(pf.logprob, cap * sizeof(float));
		// the argmax records are vocabulary indices, but only ever compared and copied out, never used as an address
		nan(pf.gidx, cap * cdiv(c.vocab_size, PF_BM) * sizeof(int)), nan(pf.greedy, cap * sizeof(int));
		// so are the top-k records: ids only compared and copied out, values NaN like every other float
		nan(pf.topv, cap * cdiv(c.vocab_size, PF_BM) * PF_TOPK_MAX * sizeof(float)), nan(pf.topi, cap * cdiv(c.vocab_size, PF_BM) * PF_TOPK_MAX * sizeof(int));
		nan(pf.top_ids, cap * PF_TOPK_MAX * sizeof(int)), nan(pf.top_lp, cap * PF_TOPK_MAX * sizeof(float));
		nan(pf.vacc, pf.vacc_floats * sizeof(float)); // (pf.vcnt, the short-block GEMM's arrival counters, steer control flow)
		// the sampled block's logit rows, tile maxima, survivor probabilities and chunk sums, and its tokens (only copied out);
		// its survivor counts and SampleStates steer the sampler like sample_count / sample_state, and pf.vsidx is an index buffer
		const size_t nch = g.sample_chunks;
		nan(pf.vlogits, VF_TOK * (size_t)c.vocab_size * sizeof(float)), nan(pf.vtmax, VF_TOK * (size_t)cdiv(c.vocab_size, PF_BM) * sizeof(float));
		nan(pf.vsprob, VF_TOK * nch * SAMPLE_CHUNK * sizeof(float)), nan(pf.vcsum, VF_TOK * nch * sizeof(float)), nan(pf.vsampled, VF_TOK * sizeof(int));
		// decode_sample_n's chunk partials and step tokens, which every call writes before it reads them (its positions,
		// read as RoPE positions, are an index buffer)
		nan(pf.snpart, (size_t)VF_TOK * c.n_heads * pf.snchunks * (c.head_dim + 2) * sizeof(float)), nan(pf.sntok, (size_t)c.seq_len * sizeof(int));
		// decode_sample_queue's step tokens and per-request tokens and states, which every call writes before it reads them
		// (its row table, read as positions and key slots, is an index buffer)
		nan(pf.sqtok, 2 * VF_TOK * sizeof(int)), nan(pf.sqout, pf.sqout_cap * sizeof(int)), nan(pf.sqst, pf.sqst_cap * sizeof(unsigned long long));
		// and its log-probability call's tile lists, merged top-k and per-request outputs (ids only compared and copied out)
		const size_t nvt = cdiv(c.vocab_size, PF_BM);
		nan(pf.sqtopv, VF_TOK * nvt * PF_TOPK_MAX * sizeof(float)), nan(pf.sqtopi, VF_TOK * nvt * PF_TOPK_MAX * sizeof(int));
		nan(pf.sqtid, VF_TOK * PF_TOPK_MAX * sizeof(int)), nan(pf.sqtlp, VF_TOK * PF_TOPK_MAX * sizeof(float));
		nan(pf.sqlp, pf.sqlp_cap * sizeof(float)), nan(pf.sqoid, pf.sqtop_cap * sizeof(int)), nan(pf.sqolp, pf.sqtop_cap * sizeof(float));
		// decode_beam's candidate lists, backpointers and pool, which every call writes before it reads them (its ancestry
		// tables, read as key slots, are index buffers)
		nan(pf.bmtid, pf.bmtrace_cap * sizeof(int)), nan(pf.bmtlp, pf.bmtrace_cap * sizeof(float)), nan(pf.bmback, pf.bmback_cap * sizeof(BmBack));
		nan(pf.bmst, sizeof(BmState));
		// and its penalty call's lanes, which k_sq_pen_admit rewrites whole for each request it admits (a poisoned count
		// word reads as seen with count 0x3fffffff), and its uploaded bias values (the uploaded tokens and bias ids and the
		// step's lanes, pf.sqlanes, read as addresses into the lanes, are index buffers)
		nan(pf.sqpcnt, SQ_ROWS * (size_t)c.vocab_size * sizeof(int)), nan(pf.sqpbias, SQ_ROWS * (size_t)c.vocab_size * sizeof(float));
		nan(pf.sqppar, SQ_ROWS * sizeof(float4)), nan(pf.sqpbval, pf.sqpb_cap * sizeof(float));
		// and its constrained call's uploaded automaton, which every such call rewrites before a step reads it (a poisoned
		// word allows every token of its 32)
		nan(pf.sqallow, pf.sqallow_cap * sizeof(uint32_t));
	}
	if (kv_from_pos < c.seq_len) { // the cache is [layer][kv head][seq_len][head_dim]: the tail of every (layer, head) row
		const size_t slot = (size_t)c.head_dim * (g.kvbits / 8), pitch = c.seq_len * slot, width = (c.seq_len - kv_from_pos) * slot;
		for (void* cache : {g.kc, g.vc})
			CUDA_CHECK(cudaMemset2DAsync((char*)cache + kv_from_pos * slot, pitch, 0xFF, width, (size_t)c.n_layers * c.n_kv_heads, g.stream));
	}
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
}

template <int DBITS>
static float matvec_impl(const void* w_device, const float* x_host, float* y_host, int n, int d, int warmup, int iters) {
	cudaStream_t st;
	CUDA_CHECK(cudaStreamCreate(&st));
	float *x, *y;
	CUDA_CHECK(cudaMalloc(&x, n * sizeof(float)));
	CUDA_CHECK(cudaMalloc(&y, d * sizeof(float)));
	CUDA_CHECK(cudaMemcpy(x, x_host, n * sizeof(float), cudaMemcpyHostToDevice));
	cudaDeviceProp prop;
	CUDA_CHECK(cudaGetDeviceProperties(&prop, g.device));
	g.sms = prop.multiProcessorCount;
	size_t smem = xs_bytes<DBITS>(n);
	int cap = max_ctas(k_matvec<DBITS>, 256, smem);
	int grid = imin(cap, cdiv((d + 1) / 2, 8));
	MatvecArgs a{x, w_device, y, n, d};
	cudaEvent_t e0, e1;
	CUDA_CHECK(cudaEventCreate(&e0));
	CUDA_CHECK(cudaEventCreate(&e1));
	for (int i = 0; i < warmup; ++i) k_matvec<DBITS><<<grid, 256, smem, st>>>(a);
	CUDA_CHECK(cudaEventRecord(e0, st));
	for (int i = 0; i < iters; ++i) k_matvec<DBITS><<<grid, 256, smem, st>>>(a);
	CUDA_CHECK(cudaEventRecord(e1, st));
	CUDA_CHECK(cudaEventSynchronize(e1));
	CUDA_CHECK(cudaGetLastError());
	g_launches += warmup + iters;
	float ms = 0;
	CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
	CUDA_CHECK(cudaMemcpy(y_host, y, d * sizeof(float), cudaMemcpyDeviceToHost));
	cudaFree(x), cudaFree(y), cudaEventDestroy(e0), cudaEventDestroy(e1), cudaStreamDestroy(st);
	return iters > 0 ? ms / iters : 0.f;
}

extern "C" float calm_b200_matvec(int dbits, const void* w_device, const float* x_host, float* y_host, int n, int d, int warmup, int iters) {
	select_device();
	if (n % 32) CALM_FATAL("matvec: n must be a multiple of 32");
	switch (dbits) {
	case 16: return matvec_impl<16>(w_device, x_host, y_host, n, d, warmup, iters);
	case 8: return matvec_impl<8>(w_device, x_host, y_host, n, d, warmup, iters);
	case 4: return matvec_impl<4>(w_device, x_host, y_host, n, d, warmup, iters);
	}
	CALM_FATAL("matvec: unsupported dbits %d", dbits);
	return 0.f;
}

// Pull the in-kernel launch stamps (summed on the device by k_stamp_accum) into the per-stage tables.
static void perf_collect() {
	if (!g.stamp_acc) return;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	std::vector<unsigned long long> acc(MAX_STAMPS + 2);
	CUDA_CHECK(cudaMemcpy(acc.data(), g.stamp_acc, acc.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
	for (int i = 0; i < ST_COUNT; ++i) g.stage_ms[i] = 0;
	for (int i = 0; i < MAX_STAMPS; ++i) g.stage_ms[g.stamp_stage[i]] += (double)acc[i] / 1e6;
	g.token_span_ms = (double)acc[MAX_STAMPS] / 1e6;
}

extern "C" void calm_b200_set_perf(int on) {
	if (!g.ready) return;
	if (!on) perf_collect();
	g.perf = on != 0;
	if (!on) return;
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	CUDA_CHECK(cudaMemset(g.stamp_acc, 0, (size_t)(MAX_STAMPS + 2) * sizeof(unsigned long long)));
	for (int i = 0; i < ST_COUNT; ++i) g.stage_ms[i] = 0, g.stage_bytes[i] = 0, g.stage_launches[i] = 0;
	g.perf_runs = 0, g.token_span_ms = 0;
}

extern "C" int calm_b200_stage_stats(int stage, char* name, int name_cap, double* ms_total, double* bytes_total, long* launches) {
	if (stage < 0 || stage >= ST_COUNT) return 0;
	if (name && name_cap > 0) {
		strncpy(name, kStageNames[stage], name_cap - 1);
		name[name_cap - 1] = 0;
	}
	if (g.perf) perf_collect();
	*ms_total = g.stage_ms[stage], *bytes_total = g.stage_bytes[stage], *launches = g.stage_launches[stage];
	return 1;
}

// (debug) the 16 in-kernel timestamps the middle layer's attention kernel left during the last profiled token
extern "C" void calm_b200_debug_stamps(unsigned long long* out16) {
	CUDA_CHECK(cudaStreamSynchronize(g.stream));
	CUDA_CHECK(cudaMemcpy(out16, g.stamps + 2 * (size_t)MAX_STAMPS, 16 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
}

extern "C" double calm_b200_perf_token_ms(void) {
	if (g.perf) perf_collect();
	return g.perf_runs ? g.token_span_ms / g.perf_runs : 0.0;
}

extern "C" void perf_cuda(void) {
	if (!g.ready || !g.perf || g.perf_runs == 0) return;
	perf_collect();
	double total = 0;
	for (int i = 0; i < ST_COUNT; ++i) total += g.stage_ms[i];
	if (total <= 0) return;
	// same shape as the reference's table (infer.cu:761-801); times are first-CTA-start to last-CTA-end of every launch of
	// the production CUDA graph, read from %globaltimer inside the kernels
	printf("\nforward breakdown (over %d runs, avg %.1f usec/run; token span %.1f usec):\n", g.perf_runs, total / g.perf_runs * 1e3, g.token_span_ms / g.perf_runs * 1e3);
	for (int i = 0; i < ST_COUNT; ++i) {
		if (g.stage_ms[i] == 0) continue;
		printf("\t[%d] %16s: %4.1f%%; %8.1f usec/run, %6.1f GB/s\n", i, kStageNames[i], g.stage_ms[i] / total * 100, g.stage_ms[i] / g.perf_runs * 1e3,
		       g.stage_bytes[i] / 1e9 / (g.stage_ms[i] / 1e3));
	}
	fflush(stdout);
}
