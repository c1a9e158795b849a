// encoder.cu -- host side of the FLAC block encoder + its C ABI (include/flac_b200.h).
//
// The host does what the reference does once per (encoder, blocksize): validate settings
// (init_stream_internal_, src/libFLAC/stream_encoder.c:725-830), generate the apodization
// tables with the HOST libm's cosf exactly as src/libFLAC/window.c:195-220 does (CUDA's
// cosf is not bit-identical to glibc's: SURVEY.md §0.4) and expand the apodization
// state machine (apply_apodization_, :4318-4392) into a static list of autocorrelation
// sections and LPC candidates. Everything per block runs in the kernels.
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <vector>

#include "fb200_internal.h"
#include "windows.h"

namespace fb200 {

static thread_local char g_err[512] = "";
void set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}
const char *get_error() { return g_err; }

struct Geometry {
	int bs = 0;
	EncK k{};
	float *d_windows = nullptr;
	float *d_secwin = nullptr;  // per-section weight tables over absolute sample indices (k_autoc4), stride bs + kSecwinSlack
	bool raw_pipeline = false;  // k_meta -> k_autoc4 -> k_lpc -> k_search5 -> k_emit3: every kernel reads the caller's PCM
	DevSection *d_secs = nullptr;
	DevCand *d_cands = nullptr;
	size_t search_smem = 0, emit_smem = 0;  // general kernels
	int fast_search3 = 0;       // 0, or R_T (32/36) of the fast search kernel (k_search5: CTA per block, warps per signal)
	int search_wps = 2;         // warps per signal in k_search5
	size_t search5_smem = 0;
	int maxord_t = 8;
	int emit3_rt = 0;           // 0, or R_T of the resident emit kernel (k_emit3)
	int or_sec = -1;            // a full-length analysis section (k_autoc4 collects the wasted-bits OR there), or -1
	bool emit3_pair = false;    // more than two channels: k_emit3<PAIR> per channel pair + k_join per frame
	int pair_words = 0;         // words of a pair's staging region
	size_t pair_smem = 0, join_smem = 0;
	size_t emit3_smem = 0;
};

}  // namespace fb200

using namespace fb200;

struct fb200_encoder {
	fb200_encoder_config cfg;  // resolved
	int device = 0;
	uint32_t max_blocks = 0;
	std::map<int, Geometry> geoms;
	// workspaces (sized for max_blocks blocks of cfg.blocksize)
	int nsig = 0;
	int32_t *d_sig = nullptr;
	SigMeta *d_meta = nullptr;
	uint32_t *d_sigor = nullptr;  // per (block, signal): OR of the samples, written by k_autoc4 (fused wasted-bits detection)
	int *d_blkflags = nullptr;
	double *d_autoc = nullptr;
	CandDesc *d_cdesc = nullptr;
	SubframePlan *d_plans = nullptr;
	uint8_t *d_slots = nullptr;
	uint32_t *d_frame_bytes = nullptr;
	uint32_t *d_chan_assign = nullptr;
	unsigned long long *d_running = nullptr;  // [2]: k_emit3 reads [run_cur] and writes [run_cur ^ 1]; k_scan updates [run_cur] in place
	int run_cur = 0;
	int *d_err = nullptr;
	uint32_t *d_stage = nullptr, *d_stage_bits = nullptr;  // channel-pair staging of the > 2 channel emit path
	size_t d_stage_words = 0;
	int *d_redo = nullptr;  // [max_blocks] limit_min_bitrate: blocks whose last channel is searched again with constants off
	// k_emit3: slicing tables, look-back status words, frame tickets
	uint16_t *d_crc_tab = nullptr;
	unsigned long long *d_lookback = nullptr;
	unsigned *d_ticket = nullptr;
	unsigned ticket_base = 0, epoch = 0;
	uint32_t file_blocks = 0;

	size_t max_nsec = 0, max_nslots = 0, lag_stride = 0;
	// stage-A outputs are double-buffered so that stage A (prep/autoc/lpc) of sub-batch i+1 can run on
	// s_a concurrently with stage B (search/emit/scan/gather) of sub-batch i on the caller's stream
	struct WS { int32_t *d_sig; SigMeta *d_meta; int *d_blkflags; double *d_autoc; CandDesc *d_cdesc; uint32_t *d_sigor; } ws[2] = {};
	cudaStream_t s_a = nullptr, s_meta = nullptr;
	// slice mode (the call's blocks fit the workspace): every chunk owns its slice of workspace set 0, so the stage A's of
	// different chunks are independent and rotate over these streams (s_as[0] == s_a) -- the latency-bound autocorrelation of
	// a small chunk no longer serialises the pipeline
	static constexpr int kStageAStreams = 4;
	cudaStream_t s_as[kStageAStreams] = {};
	bool slice_mode = false;
	std::vector<cudaEvent_t> ev_ca;  // per chunk: stage A done
	cudaEvent_t ev_meta_fork = nullptr, ev_meta_done = nullptr;
	cudaEvent_t ev_fork = nullptr, ev_a[2] = {nullptr, nullptr}, ev_b[2] = {nullptr, nullptr};
	bool ev_b_valid[2] = {false, false};
	// staging for the host entry point
	int32_t *d_pcm = nullptr;
	size_t d_pcm_cap = 0;
	uint8_t *d_packed = nullptr;  // packed 16-/24-bit input of fb200_encode_host_packed
	size_t d_packed_cap = 0;
	uint8_t *d_out = nullptr;
	size_t d_out_cap = 0;
	unsigned long long *d_offsets = nullptr;
	size_t d_offsets_cap = 0;
	cudaStream_t stream = nullptr, s_h2d = nullptr, s_d2h = nullptr;
	std::vector<cudaEvent_t> ev_h2d, ev_comp;
	unsigned long long *h_totals = nullptr;  // pinned
	size_t h_totals_cap = 0;
	uint64_t launches = 0;
	int host_chunks = 12;   // chunks per fb200_encode_host call (FB200_HOST_CHUNKS): copy/compute overlap granularity; on an H100 SXM at 400 W
	                        // (tools/sweep_host_chunks.py, packed 16-bit, 10 000 blocks) 8-16 are equal within noise and 4 / 24 are ~7 % slower at -8
	int pipe_chunks = 1;    // sub-batches per fb200_encode_device call (FB200_PIPE_CHUNKS); see fb200_encode_device
	int f64b = 0;         // FB200_SEARCH_F64B=1: the second warp of a signal runs on the FP64 pipe (slower: H100 SXM at 400 W, -8, 10 000 blocks: 4.48 vs 3.89 ms per step; kept for A/B)
	int debug_path = 0;   // FB200_DEBUG_PATH bit mask (bisecting aid): 1 = k_prep + k_autoc3 instead of k_autoc4, 2 = general search, 4 = general emit, 8 = k_meta instead of the OR fused into k_autoc4
	bool use_v1 = false;  // FB200_FORCE_GENERAL_KERNELS=1: run the general kernels for every blocksize (tests)
	// optional per-kernel CUDA-event timing (bench.py's roofline numbers)
	bool prof_on = false;
	std::vector<cudaEvent_t> prof_events;   // consecutive events; kernel id of the interval ending at event i in prof_ids[i]
	std::vector<int> prof_ids;              // -1 = interval start
	double prof_ms[FB200_PROF_KERNELS] = {0};
	uint64_t prof_launches[FB200_PROF_KERNELS] = {0};
};

static void prof_mark(fb200_encoder *e, int id, cudaStream_t st)
{
	if(!e->prof_on) return;
	cudaEvent_t ev;
	if(cudaEventCreate(&ev) != cudaSuccess) return;
	cudaEventRecord(ev, st);
	e->prof_events.push_back(ev);
	e->prof_ids.push_back(id);
}

static void prof_resolve(fb200_encoder *e)
{
	for(size_t i = 0; i < e->prof_events.size(); i++) {
		if(e->prof_ids[i] >= 0 && i > 0) {
			float ms = 0.f;
			cudaEventSynchronize(e->prof_events[i]);
			if(cudaEventElapsedTime(&ms, e->prof_events[i - 1], e->prof_events[i]) == cudaSuccess) {
				e->prof_ms[e->prof_ids[i]] += ms;
				e->prof_launches[e->prof_ids[i]]++;
			}
		}
	}
	for(cudaEvent_t ev : e->prof_events) cudaEventDestroy(ev);
	e->prof_events.clear();
	e->prof_ids.clear();
}

static int round_up(int v, int m) { return (v + m - 1) / m * m; }

static size_t max_frame_bytes_for(const fb200_encoder_config &c, int bs)
{
	// header <= 16, per channel: verbatim worst case bs*(bps+1) bits + estimate slack bs/2 bits
	// (count_rice_bits_in_partition_ underestimates by at most n/2) + warm-up/coefficients, CRC-16.
	const size_t per_ch = ((size_t)bs * (c.bits_per_sample + 2) + 7) / 8 + 256;
	return 16 + per_ch * c.channels + 2 + 16;
}

// Expand the apodization list into sections + candidates for blocksize bs
// (apply_apodization_ / set_next_subdivide_tukey, stream_encoder.c:4293-4392).
static int build_geometry(fb200_encoder *e, int bs, Geometry **out)
{
	auto it = e->geoms.find(bs);
	if(it != e->geoms.end()) { *out = &it->second; return FB200_OK; }
	const fb200_encoder_config &c = e->cfg;
	Geometry g;
	g.bs = bs;
	EncK &k = g.k;
	memset(&k, 0, sizeof k);
	k.channels = (int)c.channels; k.bps = (int)c.bits_per_sample; k.sample_rate = (int)c.sample_rate;
	k.bs = bs; k.bs_stride = round_up((int)c.blocksize, 4);
	k.do_ms = c.do_mid_side_stereo; k.loose_ms = c.loose_mid_side_stereo;
	k.nsig = e->nsig;
	k.max_order = (int)c.max_lpc_order >= bs ? bs - 1 : (int)c.max_lpc_order;
	k.lags = k.max_order + 1;
	k.lag_stride = (int)e->lag_stride;
	k.qlp_precision = (int)c.qlp_coeff_precision;
	k.prec_search = c.do_qlp_coeff_prec_search ? 1 : 0;
	k.exhaustive = c.do_exhaustive_model_search;
	{   // stream_encoder.c:3759-3761, format.c:540-548
		int o = 0, b = bs;
		while(!(b & 1)) { o++; b >>= 1; }
		if(o > 15) o = 15;
		k.max_po = o < (int)c.max_residual_partition_order ? o : (int)c.max_residual_partition_order;
		k.min_po = (int)c.min_residual_partition_order < k.max_po ? (int)c.min_residual_partition_order : k.max_po;
	}
	k.rice_limit = c.bits_per_sample > 16 ? (int)kRice2Escape : (int)kRiceEscape;
	k.limit_min_bitrate = c.limit_min_bitrate ? 1 : 0;
	k.redo = nullptr;
	k.sig_group = 0;
	k.dis_const = c.disable_constant_subframes || (c.limit_min_bitrate && c.channels == 1);  // mono: the only channel is the last one
	k.dis_fixed = c.disable_fixed_subframes; k.dis_verb = c.disable_verbatim_subframes;
	k.slot_stride = round_up((int)max_frame_bytes_for(c, (int)c.blocksize), 16);
	k.slot_words = k.slot_stride / 4;
	{
		// k_emit3's frame buffer: a subframe is never longer than its verbatim form + n/2 + one bit per partition (the search
		// keeps a candidate only if its estimate beats verbatim, and the Rice estimate undershoots by at most that); at most one
		// of two channels is a side channel (bps + 1)
		const size_t bits = 128 + (size_t)bs * ((size_t)c.bits_per_sample * c.channels + (c.channels == 2 ? 1 : 0)) + (size_t)c.channels * ((size_t)bs / 2 + 512 + 2 * c.bits_per_sample) + 16;
		const int w = (int)((bits + 31) / 32) + 4;
		k.emit3_words = w < k.slot_words ? w : k.slot_words;
	}

	std::vector<float> windows;
	std::vector<DevSection> secs;
	std::vector<DevCand> cands;
	if(k.max_order > 0 && bs > 1) {
		for(uint32_t a = 0; a < c.num_apodizations; a++) {
			const fb200_apodization &ap = c.apodizations[a];
			const int win_off = (int)windows.size();
			windows.resize(windows.size() + bs);
			fbwin::make(ap, windows.data() + win_off, bs);  // resize_buffers_, stream_encoder.c:2913-2975
			const int root = (int)secs.size();
			secs.push_back(DevSection{win_off, 0, bs, 0, 0});
			cands.push_back(DevCand{0, root, root});
			if(ap.type == FB200_APOD_SUBDIVIDE_TUKEY) {
				for(int b = 2; b <= ap.parts; b++) {
					if(bs / b <= FB200_MAX_LPC_ORDER) continue;  // :4349-4357
					const int nparts = (b == 2) ? 2 : b;
					for(int part = 0; part < nparts; part++) {
						const int sidx = (int)secs.size();
						secs.push_back(DevSection{win_off, 1, bs / b, bs / b / 2, (part * bs) / b});
						cands.push_back(DevCand{0, sidx, root});
						if(b != 2) cands.push_back(DevCand{1, sidx, root});  // depth 2 has no punch-outs (:4295-4302)
					}
				}
			}
		}
	}
	k.nsec = (int)secs.size();
	g.or_sec = secs.empty() ? -1 : 0;  // every apodization opens with its full-length section
	k.nwin = (int)cands.size();
	k.nslots = k.nwin * (k.exhaustive ? (k.max_order > 0 ? k.max_order : 1) : 1) * (k.prec_search ? kQlpPrecisionSteps : 1);
	if((size_t)k.nsec > e->max_nsec || (size_t)k.nslots > e->max_nslots) {
		set_error("internal: geometry for blocksize %d exceeds workspace (nsec %d/%zu nslots %d/%zu)", bs, k.nsec, e->max_nsec, k.nslots, e->max_nslots);
		return FB200_ERR_INVALID;
	}
	if(!windows.empty()) {
		FB_CUDA(cudaMalloc(&g.d_windows, windows.size() * sizeof(float)));
		FB_CUDA(cudaMemcpy(g.d_windows, windows.data(), windows.size() * sizeof(float), cudaMemcpyHostToDevice));
		FB_CUDA(cudaMalloc(&g.d_secs, secs.size() * sizeof(DevSection)));
		FB_CUDA(cudaMemcpy(g.d_secs, secs.data(), secs.size() * sizeof(DevSection), cudaMemcpyHostToDevice));
		FB_CUDA(cudaMalloc(&g.d_cands, cands.size() * sizeof(DevCand)));
		FB_CUDA(cudaMemcpy(g.d_cands, cands.data(), cands.size() * sizeof(DevCand), cudaMemcpyHostToDevice));
		// per-section weights over absolute sample indices: the window inside the section (lpc.c:68-94), zero elsewhere
		const size_t stride = (size_t)bs + kSecwinSlack;
		std::vector<float> sw(secs.size() * stride, 0.0f);
		for(size_t si = 0; si < secs.size(); si++) {
			const DevSection &S = secs[si];
			float *dst = sw.data() + si * stride;
			const float *w = windows.data() + S.win_off;
			if(!S.partial) for(int i = 0; i < bs; i++) dst[i] = w[i];
			else {
				for(int i = 0; i < S.part_size && S.data_shift + i < bs; i++) dst[S.data_shift + i] = w[i];
				for(int i = S.part_size; i < 2 * S.part_size && S.data_shift + i < bs; i++) dst[S.data_shift + i] = w[bs - 2 * S.part_size + i];
			}
		}
		FB_CUDA(cudaMalloc(&g.d_secwin, sw.size() * sizeof(float)));
		FB_CUDA(cudaMemcpy(g.d_secwin, sw.data(), sw.size() * sizeof(float), cudaMemcpyHostToDevice));
	}
	g.search_smem = (size_t)k.bs_stride * 8;
	{
		const int xcap = k.bs_stride + (k.bs_stride >> 5) + 1;
		g.emit_smem = (size_t)xcap * 8 + (size_t)k.slot_words * 4;
		g.maxord_t = k.max_order <= 8 ? 8 : k.max_order <= 12 ? 12 : 32;
		{
			int rt = 0;
			if(bs % (32 * 32) == 0) rt = 32;
			else if(bs % (32 * 36) == 0) rt = 36;
			const int ntl = rt ? bs / (32 * rt) : 0;  // tiles; the partition <-> lane mapping needs a power of two
			// two warps per signal; more than four signals: CTAs of four signals each (half the shared memory, twice the warps per SM)
			const int wps = 2;
			const int gsz = k.nsig <= 4 ? k.nsig : 4;
			const size_t need = rt ? search5_smem(bs, rt, gsz, wps, k.max_po) : 0;
			if(rt && (ntl & (ntl - 1)) == 0 && k.max_po <= kMaxPartitionOrder && ((bs >> k.max_po) % rt) == 0 && need <= 200 * 1024 && 32 * wps * gsz <= 256) {
				k.sig_group = k.nsig <= 4 ? 0 : gsz;
				g.fast_search3 = rt;
				g.search_wps = wps;
				g.search5_smem = need;
			}
		}
		// resident emit kernel: 1-2 channels, runs of R_T samples, one thread per run, at most 256 threads
		if(g.fast_search3 && k.channels <= 2 && (bs / g.fast_search3) >= 32 && (bs / g.fast_search3) * k.channels <= 256 && ((size_t)bs * k.channels * 4) % 16 == 0) {
			const size_t need = emit3_smem_bytes(bs, g.fast_search3, k.channels, k.emit3_words);
			if(need <= 200 * 1024) { g.emit3_rt = g.fast_search3; g.emit3_smem = need; }
		}
		// more than two channels: the same kernel per channel pair (independent channels), spliced per frame by k_join
		if(g.fast_search3 && k.channels > 2 && (bs / g.fast_search3) >= 32 && (bs / g.fast_search3) * 2 <= 256) {
			const size_t pbits = 128 + (size_t)bs * (size_t)c.bits_per_sample * 2 + 2 * ((size_t)bs / 2 + 512 + 2 * c.bits_per_sample) + 16;
			const int pw = (int)((pbits + 31) / 32) + 4;
			const size_t need = emit3_smem_bytes(bs, g.fast_search3, 2, pw), needj = join_smem(k.emit3_words);
			if(need <= 200 * 1024 && needj <= 200 * 1024) {
				g.emit3_rt = g.fast_search3; g.emit3_pair = true; g.pair_words = pw; g.pair_smem = need; g.join_smem = needj;
			}
		}
		g.raw_pipeline = g.emit3_rt != 0;
	}
	e->geoms[bs] = g;
	*out = &e->geoms[bs];
	return FB200_OK;
}

static int bs_plus_slack(int bs) { return bs + kSecwinSlack; }

// workspace set b, starting at block `off_blocks` of it (every array is laid out per block / per (block, signal) item, sized
// for max_blocks blocks with the stream's largest section / slot counts: a launch of n blocks at offset o stays inside)
static void use_ws(fb200_encoder *e, int b, size_t off_blocks = 0)
{
	const size_t oi = off_blocks * (size_t)e->nsig;
	const size_t bs_stride = (size_t)round_up((int)e->cfg.blocksize, 4);
	e->d_sig = e->ws[b].d_sig + oi * bs_stride; e->d_meta = e->ws[b].d_meta + oi; e->d_blkflags = e->ws[b].d_blkflags + off_blocks;
	e->d_sigor = e->ws[b].d_sigor + oi;
	e->d_autoc = e->ws[b].d_autoc + oi * (e->max_nsec ? e->max_nsec : 1) * e->lag_stride;
	e->d_cdesc = e->ws[b].d_cdesc + oi * (e->max_nslots ? e->max_nslots : 1);
}

// Stage A of nb blocks of size g.bs starting at d_pcm: k_prep, k_autoc, k_lpc (writes the current workspace set).
static int run_stage_a(fb200_encoder *e, Geometry &g, const int32_t *d_pcm, int nb, cudaStream_t st)
{
	EncK k = g.k;
	const int nitems = nb * k.nsig;
	prof_mark(e, -1, st);
	const bool raw = g.raw_pipeline && !e->use_v1 && (e->debug_path & 7) == 0 && ((uintptr_t)d_pcm & 15) == 0;
	// Wasted-bits detection needs nothing but the OR of a signal's samples. With a full-length analysis section k_autoc4 collects
	// it on the way (its chains read every sample anyway) and k_lpc derives wasted bits / subframe bps: no kernel reads the block
	// just for that. Otherwise k_meta does it -- concurrently with k_autoc4 on a second stream when the autocorrelation does not
	// need the meta data (it does under loose mid-side, to skip the inactive pair); k_lpc joins them.
	const bool fused = raw && k.nwin > 0 && !k.loose_ms && g.or_sec >= 0 && g.fast_search3 && g.emit3_rt && !(e->debug_path & 8);
	const bool overlap = !fused && raw && k.nwin > 0 && !k.loose_ms && !e->prof_on;
	if(fused) {}
	else if(overlap) {
		FB_CUDA(cudaEventRecord(e->ev_meta_fork, st));
		FB_CUDA(cudaStreamWaitEvent(e->s_meta, e->ev_meta_fork, 0));
		launch_meta(k, d_pcm, e->d_meta, e->d_blkflags, nb, e->s_meta);
		FB_CUDA(cudaEventRecord(e->ev_meta_done, e->s_meta));
	}
	else if(raw) launch_meta(k, d_pcm, e->d_meta, e->d_blkflags, nb, st);  // no planar copy: the fast kernels read the caller's PCM
	else launch_prep(k, d_pcm, e->d_sig, e->d_meta, e->d_blkflags, nb, st);
	prof_mark(e, FB200_PROF_PREP, st);
	if(!fused) e->launches++;
	if(k.nwin > 0) {
		if(raw) launch_autoc4(k, d_pcm, (overlap || fused) ? nullptr : e->d_meta, g.d_secwin, bs_plus_slack(k.bs), g.d_secs, e->d_autoc, nitems, fused ? e->d_sigor : nullptr, g.or_sec, st);
		else if(e->use_v1) launch_autoc_general(k, e->d_sig, e->d_meta, g.d_windows, g.d_secs, e->d_autoc, nitems, st);
		else launch_autoc3(k, e->d_sig, e->d_meta, g.d_windows, g.d_secs, e->d_autoc, nitems, st);
		prof_mark(e, FB200_PROF_AUTOC, st);
		if(overlap) FB_CUDA(cudaStreamWaitEvent(st, e->ev_meta_done, 0));
		launch_lpc(k, e->d_autoc, g.d_cands, e->d_meta, fused ? e->d_sigor : nullptr, e->d_cdesc, nitems, (overlap || fused) ? 1 : 0, st);
		prof_mark(e, FB200_PROF_LPC, st);
		e->launches += 2;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

// Stage B: search + emit (reads the current workspace set). Regular blocksizes: k_search4 + k_emit3 (frames go straight
// to their final offsets); everything else: the general k_search + k_emit + k_scan + k_gather.
static int run_stage_b(fb200_encoder *e, Geometry &g, const int32_t *d_pcm, int nb, uint32_t first_frame, uint64_t frame_index0,
                       uint8_t *d_out, size_t out_cap, unsigned long long *d_offsets, cudaStream_t st)
{
	EncK k = g.k;
	k.first_frame = first_frame;
	k.blk0 = (uint32_t)frame_index0;
	k.f64b = e->f64b;
	k.file_blocks = (int)e->file_blocks;
	const int nitems = nb * k.nsig;
	prof_mark(e, -1, st);
	if(g.fast_search3 && !e->use_v1 && !(e->debug_path & 2)) launch_search5(k, g.fast_search3, g.maxord_t, g.search_wps, g.search5_smem, d_pcm, e->d_meta, e->d_cdesc, e->d_plans, nb, st);
	else launch_search_general(k, g.search_smem, e->d_sig, e->d_meta, e->d_cdesc, e->d_plans, nitems, st);
	if(k.limit_min_bitrate && k.channels > 1 && !k.dis_const) {
		// stream_encoder.c:3874-3879: blocks whose channels 0 .. n-2 all came out constant search their last channel (and mid /
		// side) again with constant subframes disabled
		launch_minbr_flags(k, e->d_plans, k.loose_ms ? e->d_blkflags : nullptr, nb, e->d_redo, st);
		EncK k2 = k;
		k2.dis_const = 1;
		k2.redo = e->d_redo;
		if(g.fast_search3 && !e->use_v1 && !(e->debug_path & 2)) launch_search5(k2, g.fast_search3, g.maxord_t, g.search_wps, g.search5_smem, d_pcm, e->d_meta, e->d_cdesc, e->d_plans, nb, st);
		else launch_search_general(k2, g.search_smem, e->d_sig, e->d_meta, e->d_cdesc, e->d_plans, nitems, st);
		e->launches += 2;
	}
	prof_mark(e, FB200_PROF_SEARCH, st);
	if(g.emit3_rt && !e->use_v1 && !(e->debug_path & 4) && ((uintptr_t)d_pcm & 15) == 0) {
		if((++e->epoch & kLbEpochMask) == 0) {
			FB_CUDA(cudaMemsetAsync(e->d_lookback, 0, (size_t)e->max_blocks * sizeof(unsigned long long), st));
			e->epoch = 1;
		}
		Emit3Args a;
		a.pcm = d_pcm; a.meta = e->d_meta; a.blkflags = e->d_blkflags; a.plans = e->d_plans; a.crc_tab = e->d_crc_tab;
		a.out = d_out; a.out_cap = (unsigned long long)out_cap; a.offsets = d_offsets + frame_index0;
		a.running_in = e->d_running + e->run_cur; a.running_out = e->d_running + (e->run_cur ^ 1);
		a.lookback = e->d_lookback; a.ticket = e->d_ticket; a.ticket_base = e->ticket_base; a.epoch = e->epoch;
		a.nb = nb; a.chan_assign_out = e->d_chan_assign; a.err = e->d_err;
		a.stage = nullptr; a.stage_bits = nullptr; a.pair_words = g.pair_words; a.join_words = k.emit3_words;
		if(g.emit3_pair) {
			const size_t npairs = ((size_t)k.channels + 1) / 2;
			const size_t need = (size_t)e->max_blocks * npairs * (size_t)g.pair_words;
			if(need > e->d_stage_words) {  // first use with this geometry (synchronous, once)
				FB_CUDA(cudaStreamSynchronize(st));
				cudaFree(e->d_stage); cudaFree(e->d_stage_bits); e->d_stage = nullptr; e->d_stage_bits = nullptr; e->d_stage_words = 0;
				FB_CUDA(cudaMalloc(&e->d_stage, need * sizeof(uint32_t)));
				FB_CUDA(cudaMalloc(&e->d_stage_bits, (size_t)e->max_blocks * npairs * sizeof(uint32_t)));
				e->d_stage_words = need;
			}
			a.stage = e->d_stage; a.stage_bits = e->d_stage_bits;
			launch_emit3_pairs(k, g.emit3_rt, g.maxord_t, g.pair_smem, g.join_smem, a, nb, st);
		}
		else launch_emit3(k, g.emit3_rt, g.maxord_t, g.emit3_smem, a, nb, st);
		e->ticket_base += (unsigned)nb;
		e->run_cur ^= 1;
		prof_mark(e, FB200_PROF_EMIT, st);
		e->launches += 2;
	}
	else {
		launch_emit_general(k, g.emit_smem, e->d_sig, e->d_blkflags, e->d_plans, e->d_slots, e->d_frame_bytes, e->d_chan_assign, nb, st);
		prof_mark(e, FB200_PROF_EMIT, st);
		launch_scan(e->d_frame_bytes, nb, d_offsets + frame_index0, e->d_running + e->run_cur, st);
		prof_mark(e, FB200_PROF_SCAN, st);
		launch_gather(k, e->d_slots, e->d_frame_bytes, d_offsets + frame_index0, d_out, (unsigned long long)out_cap, e->d_err, nb, st);
		prof_mark(e, FB200_PROF_GATHER, st);
		e->launches += 4;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

struct PipeChunk { uint64_t first; uint32_t nb; uint32_t blocksize; cudaEvent_t wait_before_a; };

// Enqueue chunk `idx` of a call: stage A on a stage-A stream, stage B on `sb`. Slice mode: the chunk works in its own slice of
// workspace set 0; otherwise consecutive chunks alternate between the two sets and wait for the set's previous user.
static cudaStream_t stage_a_stream(fb200_encoder *e, size_t idx) { return e->slice_mode ? e->s_as[idx % fb200_encoder::kStageAStreams] : e->s_a; }

static int enqueue_chunk(fb200_encoder *e, size_t idx, const PipeChunk &c, const int32_t *d_pcm_base, uint32_t first_frame_number,
                         uint8_t *d_out, size_t out_cap, unsigned long long *d_offsets, cudaStream_t sb)
{
	const uint32_t bs = e->cfg.blocksize, ch = e->cfg.channels;
	const int b = e->slice_mode ? 0 : (int)(idx & 1);
	cudaStream_t sa = stage_a_stream(e, idx);
	Geometry *g = nullptr;
	int rc;
	if((rc = build_geometry(e, (int)c.blocksize, &g)) != FB200_OK) return rc;
	if(c.wait_before_a) FB_CUDA(cudaStreamWaitEvent(sa, c.wait_before_a, 0));
	if(!e->slice_mode && e->ev_b_valid[b]) FB_CUDA(cudaStreamWaitEvent(sa, e->ev_b[b], 0));  // stage B two chunks ago is done with this set
	use_ws(e, b, e->slice_mode ? (size_t)c.first : 0);
	if((rc = run_stage_a(e, *g, d_pcm_base + (size_t)c.first * bs * ch, (int)c.nb, sa)) != FB200_OK) return rc;
	cudaEvent_t done_a = e->ev_a[b];
	if(e->slice_mode) {
		while(e->ev_ca.size() <= idx) {
			cudaEvent_t ev;
			FB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
			e->ev_ca.push_back(ev);
		}
		done_a = e->ev_ca[idx];
	}
	FB_CUDA(cudaEventRecord(done_a, sa));
	FB_CUDA(cudaStreamWaitEvent(sb, done_a, 0));
	if((rc = run_stage_b(e, *g, d_pcm_base + (size_t)c.first * bs * ch, (int)c.nb, first_frame_number, c.first, d_out, out_cap, d_offsets, sb)) != FB200_OK) return rc;
	if(!e->slice_mode) {
		FB_CUDA(cudaEventRecord(e->ev_b[b], sb));
		e->ev_b_valid[b] = true;
	}
	return FB200_OK;
}

// after the call's set-up work was enqueued on `st`: every stage-A stream starts behind it
static int fork_stage_a(fb200_encoder *e, cudaStream_t st)
{
	FB_CUDA(cudaEventRecord(e->ev_fork, st));
	for(int i = 0; i < (e->slice_mode ? fb200_encoder::kStageAStreams : 1); i++) FB_CUDA(cudaStreamWaitEvent(e->s_as[i], e->ev_fork, 0));
	return FB200_OK;
}

extern "C" {

const char *fb200_version(void) { return "flac_b200 0.1 (sm_90a)"; }
const char *fb200_last_error(void) { return fb200::get_error(); }

int fb200_device_count(void)
{
	int n = 0;
	const cudaError_t e = cudaGetDeviceCount(&n);
	if(e != cudaSuccess) {
		set_error("cudaGetDeviceCount: %s", cudaGetErrorString(e));
		return FB200_ERR_CUDA;
	}
	return n;
}

int fb200_encoder_config_preset(fb200_encoder_config *cfg, uint32_t channels, uint32_t bps, uint32_t sample_rate, uint32_t level, uint32_t blocksize)
{
	// src/libFLAC/stream_encoder.c:117-140 compression_levels_
	static const struct { int ms, loose; uint32_t lpc, maxpo; int parts; } L[9] = {
		{0, 0, 0, 3, 0}, {1, 1, 0, 3, 0}, {1, 0, 0, 3, 0}, {0, 0, 6, 4, 0}, {1, 1, 8, 4, 0},
		{1, 0, 8, 5, 0}, {1, 0, 8, 6, 2}, {1, 0, 12, 6, 2}, {1, 0, 12, 6, 3}};
	if(!cfg) return FB200_ERR_INVALID;
	if(level > 8) level = 8;
	memset(cfg, 0, sizeof *cfg);
	cfg->channels = channels; cfg->bits_per_sample = bps; cfg->sample_rate = sample_rate; cfg->blocksize = blocksize;
	cfg->do_mid_side_stereo = L[level].ms; cfg->loose_mid_side_stereo = L[level].loose;
	cfg->max_lpc_order = L[level].lpc;
	cfg->max_residual_partition_order = L[level].maxpo;
	cfg->num_apodizations = 1;
	if(L[level].parts) {
		const float p = 5e-1;  // stream_encoder.c:2040-2049
		cfg->apodizations[0].type = FB200_APOD_SUBDIVIDE_TUKEY;
		cfg->apodizations[0].parts = L[level].parts;
		cfg->apodizations[0].p = p / L[level].parts;
	}
	else {
		cfg->apodizations[0].type = FB200_APOD_TUKEY;
		cfg->apodizations[0].p = 0.5f;
	}
	return FB200_OK;
}

// FLAC__stream_encoder_set_apodization (stream_encoder.c:1940-2065): ';'-separated window names.
// Unknown names are skipped; an empty result falls back to tukey(0.5); at most 32 windows.
// Kept quirks: the '/' separators of the *_tukey(...) forms are searched with strchr from the
// start of the current item to the end of the whole string (:1994, :2015, :2037), and
// partial_/punchout_tukey expand only while num + parts < 32 (:2004, :2025).
int fb200_encoder_config_set_apodization(fb200_encoder_config *cfg, const char *spec)
{
	if(!cfg || !spec) return FB200_ERR_INVALID;
	static const struct { const char *name; int32_t type; } plain[] = {
		{"bartlett", FB200_APOD_BARTLETT}, {"bartlett_hann", FB200_APOD_BARTLETT_HANN}, {"blackman", FB200_APOD_BLACKMAN},
		{"blackman_harris_4term_92db", FB200_APOD_BLACKMAN_HARRIS_4TERM_92DB_SIDELOBE}, {"connes", FB200_APOD_CONNES},
		{"flattop", FB200_APOD_FLATTOP}, {"hamming", FB200_APOD_HAMMING}, {"hann", FB200_APOD_HANN},
		{"kaiser_bessel", FB200_APOD_KAISER_BESSEL}, {"nuttall", FB200_APOD_NUTTALL}, {"rectangle", FB200_APOD_RECTANGLE},
		{"triangle", FB200_APOD_TRIANGLE}, {"welch", FB200_APOD_WELCH}};
	uint32_t &num = cfg->num_apodizations;
	num = 0;
	auto push = [&](int32_t type, float p, int32_t parts, float start, float end) {
		fb200_apodization &a = cfg->apodizations[num++];
		a.type = type; a.p = p; a.parts = parts; a.start = start; a.end = end;
	};
	auto starts = [&](const char *prefix) { return 0 == strncmp(prefix, spec, strlen(prefix)); };
	for(;;) {
		const char *semi = strchr(spec, ';');
		const size_t n = semi ? (size_t)(semi - spec) : strlen(spec);
		bool matched = false;
		for(const auto &pl : plain)
			if(n == strlen(pl.name) && 0 == strncmp(pl.name, spec, n)) { push(pl.type, 0.0f, 0, 0.0f, 0.0f); matched = true; break; }
		if(matched) {}
		else if(n > 7 && starts("gauss(")) {
			const float stddev = (float)strtod(spec + 6, 0);
			if(stddev > 0.0 && stddev <= 0.5) push(FB200_APOD_GAUSS, stddev, 0, 0.0f, 0.0f);
		}
		else if(n > 7 && starts("tukey(")) {
			const float p = (float)strtod(spec + 6, 0);
			if(p >= 0.0 && p <= 1.0) push(FB200_APOD_TUKEY, p, 0, 0.0f, 0.0f);
		}
		else if((n > 15 && starts("partial_tukey(")) || (n > 16 && starts("punchout_tukey("))) {
			const bool partial = spec[1] == 'a';
			const int32_t parts = (int32_t)strtod(spec + (partial ? 14 : 15), 0);
			const char *s1 = strchr(spec, '/');
			const float ov_in = s1 ? (float)strtod(s1 + 1, 0) : 0.0f;
			const float overlap = s1 ? (ov_in < 0.99f ? ov_in : 0.99f) : (partial ? 0.1f : 0.2f);
			const float overlap_units = 1.0f / (1.0f - overlap) - 1.0f;
			const char *s2 = strchr(s1 ? s1 + 1 : spec, '/');
			const float tukey_p = s2 ? (float)strtod(s2 + 1, 0) : 0.2f;
			if(parts <= 1) push(FB200_APOD_TUKEY, tukey_p, 0, 0.0f, 0.0f);
			else if(num + parts < 32)
				for(int32_t m = 0; m < parts; m++)
					push(partial ? FB200_APOD_PARTIAL_TUKEY : FB200_APOD_PUNCHOUT_TUKEY, tukey_p, 0,
					     m / (parts + overlap_units), (m + 1 + overlap_units) / (parts + overlap_units));
		}
		else if(n > 17 && starts("subdivide_tukey(")) {
			const int32_t parts = (int32_t)strtod(spec + 16, 0);
			if(parts > 1) {
				const char *s1 = strchr(spec, '/');
				float p = s1 ? (float)strtod(s1 + 1, 0) : 5e-1;
				if(p > 1) p = 1;
				else if(p < 0) p = 0;
				push(FB200_APOD_SUBDIVIDE_TUKEY, p / parts, parts, 0.0f, 0.0f);
			}
		}
		if(num == 32) break;
		if(!semi) break;
		spec = semi + 1;
	}
	if(num == 0) push(FB200_APOD_TUKEY, 0.5f, 0, 0.0f, 0.0f);
	return FB200_OK;
}

// One window table, as the encoder uploads it (tests compare it with the reference's FLAC__window_*).
int fb200_window(const fb200_apodization *apodization, int32_t length, float *out)
{
	if(!apodization || !out || length < 2) return FB200_ERR_INVALID;
	return fbwin::make(*apodization, out, length) ? FB200_OK : FB200_ERR_INVALID;
}

int fb200_encoder_create(const fb200_encoder_config *cfg_in, int device, uint32_t max_blocks, fb200_encoder **out)
{
	if(!cfg_in || !out) return FB200_ERR_INVALID;
	*out = nullptr;
	fb200_encoder_config c = *cfg_in;
	// ---- init_stream_internal_ validation / defaults (stream_encoder.c:725-830)
	if(c.channels == 0 || c.channels > FB200_MAX_CHANNELS) { set_error("invalid number of channels %u", c.channels); return FB200_ERR_INVALID; }
	if(c.channels != 2) { c.do_mid_side_stereo = 0; c.loose_mid_side_stereo = 0; }
	else if(!c.do_mid_side_stereo) c.loose_mid_side_stereo = 0;
	if(c.bits_per_sample < 4 || c.bits_per_sample > 32) { set_error("invalid bits per sample %u", c.bits_per_sample); return FB200_ERR_INVALID; }
	if(c.bits_per_sample > 24) { set_error("bits_per_sample %u > 24 (33-bit side channel path) is outside this engine's scope", c.bits_per_sample); return FB200_ERR_UNSUPPORTED; }
	if(c.sample_rate == 0 || c.sample_rate > 1048575u) { set_error("invalid sample rate %u", c.sample_rate); return FB200_ERR_INVALID; }
	if(c.blocksize == 0) c.blocksize = c.max_lpc_order == 0 ? 1152 : 4096;
	if(c.blocksize < 16 || c.blocksize > 65535) { set_error("invalid blocksize %u", c.blocksize); return FB200_ERR_INVALID; }
	if(c.max_lpc_order > FB200_MAX_LPC_ORDER) { set_error("invalid max LPC order %u", c.max_lpc_order); return FB200_ERR_INVALID; }
	if(c.blocksize < c.max_lpc_order) { set_error("blocksize too small for LPC order"); return FB200_ERR_INVALID; }
	if(c.qlp_coeff_precision == 0) {
		if(c.bits_per_sample < 16) {
			const uint32_t v = 2 + c.bits_per_sample / 2;
			c.qlp_coeff_precision = v > kMinQlpPrecision ? v : kMinQlpPrecision;
		}
		else if(c.bits_per_sample == 16) {
			if(c.blocksize <= 192) c.qlp_coeff_precision = 7;
			else if(c.blocksize <= 384) c.qlp_coeff_precision = 8;
			else if(c.blocksize <= 576) c.qlp_coeff_precision = 9;
			else if(c.blocksize <= 1152) c.qlp_coeff_precision = 10;
			else if(c.blocksize <= 2304) c.qlp_coeff_precision = 11;
			else if(c.blocksize <= 4608) c.qlp_coeff_precision = 12;
			else c.qlp_coeff_precision = 13;
		}
		else {
			if(c.blocksize <= 384) c.qlp_coeff_precision = kMaxQlpPrecision - 2;
			else if(c.blocksize <= 1152) c.qlp_coeff_precision = kMaxQlpPrecision - 1;
			else c.qlp_coeff_precision = kMaxQlpPrecision;
		}
	}
	else if(c.qlp_coeff_precision < kMinQlpPrecision || c.qlp_coeff_precision > kMaxQlpPrecision) { set_error("invalid qlp coeff precision %u", c.qlp_coeff_precision); return FB200_ERR_INVALID; }
	if(c.max_residual_partition_order >= (1u << kRiceOrderLen)) c.max_residual_partition_order = (1u << kRiceOrderLen) - 1;
	if(c.min_residual_partition_order >= c.max_residual_partition_order) c.min_residual_partition_order = c.max_residual_partition_order;
	// ---- engine scope (fail loudly, no fallback)
	if(c.max_residual_partition_order > (uint32_t)kMaxPartitionOrder) { set_error("max_residual_partition_order %u > %d unsupported", c.max_residual_partition_order, kMaxPartitionOrder); return FB200_ERR_UNSUPPORTED; }
	if(c.num_apodizations == 0 || c.num_apodizations > FB200_MAX_APODIZATIONS) { set_error("invalid number of apodizations"); return FB200_ERR_INVALID; }
	for(uint32_t a = 0; a < c.num_apodizations; a++)
		if(c.apodizations[a].type < FB200_APOD_TUKEY || c.apodizations[a].type > FB200_APOD_WELCH) { set_error("apodization type %d unknown", c.apodizations[a].type); return FB200_ERR_INVALID; }

	int ndev = 0;
	if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
		set_error("no CUDA device: the FLAC block engine has no CPU fallback");
		return FB200_ERR_CUDA;
	}
	if(device < 0 || device >= ndev) { set_error("invalid device %d", device); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(device));

	fb200_encoder *e = new fb200_encoder();
	e->cfg = c;
	e->device = device;
	e->max_blocks = max_blocks ? max_blocks : 4096;
	e->nsig = (int)c.channels + ((c.channels == 2 && c.do_mid_side_stereo) ? 2 : 0);
	{
		const int lags = (int)c.max_lpc_order + 1;
		e->lag_stride = lags <= 7 ? 7 : lags <= 9 ? 9 : lags <= 13 ? 13 : lags <= 17 ? 17 : 33;
		size_t nsec = 0, nwin = 0;
		for(uint32_t a = 0; a < c.num_apodizations; a++) {
			nsec++; nwin++;
			if(c.apodizations[a].type == FB200_APOD_SUBDIVIDE_TUKEY)
				for(int b = 2; b <= c.apodizations[a].parts; b++) {
					const int np = (b == 2) ? 2 : b;
					nsec += np;
					nwin += (b == 2) ? np : 2 * np;
				}
		}
		e->max_nsec = nsec;
		e->max_nslots = nwin * (c.do_exhaustive_model_search ? (c.max_lpc_order ? c.max_lpc_order : 1) : 1) * (c.do_qlp_coeff_prec_search ? kQlpPrecisionSteps : 1);
	}
	const size_t nb = e->max_blocks, nitems = nb * e->nsig;
	const size_t bs_stride = (size_t)round_up((int)c.blocksize, 4);
	const size_t slot = (size_t)round_up((int)max_frame_bytes_for(c, (int)c.blocksize), 16);
#define ALLOC(ptr, bytes)                                                                     \
	do {                                                                                      \
		if(cudaMalloc(&(ptr), (bytes)) != cudaSuccess) {                                      \
			set_error("cudaMalloc(%zu) failed: %s", (size_t)(bytes), cudaGetErrorString(cudaGetLastError())); \
			fb200_encoder_destroy(e);                                                         \
			return FB200_ERR_ALLOC;                                                           \
		}                                                                                     \
	} while(0)
	for(int b = 0; b < 2; b++) {
		ALLOC(e->ws[b].d_sig, (nitems * bs_stride + 1024) * sizeof(int32_t));  // + slack: k_autoc2 reads whole int4 bodies past the last run
		ALLOC(e->ws[b].d_meta, nitems * sizeof(SigMeta));
		ALLOC(e->ws[b].d_sigor, nitems * sizeof(uint32_t));
		ALLOC(e->ws[b].d_blkflags, nb * sizeof(int));
		ALLOC(e->ws[b].d_autoc, (e->max_nsec ? e->max_nsec : 1) * nitems * e->lag_stride * sizeof(double));
		ALLOC(e->ws[b].d_cdesc, (e->max_nslots ? e->max_nslots : 1) * nitems * sizeof(CandDesc));
	}
	use_ws(e, 0);
	ALLOC(e->d_plans, nitems * sizeof(SubframePlan));
	ALLOC(e->d_slots, nb * slot);
	ALLOC(e->d_frame_bytes, nb * sizeof(uint32_t));
	ALLOC(e->d_chan_assign, nb * sizeof(uint32_t));
	ALLOC(e->d_running, 2 * sizeof(unsigned long long));
	ALLOC(e->d_crc_tab, (size_t)kCrcTabEntries * sizeof(uint16_t));
	ALLOC(e->d_lookback, nb * sizeof(unsigned long long));
	ALLOC(e->d_ticket, sizeof(unsigned));
	ALLOC(e->d_err, sizeof(int));
	ALLOC(e->d_redo, nb * sizeof(int));
#undef ALLOC
	bool streams_ok = true;
	for(int i = 0; i < fb200_encoder::kStageAStreams; i++) streams_ok = streams_ok && cudaStreamCreateWithFlags(&e->s_as[i], cudaStreamNonBlocking) == cudaSuccess;
	e->s_a = e->s_as[0];
	if(!streams_ok || cudaStreamCreateWithFlags(&e->s_meta, cudaStreamNonBlocking) != cudaSuccess ||
	   cudaEventCreateWithFlags(&e->ev_meta_fork, cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e->ev_meta_done, cudaEventDisableTiming) != cudaSuccess ||
	   cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
	   cudaEventCreateWithFlags(&e->ev_a[0], cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e->ev_a[1], cudaEventDisableTiming) != cudaSuccess ||
	   cudaEventCreateWithFlags(&e->ev_b[0], cudaEventDisableTiming) != cudaSuccess || cudaEventCreateWithFlags(&e->ev_b[1], cudaEventDisableTiming) != cudaSuccess ||
	   cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) {
		set_error("cudaStreamCreate failed");
		fb200_encoder_destroy(e);
		return FB200_ERR_CUDA;
	}
	cudaMemset(e->d_lookback, 0, nb * sizeof(unsigned long long));
	cudaMemset(e->d_ticket, 0, sizeof(unsigned));
	launch_crc16_tables(e->d_crc_tab, 0);
	Geometry *g = nullptr;
	int rc = build_geometry(e, (int)c.blocksize, &g);
	if(rc != FB200_OK) { fb200_encoder_destroy(e); return rc; }
	cudaDeviceProp prop;
	cudaGetDeviceProperties(&prop, device);
	if(!g->fast_search3 && (g->search_smem + 8192 > prop.sharedMemPerBlockOptin || g->emit_smem + 4096 > prop.sharedMemPerBlockOptin)) {
		set_error("blocksize %u x %u channels needs more shared memory than the device offers (search %zu, emit %zu)", c.blocksize, c.channels, g->search_smem, g->emit_smem);
		fb200_encoder_destroy(e);
		return FB200_ERR_UNSUPPORTED;
	}
	if(!g->emit3_rt && g->emit_smem + 4096 > prop.sharedMemPerBlockOptin) {
		set_error("blocksize %u x %u channels: a frame does not fit shared memory (emit %zu)", c.blocksize, c.channels, g->emit_smem);
		fb200_encoder_destroy(e);
		return FB200_ERR_UNSUPPORTED;
	}
	{
		// dynamic shared-memory opt-ins are per function and per device: raised once to fixed maxima, never per encoder
		// (two encoders with different blocksizes in one process must not lower each other's limit). The maxima (160 KB for
		// k_autoc4, 200 KB for k_search5 / k_emit3 / k_join) and the kernels' launch shapes were chosen on a previous GPU
		// and carried over unmeasured: they fit H100's 227 KB per block, and its per-SM registers and shared memory are the same.
		static bool inited[64] = {false};
		if(device < 64 && !inited[device]) {
			general_kernels_init(device);
			autoc3_init(device);
			autoc4_init(device);
			search5_init(device);
			emit3_init(device);
			inited[device] = true;
		}
	}
	{
		const char *env = getenv("FB200_FORCE_GENERAL_KERNELS");
		e->use_v1 = env && env[0] == '1';
		const char *fb = getenv("FB200_SEARCH_F64B");
		if(fb) e->f64b = atoi(fb) != 0;
		const char *dp = getenv("FB200_DEBUG_PATH");
		if(dp) e->debug_path = atoi(dp);
		const char *hc = getenv("FB200_HOST_CHUNKS");
		if(hc && atoi(hc) >= 1 && atoi(hc) <= 256) e->host_chunks = atoi(hc);
		const char *pc = getenv("FB200_PIPE_CHUNKS");
		if(pc && atoi(pc) >= 1 && atoi(pc) <= 64) e->pipe_chunks = atoi(pc);
	}
	*out = e;
	return FB200_OK;
}

void fb200_encoder_destroy(fb200_encoder *e)
{
	if(!e) return;
	cudaSetDevice(e->device);
	for(auto &kv : e->geoms) {
		cudaFree(kv.second.d_windows); cudaFree(kv.second.d_secs); cudaFree(kv.second.d_cands); cudaFree(kv.second.d_secwin);
	}
	for(int b = 0; b < 2; b++) {
		cudaFree(e->ws[b].d_sig); cudaFree(e->ws[b].d_meta); cudaFree(e->ws[b].d_sigor); cudaFree(e->ws[b].d_blkflags); cudaFree(e->ws[b].d_autoc); cudaFree(e->ws[b].d_cdesc);
		if(e->ev_a[b]) cudaEventDestroy(e->ev_a[b]);
		if(e->ev_b[b]) cudaEventDestroy(e->ev_b[b]);
	}
	if(e->ev_fork) cudaEventDestroy(e->ev_fork);
	for(int i = 0; i < fb200_encoder::kStageAStreams; i++) if(e->s_as[i]) cudaStreamDestroy(e->s_as[i]);
	for(cudaEvent_t ev : e->ev_ca) cudaEventDestroy(ev);
	if(e->s_meta) cudaStreamDestroy(e->s_meta);
	if(e->ev_meta_fork) cudaEventDestroy(e->ev_meta_fork);
	if(e->ev_meta_done) cudaEventDestroy(e->ev_meta_done);
	cudaFree(e->d_plans); cudaFree(e->d_slots); cudaFree(e->d_frame_bytes); cudaFree(e->d_chan_assign);
	cudaFree(e->d_running); cudaFree(e->d_err); cudaFree(e->d_redo); cudaFree(e->d_stage); cudaFree(e->d_stage_bits);
	cudaFree(e->d_crc_tab); cudaFree(e->d_lookback); cudaFree(e->d_ticket);
	cudaFree(e->d_pcm); cudaFree(e->d_packed); cudaFree(e->d_out); cudaFree(e->d_offsets);
	if(e->stream) cudaStreamDestroy(e->stream);
	if(e->s_h2d) cudaStreamDestroy(e->s_h2d);
	if(e->s_d2h) cudaStreamDestroy(e->s_d2h);
	for(cudaEvent_t ev : e->ev_h2d) cudaEventDestroy(ev);
	for(cudaEvent_t ev : e->ev_comp) cudaEventDestroy(ev);
	if(e->h_totals) cudaFreeHost(e->h_totals);
	prof_resolve(e);
	delete e;
}

int fb200_encoder_get_config(const fb200_encoder *e, fb200_encoder_config *resolved)
{
	if(!e || !resolved) return FB200_ERR_INVALID;
	*resolved = e->cfg;
	return FB200_OK;
}

size_t fb200_encoder_max_frame_bytes(const fb200_encoder *e) { return e ? max_frame_bytes_for(e->cfg, (int)e->cfg.blocksize) : 0; }
uint64_t fb200_encoder_launch_count(const fb200_encoder *e) { return e ? e->launches : 0; }

int fb200_encode_device(fb200_encoder *e, const int32_t *d_pcm, uint64_t samples, uint32_t first_frame_number,
                        uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint32_t *nframes,
                        uint64_t *total_bytes, void *cuda_stream, int sync)
{
	if(!e || !d_pcm || !d_out || !d_frame_offsets) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(e->device));
	cudaStream_t st = (cudaStream_t)cuda_stream;
	const uint32_t bs = e->cfg.blocksize, ch = e->cfg.channels;
	const uint64_t nfull = samples / bs;
	const uint32_t tail = (uint32_t)(samples % bs);
	if(nframes) *nframes = (uint32_t)(nfull + (tail ? 1 : 0));
	FB_CUDA(cudaMemsetAsync(e->d_running, 0, 2 * sizeof(unsigned long long), st));
	FB_CUDA(cudaMemsetAsync(e->d_err, 0, sizeof(int), st));
	unsigned long long *offs = reinterpret_cast<unsigned long long *>(d_frame_offsets);
	if(samples == 0) FB_CUDA(cudaMemsetAsync(offs, 0, sizeof(unsigned long long), st));
	// Sub-batches of at most max_blocks blocks; stage A (prep/autoc/lpc) of one overlaps stage B (search/emit) of the
	// previous on a second stream. Measured on an H100 SXM at 400 W (tools/sweep_chunks.sh, 10 000 blocks): one launch set
	// per call is fastest at -5 (1.24 ms per step vs 1.34 with 4 sub-batches) and no sub-batch count wins at -8 (3.83-3.89 ms for
	// 1-4) -- every kernel is more efficient at full batch size than the overlap wins back, so the default is as few
	// sub-batches as the workspace allows.
	uint64_t chunk = (nfull + e->pipe_chunks - 1) / e->pipe_chunks;
	if(chunk < 512) chunk = 512;
	if(chunk > e->max_blocks) chunk = e->max_blocks;
	std::vector<PipeChunk> chunks;
	for(uint64_t done = 0; done < nfull; done += chunk)
		chunks.push_back(PipeChunk{done, (uint32_t)((nfull - done) < chunk ? (nfull - done) : chunk), bs, nullptr});
	if(tail) chunks.push_back(PipeChunk{nfull, 1, tail, nullptr});  // short last block: own windows / header blocksize (stream_encoder.c:1703-1711)
	e->slice_mode = nfull + (tail ? 1 : 0) <= e->max_blocks;
	{ const int rc = fork_stage_a(e, st); if(rc != FB200_OK) return rc; }
	e->ev_b_valid[0] = e->ev_b_valid[1] = false;
	for(size_t i = 0; i < chunks.size(); i++) {
		const int rc = enqueue_chunk(e, i, chunks[i], d_pcm, first_frame_number, d_out, out_capacity, offs, st);
		if(rc != FB200_OK) return rc;
	}
	if(sync) {
		FB_CUDA(cudaStreamSynchronize(st));
		int err = 0;
		unsigned long long total = 0;
		FB_CUDA(cudaMemcpy(&err, e->d_err, sizeof err, cudaMemcpyDeviceToHost));
		FB_CUDA(cudaMemcpy(&total, e->d_running + e->run_cur, sizeof total, cudaMemcpyDeviceToHost));
		if(total_bytes) *total_bytes = total;
		if(err == 2) { set_error("internal: frame exceeded its size bound"); return FB200_ERR_CUDA; }
		if(err) { set_error("output buffer too small"); return FB200_ERR_OUTPUT_TOO_SMALL; }
	}
	return FB200_OK;
}

static int encode_host_impl(fb200_encoder *e, const void *pcm_any, uint32_t bytes_per_sample, uint64_t samples, uint32_t first_frame_number,
                            uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint32_t *nframes)
{
	// Host-buffer path: the batch is cut into chunks; chunk i+1's H2D copy, chunk i's kernels and
	// chunk i-1's D2H copy run on three streams (truly asynchronous when the caller's buffers are
	// pinned; pageable buffers still work, the copies then serialise inside the driver).
	if(!e || (!pcm_any && samples) || !out || !frame_offsets) return FB200_ERR_INVALID;
	if(bytes_per_sample != 2 && bytes_per_sample != 3 && bytes_per_sample != 4) { set_error("bytes_per_sample must be 2, 3 or 4"); return FB200_ERR_INVALID; }
	if(e->cfg.bits_per_sample > 8 * bytes_per_sample) { set_error("%u-bit samples do not fit %u bytes", e->cfg.bits_per_sample, bytes_per_sample); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(e->device));
	const uint32_t bs = e->cfg.blocksize, ch = e->cfg.channels;
	const uint64_t nfull = samples / bs;
	const uint32_t tail = (uint32_t)(samples % bs);
	const uint64_t nfr = nfull + (tail ? 1 : 0);
	if(nframes) *nframes = (uint32_t)nfr;
	if(nfr == 0) { frame_offsets[0] = 0; return FB200_OK; }
	const bool packed = bytes_per_sample != 4;
	const uint8_t *pcm_bytes_host = static_cast<const uint8_t *>(pcm_any);
	if(packed) {
		const size_t need = (size_t)samples * ch * bytes_per_sample + 256;
		if(need > e->d_packed_cap) {
			cudaFree(e->d_packed); e->d_packed = nullptr; e->d_packed_cap = 0;
			FB_CUDA(cudaMalloc(&e->d_packed, need));
			e->d_packed_cap = need;
		}
	}
	const size_t pcm_bytes = (size_t)samples * ch * sizeof(int32_t);
	const size_t need_out = (size_t)nfr * max_frame_bytes_for(e->cfg, (int)bs) + 64;
	if(pcm_bytes > e->d_pcm_cap) {
		cudaFree(e->d_pcm); e->d_pcm = nullptr; e->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&e->d_pcm, pcm_bytes + 256));
		e->d_pcm_cap = pcm_bytes + 256;
	}
	if(need_out > e->d_out_cap) {
		cudaFree(e->d_out); e->d_out = nullptr; e->d_out_cap = 0;
		FB_CUDA(cudaMalloc(&e->d_out, need_out));
		e->d_out_cap = need_out;
	}
	if((nfr + 1) > e->d_offsets_cap) {
		cudaFree(e->d_offsets); e->d_offsets = nullptr; e->d_offsets_cap = 0;
		FB_CUDA(cudaMalloc(&e->d_offsets, (nfr + 1) * sizeof(unsigned long long)));
		e->d_offsets_cap = nfr + 1;
	}
	if(!e->s_h2d) FB_CUDA(cudaStreamCreateWithFlags(&e->s_h2d, cudaStreamNonBlocking));
	if(!e->s_d2h) FB_CUDA(cudaStreamCreateWithFlags(&e->s_d2h, cudaStreamNonBlocking));
	// chunking: host_chunks (default 12) chunks per call, between 256 blocks and the launch capacity; the short last block is its own chunk
	uint64_t chunk = (nfull + e->host_chunks - 1) / e->host_chunks;
	if(chunk < 256) chunk = 256;
	if(chunk > e->max_blocks) chunk = e->max_blocks;
	std::vector<PipeChunk> chunks;
	for(uint64_t done = 0; done < nfull; done += chunk)
		chunks.push_back(PipeChunk{done, (uint32_t)((nfull - done) < chunk ? (nfull - done) : chunk), bs, nullptr});
	if(tail) chunks.push_back(PipeChunk{nfull, 1, tail, nullptr});
	const size_t used = chunks.size();
	if(used > e->h_totals_cap) {
		if(e->h_totals) cudaFreeHost(e->h_totals);
		e->h_totals = nullptr; e->h_totals_cap = 0;
		FB_CUDA(cudaMallocHost(&e->h_totals, (used + 16) * sizeof(unsigned long long)));
		e->h_totals_cap = used + 16;
	}
	while(e->ev_h2d.size() < used) {
		cudaEvent_t ea, eb;
		FB_CUDA(cudaEventCreateWithFlags(&ea, cudaEventDisableTiming));
		FB_CUDA(cudaEventCreateWithFlags(&eb, cudaEventDisableTiming));
		e->ev_h2d.push_back(ea); e->ev_comp.push_back(eb);
	}
	cudaStream_t sc = e->stream;
	FB_CUDA(cudaMemsetAsync(e->d_running, 0, 2 * sizeof(unsigned long long), sc));
	FB_CUDA(cudaMemsetAsync(e->d_err, 0, sizeof(int), sc));
	e->slice_mode = nfr <= e->max_blocks;
	{ const int rc = fork_stage_a(e, sc); if(rc != FB200_OK) return rc; }  // the error word is cleared before any kernel of this call may set it
	e->ev_b_valid[0] = e->ev_b_valid[1] = false;
	for(size_t ci = 0; ci < used; ci++) {
		PipeChunk &c = chunks[ci];
		const size_t off_elems = (size_t)c.first * bs * ch;
		const size_t nsamp = (size_t)c.nb * c.blocksize;
		if(!packed) FB_CUDA(cudaMemcpyAsync(e->d_pcm + off_elems, pcm_bytes_host + off_elems * 4, nsamp * ch * sizeof(int32_t), cudaMemcpyHostToDevice, e->s_h2d));
		else {
			// packed 16-/24-bit PCM crosses PCIe as it is; one unpack kernel widens it to the int32 layout the pipeline reads
			FB_CUDA(cudaMemcpyAsync(e->d_packed + off_elems * bytes_per_sample, pcm_bytes_host + off_elems * bytes_per_sample, nsamp * ch * bytes_per_sample, cudaMemcpyHostToDevice, e->s_h2d));
		}
		FB_CUDA(cudaEventRecord(e->ev_h2d[ci], e->s_h2d));
		c.wait_before_a = e->ev_h2d[ci];
		if(packed) {
			// the unpack kernel runs on the compute stream, so the copy stream carries nothing but copies (back to back)
			cudaStream_t sa = stage_a_stream(e, ci);
			FB_CUDA(cudaStreamWaitEvent(sa, e->ev_h2d[ci], 0));
			launch_unpack(e->d_packed + off_elems * bytes_per_sample, (int)bytes_per_sample, e->d_pcm + off_elems, (unsigned long long)nsamp * ch, (int)e->cfg.bits_per_sample, e->d_err, sa);
			e->launches++;
			c.wait_before_a = nullptr;
		}
		const int rc = enqueue_chunk(e, ci, c, e->d_pcm, first_frame_number, e->d_out, e->d_out_cap, e->d_offsets, sc);
		if(rc != FB200_OK) return rc;
		FB_CUDA(cudaMemcpyAsync(&e->h_totals[ci], e->d_running + e->run_cur, sizeof(unsigned long long), cudaMemcpyDeviceToHost, sc));
		FB_CUDA(cudaEventRecord(e->ev_comp[ci], sc));
	}
	unsigned long long prev = 0;
	for(size_t i = 0; i < used; i++) {
		FB_CUDA(cudaEventSynchronize(e->ev_comp[i]));
		const unsigned long long tot = e->h_totals[i];
		if(tot > out_capacity) { cudaStreamSynchronize(sc); set_error("output buffer too small: need more than %llu bytes", tot); return FB200_ERR_OUTPUT_TOO_SMALL; }
		if(tot > prev) FB_CUDA(cudaMemcpyAsync(out + prev, e->d_out + prev, (size_t)(tot - prev), cudaMemcpyDeviceToHost, e->s_d2h));
		prev = tot;
	}
	FB_CUDA(cudaMemcpyAsync(frame_offsets, e->d_offsets, (nfr + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->s_d2h));
	FB_CUDA(cudaStreamSynchronize(e->s_d2h));
	FB_CUDA(cudaStreamSynchronize(sc));
	int err = 0;
	FB_CUDA(cudaMemcpy(&err, e->d_err, sizeof err, cudaMemcpyDeviceToHost));
	if(err == 3) { set_error("a sample does not fit bits_per_sample"); return FB200_ERR_INVALID; }
	if(err == 2) { set_error("internal: frame exceeded its size bound"); return FB200_ERR_CUDA; }
	if(err) { set_error("internal output buffer too small"); return FB200_ERR_OUTPUT_TOO_SMALL; }
	return FB200_OK;
}

int fb200_encode_host(fb200_encoder *e, const int32_t *pcm, uint64_t samples, uint32_t first_frame_number,
                      uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint32_t *nframes)
{
	return encode_host_impl(e, pcm, 4, samples, first_frame_number, out, out_capacity, frame_offsets, nframes);
}

int fb200_encode_host_packed(fb200_encoder *e, const void *pcm, uint32_t bytes_per_sample, uint64_t samples, uint32_t first_frame_number,
                             uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint32_t *nframes)
{
	return encode_host_impl(e, pcm, bytes_per_sample, samples, first_frame_number, out, out_capacity, frame_offsets, nframes);
}

int fb200_encoder_set_file_blocks(fb200_encoder *e, uint32_t blocks_per_file)
{
	if(!e) return FB200_ERR_INVALID;
	e->file_blocks = blocks_per_file;
	return FB200_OK;
}

int fb200_encoder_set_profiling(fb200_encoder *e, int on)
{
	if(!e) return FB200_ERR_INVALID;
	cudaSetDevice(e->device);
	prof_resolve(e);
	e->prof_on = on != 0;
	return FB200_OK;
}

int fb200_encoder_get_profile(fb200_encoder *e, double ms[FB200_PROF_KERNELS], uint64_t launches[FB200_PROF_KERNELS], int reset)
{
	if(!e) return FB200_ERR_INVALID;
	cudaSetDevice(e->device);
	prof_resolve(e);
	for(int i = 0; i < FB200_PROF_KERNELS; i++) {
		if(ms) ms[i] = e->prof_ms[i];
		if(launches) launches[i] = e->prof_launches[i];
		if(reset) { e->prof_ms[i] = 0; e->prof_launches[i] = 0; }
	}
	return FB200_OK;
}

// device restatement of the host libm's log() vs the host's own (tests/test_gpu_log.py)
int fb200_debug_log(const double *x, double *y, uint32_t n, int device)
{
	if(!x || !y) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(device));
	double *dx = nullptr, *dy = nullptr;
	FB_CUDA(cudaMalloc(&dx, (size_t)n * sizeof(double)));
	FB_CUDA(cudaMalloc(&dy, (size_t)n * sizeof(double)));
	FB_CUDA(cudaMemcpy(dx, x, (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
	launch_debug_log(dx, dy, (int)n);
	FB_CUDA(cudaMemcpy(y, dy, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
	cudaFree(dx); cudaFree(dy);
	return FB200_OK;
}

// ---- debug/stage-level access for the parity tests (plans of the last launch) ----
int fb200_debug_copy_plans(fb200_encoder *e, uint32_t nblocks, void *host_plans, size_t plan_bytes, uint32_t *host_chan_assign)
{
	if(!e || !host_plans) return FB200_ERR_INVALID;
	if(plan_bytes != sizeof(SubframePlan)) { set_error("plan size mismatch %zu != %zu", plan_bytes, sizeof(SubframePlan)); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(e->device));
	FB_CUDA(cudaDeviceSynchronize());
	FB_CUDA(cudaMemcpy(host_plans, e->d_plans, (size_t)nblocks * e->nsig * sizeof(SubframePlan), cudaMemcpyDeviceToHost));
	if(host_chan_assign) FB_CUDA(cudaMemcpy(host_chan_assign, e->d_chan_assign, nblocks * sizeof(uint32_t), cudaMemcpyDeviceToHost));
	return FB200_OK;
}

}  // extern "C"
