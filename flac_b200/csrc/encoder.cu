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
#if defined(__x86_64__)
#include <cpuid.h>
#endif

#include "fb200_internal.h"
#include "flac_metadata.h"
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
	DevSection *d_secs = nullptr;
	DevCand *d_cands = nullptr;
	size_t search_smem = 0, emit_smem = 0;  // general kernels
	int fast_search3 = 0;       // 0, or R_T (32/36) of the fast search kernel (k_search5: CTA per block, warps per signal)
	int search_wps = 2;         // warps per signal in k_search5
	size_t search5_smem = 0;
	int maxord_t = 8;
	int emit3_rt = 0;           // 0, or R_T of the resident emit kernel (k_emit3)
	bool emit3_pair = false;    // more than two channels: k_emit3<PAIR> per channel pair + k_join per frame
	int pair_words = 0;         // words of a pair's staging region
	size_t pair_smem = 0, join_smem = 0;
	size_t emit3_smem = 0;
	// the general k_search / k_emit do not fit the device's shared memory: k_search_tiled / k_emit_tiled + k_join_tiled take
	// their blocks (FB200_DEBUG_PATH bit 16: take them anyway)
	bool tiled_search = false, tiled_emit = false;
	int sub_words = 0;          // words of a subframe's staging region (k_emit_tiled)
	uint32_t sub_cap_bits = 0;  // a subframe's size bound: max_frame_bytes_for's per-channel share
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
	uint32_t *d_tstage = nullptr, *d_tstage_bits = nullptr;  // per-subframe staging of the tiled emit path
	size_t d_tstage_words = 0;
	size_t smem_optin = 0;  // the device's sharedMemPerBlockOptin
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
	cudaStream_t s_a = nullptr;
	// slice mode (the call's blocks fit the workspace): every chunk owns its slice of workspace set 0, so the stage A's of
	// different chunks are independent and rotate over these streams (s_as[0] == s_a) -- the latency-bound autocorrelation of
	// a small chunk no longer serialises the pipeline
	static constexpr int kStageAStreams = 4;
	cudaStream_t s_as[kStageAStreams] = {};
	bool slice_mode = false;
	// the last call's full-block chunks (first block, blocks, StageA route) as stage A left them in workspace set 0 in slice
	// mode: only fb200_debug_copy_autoc reads this
	struct ChunkA { uint64_t first; uint32_t nb; int route; };
	std::vector<ChunkA> chunks_a;
	std::vector<cudaEvent_t> ev_ca;  // per chunk: stage A done
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
	// fb200_encode_files_*: the call's tables, frame numbers and digests (d_files), the file-major output of the host entry point
	// (d_fout), the MD5 stream and the per-block frame numbers the stage-B kernels read during such a call (else null)
	uint8_t *d_files = nullptr;
	size_t d_files_cap = 0;
	uint8_t *d_fout = nullptr;
	size_t d_fout_cap = 0;
	cudaStream_t s_md5 = nullptr;
	cudaEvent_t ev_md5_fork = nullptr, ev_md5_done = nullptr;
	cudaStream_t s_rg = nullptr;  // ReplayGain analysis of fb200_encode_pcm_files_*, forked like the MD5
	cudaEvent_t ev_rg_fork = nullptr;
	const uint32_t *files_frame_no = nullptr;
	// geometries of short last blocks built by fb200_encode_files_*: length -> number of the call that last used it. At most
	// kTailGeomCache stay between calls (least recently used go first): recurring lengths are not rebuilt, and a library of
	// thousands of distinct lengths does not pile up geometries.
	static constexpr size_t kTailGeomCache = 256;
	std::map<int, uint64_t> tail_geom_use;
	uint64_t files_calls = 0;
	// host staging of the files calls, kept across calls so that a batch carrying megabytes of metadata (cover art) does not
	// allocate and fault in fresh pages every call: the header plan of fb200_encode_flac_files_* and the one upload
	FlacHeaderPlan flac_plan;
	std::vector<uint8_t> files_upload;
	// verify (fb200_encoder_set_verify): k_dec_crc's table, the last files call's records (valid only if that call verified) and
	// the flips fb200_debug_perturb_verify queued for the next files call
	bool verify = false;
	uint16_t *d_vcrc_tab = nullptr;
	std::vector<fb200_file_verify_info> verify_info;
	bool verify_valid = false;
	struct Perturb { uint32_t file, what, a, b, mask; };
	std::vector<Perturb> perturb;
	cudaStream_t stream = nullptr, s_h2d = nullptr, s_d2h = nullptr;
	std::vector<cudaEvent_t> ev_h2d, ev_comp;
	unsigned long long *h_totals = nullptr;  // pinned
	size_t h_totals_cap = 0;
	uint64_t launches = 0;
	int host_chunks = 12;   // chunks per fb200_encode_host call (FB200_HOST_CHUNKS): copy/compute overlap granularity; on an H100 SXM at 400 W
	                        // (tools/sweep_host_chunks.py, packed 16-bit, 10 000 blocks) 8-16 are equal within noise and 4 / 24 are ~7 % slower at -8
	int pipe_chunks = 1;    // sub-batches per fb200_encode_device call (FB200_PIPE_CHUNKS); see fb200_encode_device
	int debug_path = 0;   // FB200_DEBUG_PATH bit mask (bisecting aid): 1 = k_prep + k_autoc3 instead of k_autoc4, 2 = general search, 4 = general emit,
	                      // 16 = the tiled kernels wherever the general search / emit would run
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
	k.x86_avx2_fixed_guess = c.x86_avx2_fixed_guess;
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
			const size_t need = rt ? search5_smem(bs, rt, gsz, wps, k.max_po, k.bps > 16) : 0;
			// k_search5 has no x86_avx2_fixed_guess branch and needs none: the blocksizes it takes are multiples of 32 * rt, so
			// bs - 4 is a multiple of 4, where the x86 AVX2 routine's fixed-guess sums equal the C routine's
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
	}
	// Where the general kernels would run but their signal / frame does not fit one CTA's shared memory, the tiled kernels
	// run instead. Strides come from the configured blocksize, so a short last block goes the way its full blocks go.
	g.tiled_search = g.search_smem + 8192 > e->smem_optin;
	g.tiled_emit = g.emit_smem + 4096 > e->smem_optin;
	{
		const size_t per_ch = ((size_t)c.blocksize * (c.bits_per_sample + 2) + 7) / 8 + 256;  // as max_frame_bytes_for
		g.sub_cap_bits = (uint32_t)(per_ch * 8);
		g.sub_words = round_up((int)(per_ch / 4) + 2, 4);
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

// What a chunk runs, decided once per chunk. k_autoc4, k_search5 and k_emit3 copy raw blocks of the caller's PCM with TMA, so
// a chunk that starts off 16 bytes (the short last block behind an odd blocksize x channels) takes the planar kernels.
enum class StageA {
	fused = FB200_STAGE_A_FUSED,    // k_autoc4 on the caller's PCM collects the wasted-bits OR on the way; k_lpc derives wasted bits from it
	meta = FB200_STAGE_A_META,      // k_meta first (no LPC analysis, or loose mid-side: k_autoc4 reads the meta to skip the inactive pair), then k_autoc4
	planar = FB200_STAGE_A_PLANAR,  // k_prep's planar copy, then k_autoc3
};
enum class Kernel { fast, tiled, general };  // search: k_search5 / tiled / general; emit: k_emit3 / tiled / general + k_scan + k_gather
struct Route { StageA a; Kernel search, emit; };

static Route route_chunk(const fb200_encoder *e, const Geometry &g, const int32_t *pcm)
{
	const int dbg = e->debug_path;
	const bool aligned = ((uintptr_t)pcm & 15) == 0;
	Route r;
	r.search = g.fast_search3 && aligned && !(dbg & 2) ? Kernel::fast : g.tiled_search || (dbg & 16) ? Kernel::tiled : Kernel::general;
	r.emit = g.emit3_rt && aligned && !(dbg & 4) ? Kernel::fast : g.tiled_emit || (dbg & 16) ? Kernel::tiled : Kernel::general;
	// stage A may skip the planar copy only when the search and the emit both read the caller's PCM
	if(r.search != Kernel::fast || r.emit != Kernel::fast || (dbg & 1)) r.a = StageA::planar;
	else r.a = g.k.nwin > 0 && !g.k.loose_ms ? StageA::fused : StageA::meta;
	return r;
}

// Stage A of nb blocks of size g.bs starting at d_pcm: k_prep / k_meta, k_autoc4 / k_autoc3, k_lpc (writes the current
// workspace set).
static int run_stage_a(fb200_encoder *e, Geometry &g, StageA how, const int32_t *d_pcm, int nb, cudaStream_t st)
{
	EncK k = g.k;
	const int nitems = nb * k.nsig;
	const bool fused = how == StageA::fused;
	prof_mark(e, -1, st);
	if(how == StageA::meta) launch_meta(k, d_pcm, e->d_meta, e->d_blkflags, nb, st);
	else if(how == StageA::planar) launch_prep(k, d_pcm, e->d_sig, e->d_meta, e->d_blkflags, nb, st);
	prof_mark(e, FB200_PROF_PREP, st);
	if(!fused) e->launches++;
	if(k.nwin > 0) {
		// k_autoc4 ORs section 0's samples: every apodization opens with its full-length section
		if(how == StageA::planar) launch_autoc3(k, e->d_sig, e->d_meta, g.d_windows, g.d_secs, e->d_autoc, nitems, st);
		else launch_autoc4(k, d_pcm, fused ? nullptr : e->d_meta, g.d_secwin, bs_plus_slack(k.bs), g.d_secs, e->d_autoc, nitems, fused ? e->d_sigor : nullptr, 0, st);
		prof_mark(e, FB200_PROF_AUTOC, st);
		launch_lpc(k, e->d_autoc, g.d_cands, e->d_meta, fused ? e->d_sigor : nullptr, e->d_cdesc, nitems, fused ? 1 : 0, st);
		prof_mark(e, FB200_PROF_LPC, st);
		e->launches += 2;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

// Grows a pair of stage-B staging arrays to `regions` regions of `words` words and one bit count per region. Growing
// synchronises `st` first (once per geometry): kernels queued on it may still use the old arrays.
static int grow_staging(cudaStream_t st, uint32_t **d_words, uint32_t **d_bits, size_t *cap_words, size_t regions, size_t words)
{
	const size_t need = regions * words;
	if(need <= *cap_words) return FB200_OK;
	FB_CUDA(cudaStreamSynchronize(st));
	cudaFree(*d_words); cudaFree(*d_bits); *d_words = nullptr; *d_bits = nullptr; *cap_words = 0;
	FB_CUDA(cudaMalloc(d_words, need * sizeof(uint32_t)));
	FB_CUDA(cudaMalloc(d_bits, regions * sizeof(uint32_t)));
	*cap_words = need;
	return FB200_OK;
}

// Stage B: search + emit (reads the current workspace set). k_emit3 writes frames straight to their final offsets; the tiled
// and general emits write slots that k_scan + k_gather place.
static int run_stage_b(fb200_encoder *e, Geometry &g, const Route &r, const int32_t *d_pcm, int nb, uint32_t first_frame, uint64_t frame_index0,
                       uint8_t *d_out, size_t out_cap, unsigned long long *d_offsets, cudaStream_t st)
{
	EncK k = g.k;
	k.first_frame = first_frame;
	k.blk0 = (uint32_t)frame_index0;
	k.file_blocks = (int)e->file_blocks;
	k.frame_no = e->files_frame_no;
	const int nitems = nb * k.nsig;
	int rc;
	prof_mark(e, -1, st);
	auto search = [&](const EncK &kk) {
		if(r.search == Kernel::fast) launch_search5(kk, g.fast_search3, g.maxord_t, g.search_wps, g.search5_smem, d_pcm, e->d_meta, e->d_cdesc, e->d_plans, nb, st);
		else if(r.search == Kernel::tiled) launch_search_tiled(kk, e->d_sig, e->d_meta, e->d_cdesc, e->d_plans, nitems, st);
		else launch_search_general(kk, g.search_smem, e->d_sig, e->d_meta, e->d_cdesc, e->d_plans, nitems, st);
	};
	search(k);
	if(k.limit_min_bitrate && k.channels > 1 && !k.dis_const) {
		// stream_encoder.c:3874-3879: blocks whose channels 0 .. n-2 all came out constant search their last channel (and mid /
		// side) again with constant subframes disabled
		launch_minbr_flags(k, e->d_plans, k.loose_ms ? e->d_blkflags : nullptr, nb, e->d_redo, st);
		EncK k2 = k;
		k2.dis_const = 1;
		k2.redo = e->d_redo;
		search(k2);
		e->launches += 2;
	}
	prof_mark(e, FB200_PROF_SEARCH, st);
	if(r.emit == Kernel::fast) {
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
			const size_t regions = (size_t)e->max_blocks * (((size_t)k.channels + 1) / 2);
			if((rc = grow_staging(st, &e->d_stage, &e->d_stage_bits, &e->d_stage_words, regions, (size_t)g.pair_words)) != FB200_OK) return rc;
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
		if(r.emit == Kernel::tiled) {
			const size_t regions = (size_t)e->max_blocks * k.channels;
			if((rc = grow_staging(st, &e->d_tstage, &e->d_tstage_bits, &e->d_tstage_words, regions, (size_t)g.sub_words)) != FB200_OK) return rc;
			launch_emit_tiled(k, e->d_sig, e->d_blkflags, e->d_plans, e->d_tstage, e->d_tstage_bits, g.sub_words, g.sub_cap_bits, e->d_slots,
			                  e->d_frame_bytes, e->d_chan_assign, e->d_err, nb, st);
			e->launches++;
		}
		else launch_emit_general(k, g.emit_smem, e->d_sig, e->d_blkflags, e->d_plans, e->d_slots, e->d_frame_bytes, e->d_chan_assign, nb, st);
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

// pcm: the chunk's first sample, or null for d_pcm_base + first full blocks (a group of short tails lies elsewhere)
struct PipeChunk { uint64_t first; uint32_t nb; uint32_t blocksize; cudaEvent_t wait_before_a; const int32_t *pcm = nullptr; };

// A call's nfull full blocks in chunks of ceil(nfull / parts) blocks, at least min_chunk and at most max_blocks each. The
// caller appends its short blocks.
static std::vector<PipeChunk> full_block_chunks(const fb200_encoder *e, uint64_t nfull, int parts, uint64_t min_chunk)
{
	uint64_t chunk = (nfull + parts - 1) / parts;
	if(chunk < min_chunk) chunk = min_chunk;
	if(chunk > e->max_blocks) chunk = e->max_blocks;
	std::vector<PipeChunk> chunks;
	for(uint64_t done = 0; done < nfull; done += chunk)
		chunks.push_back(PipeChunk{done, (uint32_t)((nfull - done) < chunk ? (nfull - done) : chunk), e->cfg.blocksize, nullptr});
	return chunks;
}

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
	const int32_t *pcm = c.pcm ? c.pcm : d_pcm_base + (size_t)c.first * bs * ch;
	const Route r = route_chunk(e, *g, pcm);
	if(c.blocksize == e->cfg.blocksize) e->chunks_a.push_back(fb200_encoder::ChunkA{c.first, c.nb, (int)r.a});
	if((rc = run_stage_a(e, *g, r.a, pcm, (int)c.nb, sa)) != FB200_OK) return rc;
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
	if((rc = run_stage_b(e, *g, r, pcm, (int)c.nb, first_frame_number, c.first, d_out, out_cap, d_offsets, sb)) != FB200_OK) return rc;
	if(!e->slice_mode) {
		FB_CUDA(cudaEventRecord(e->ev_b[b], sb));
		e->ev_b_valid[b] = true;
	}
	return FB200_OK;
}

// Starts a call's pipeline of nblocks blocks after its set-up work was enqueued on `st`: slice mode when the blocks fit the
// workspace, every stage-A stream of that mode behind `st`, and no wait on a previous call's stage B.
static int fork_stage_a(fb200_encoder *e, uint64_t nblocks, cudaStream_t st)
{
	e->slice_mode = nblocks <= e->max_blocks;
	e->chunks_a.clear();
	FB_CUDA(cudaEventRecord(e->ev_fork, st));
	for(int i = 0; i < (e->slice_mode ? fb200_encoder::kStageAStreams : 1); i++) FB_CUDA(cudaStreamWaitEvent(e->s_as[i], e->ev_fork, 0));
	e->ev_b_valid[0] = e->ev_b_valid[1] = false;
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

// x86_cpu_info (cpu.c:151-200) as an x86-64 libFLAC built with AVX support runs it: cpuinfo.x86.avx2, and with it the AVX2
// fixed-order guess (stream_encoder.c:1085-1090), needs AVX and OSXSAVE in CPUID leaf 1 ECX, the OS saving the XMM and YMM
// state (XCR0 bits 1 and 2) and AVX2 in leaf 7 EBX. cpuinfo_x86 reads a leaf above the maximum as zeros.
int fb200_host_x86_avx2_fixed_guess(void)
{
#if defined(__x86_64__)
	const unsigned max_leaf = __get_cpuid_max(0, nullptr);
	unsigned a, b, c, d;
	if(max_leaf < 7) return 0;
	__cpuid_count(1, 0, a, b, c, d);
	if(!(c & (1u << 28)) || !(c & (1u << 27))) return 0;
	unsigned xcr0_lo, xcr0_hi;
	__asm__ volatile(".byte 0x0f, 0x01, 0xd0" : "=a"(xcr0_lo), "=d"(xcr0_hi) : "c"(0));  // XGETBV(0)
	(void)a; (void)d; (void)xcr0_hi;
	if((xcr0_lo & 6u) != 6u) return 0;
	__cpuid_count(7, 0, a, b, c, d);
	return (b & (1u << 5)) ? 1 : 0;
#else
	return 0;
#endif
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

static int create_impl(const fb200_encoder_config *cfg_in, int device, uint32_t max_blocks, bool bound_tiled, fb200_encoder **out)
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
	if(c.x86_avx2_fixed_guess != 0 && c.x86_avx2_fixed_guess != 1) { set_error("invalid x86_avx2_fixed_guess %d (0 or 1)", c.x86_avx2_fixed_guess); return FB200_ERR_INVALID; }

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
	{
		cudaDeviceProp prop;
		cudaGetDeviceProperties(&prop, device);
		e->smem_optin = prop.sharedMemPerBlockOptin;
	}
	e->nsig =(int)c.channels + ((c.channels == 2 && c.do_mid_side_stereo) ? 2 : 0);
	{
		e->lag_stride = (size_t)autoc_kernel_lags((int)c.max_lpc_order + 1);
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
	Geometry *g = nullptr;
	{
		const int rc = build_geometry(e, (int)c.blocksize, &g);
		if(rc != FB200_OK) { fb200_encoder_destroy(e); return rc; }
	}
	{
		// a configuration on the tiled path holds frames of up to 65535 x 8 samples: its default capacity comes from a sample
		// budget instead of a block count (4096 such blocks would need ~17 GB for the planar signals alone)
		const bool tiled = (g->tiled_search && !g->fast_search3) || (g->tiled_emit && !g->emit3_rt);
		uint32_t budget = (uint32_t)(FB200_TILED_SAMPLE_BUDGET / ((uint64_t)c.blocksize * c.channels));
		budget = budget < 1 ? 1 : budget > 4096 ? 4096 : budget;
		e->max_blocks = max_blocks ? max_blocks : 4096;
		if(tiled && (max_blocks == 0 || (bound_tiled && max_blocks > budget))) e->max_blocks = budget;
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
	if(!streams_ok || cudaEventCreateWithFlags(&e->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
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
			tiled_init(device);
			inited[device] = true;
		}
	}
	{
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

int fb200_encoder_create(const fb200_encoder_config *cfg, int device, uint32_t max_blocks, fb200_encoder **out)
{
	return create_impl(cfg, device, max_blocks, false, out);
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
	cudaFree(e->d_plans); cudaFree(e->d_slots); cudaFree(e->d_frame_bytes); cudaFree(e->d_chan_assign);
	cudaFree(e->d_running); cudaFree(e->d_err); cudaFree(e->d_redo); cudaFree(e->d_stage); cudaFree(e->d_stage_bits);
	cudaFree(e->d_tstage); cudaFree(e->d_tstage_bits);
	cudaFree(e->d_crc_tab); cudaFree(e->d_lookback); cudaFree(e->d_ticket);
	cudaFree(e->d_pcm); cudaFree(e->d_packed); cudaFree(e->d_out); cudaFree(e->d_offsets);
	cudaFree(e->d_files); cudaFree(e->d_fout); cudaFree(e->d_vcrc_tab);
	if(e->s_md5) cudaStreamDestroy(e->s_md5);
	if(e->ev_md5_fork) cudaEventDestroy(e->ev_md5_fork);
	if(e->ev_md5_done) cudaEventDestroy(e->ev_md5_done);
	if(e->s_rg) cudaStreamDestroy(e->s_rg);
	if(e->ev_rg_fork) cudaEventDestroy(e->ev_rg_fork);
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

// The block entry points are not verified: fb200_encode_device writes into the caller's buffer, which the decode kernels' bit
// reader may not read past. With verify on they refuse rather than return unchecked frames.
static int refuse_unverified()
{
	set_error("verify is on: only fb200_encode_files_host / _device verify their frames; turn verify off for the block entry points");
	return FB200_ERR_UNSUPPORTED;
}

int fb200_encode_device(fb200_encoder *e, const int32_t *d_pcm, uint64_t samples, uint32_t first_frame_number,
                        uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint32_t *nframes,
                        uint64_t *total_bytes, void *cuda_stream, int sync)
{
	if(!e || !d_pcm || !d_out || !d_frame_offsets) return FB200_ERR_INVALID;
	if(e->verify) return refuse_unverified();
	FB_CUDA(cudaSetDevice(e->device));
	cudaStream_t st = (cudaStream_t)cuda_stream;
	const uint32_t bs = e->cfg.blocksize;
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
	std::vector<PipeChunk> chunks = full_block_chunks(e, nfull, e->pipe_chunks, 512);
	if(tail) chunks.push_back(PipeChunk{nfull, 1, tail, nullptr});  // short last block: own windows / header blocksize (stream_encoder.c:1703-1711)
	{ const int rc = fork_stage_a(e, nfull + (tail ? 1 : 0), st); if(rc != FB200_OK) return rc; }
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
	if(e->verify) return refuse_unverified();
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
	std::vector<PipeChunk> chunks = full_block_chunks(e, nfull, e->host_chunks, 256);
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
	{ const int rc = fork_stage_a(e, nfr, sc); if(rc != FB200_OK) return rc; }  // the error word is cleared before any kernel of this call may set it
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

// grow-only device buffer (kept across calls)
static int grow(void **p, size_t *cap, size_t need)
{
	if(need <= *cap) return FB200_OK;
	cudaFree(*p);
	*p = nullptr;
	*cap = 0;
	FB_CUDA(cudaMalloc(p, need));
	*cap = need;
	return FB200_OK;
}

static size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

// fb200_encode_files_host / _device. Encode order: every file's full blocks (file by file: one block-major region, the layout
// the kernels read for a single stream), then the tails grouped by length. The full blocks run in the chunks of
// fb200_encode_device, each tail length in launches of up to max_blocks blocks; per-block frame numbers number every file from 0.
// k_files_gather then writes each file's frames together, file after file. The host entry point copies the whole input before
// the first kernel (no copy / compute overlap). k_flac_file_headers then builds every file's STREAMINFO; with flac_files
// (fb200_encode_flac_files_*) each file's frames start after room for its header, which the same kernel writes there.
static int encode_files_impl(fb200_encoder *e, const void *pcm, uint32_t bytes_per_sample, bool device, const uint64_t *file_samples, uint32_t nfiles,
                             int do_md5, const uint8_t *metadata, const uint64_t *metadata_offsets, uint8_t *out, size_t out_capacity,
                             uint64_t *frame_offsets, uint64_t *nframes, fb200_file_info *files, fb200_flac_file_info *flac_files, cudaStream_t st,
                             const PcmSource *pcm_src = nullptr)
{
	if(!e) return FB200_ERR_INVALID;
	e->verify_valid = false;
	std::vector<fb200_encoder::Perturb> perturb;  // queued for this call only
	perturb.swap(e->perturb);
	const bool flac = flac_files != nullptr;
	if(!pcm || !file_samples || !out || (!frame_offsets && !flac) || !nframes || (!files && !flac)) return FB200_ERR_INVALID;
	if(nfiles == 0) { set_error("no files"); return FB200_ERR_INVALID; }
	if(flac && !metadata != !metadata_offsets) { set_error("metadata and metadata_offsets must both be given or both be NULL"); return FB200_ERR_INVALID; }
	FlacHeaderPlan &plan = e->flac_plan;
	plan.heads.clear();
	plan.pts.clear();
	plan.blob.clear();
	if(flac) {
		const int rc = plan_flac_headers(metadata, metadata_offsets, nfiles, &plan);
		if(rc != FB200_OK) return rc;
	}
	const ReplayGainJob *rg = pcm_src ? pcm_src->rg : nullptr;
	// ReplayGain's tag edits make each header at most this much longer once the analysis is in
	const size_t rg_slack = rg ? 190 * (size_t)nfiles : 0;
	unsigned long long header_bytes = rg_slack;
	for(const FlacHead &h : plan.heads) header_bytes += h.bytes;
	if(!perturb.empty() && do_md5) { set_error("a verify perturbation cannot be combined with MD5 (both read the input copy)"); return FB200_ERR_INVALID; }
	if(bytes_per_sample != 2 && bytes_per_sample != 3 && bytes_per_sample != 4) { set_error("bytes_per_sample must be 2, 3 or 4"); return FB200_ERR_INVALID; }
	if(e->cfg.bits_per_sample > 8 * bytes_per_sample) { set_error("%u-bit samples do not fit %u bytes", e->cfg.bits_per_sample, bytes_per_sample); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(e->device));
	const uint64_t bs = e->cfg.blocksize, ch = e->cfg.channels;
	std::map<uint32_t, std::vector<uint32_t>> groups;  // tail length -> its files, in file order
	uint64_t nfull_all = 0, in_elems = 0;
	for(uint32_t f = 0; f < nfiles; f++) {
		if(file_samples[f] == 0) { set_error("file %u has no samples", f); return FB200_ERR_INVALID; }
		nfull_all += file_samples[f] / bs;
		if(file_samples[f] % bs) groups[(uint32_t)(file_samples[f] % bs)].push_back(f);
		in_elems += file_samples[f] * ch;
	}
	uint64_t nv = nfull_all;
	for(auto &g : groups) nv += g.second.size();
	// one k_files_gather CTA per frame (grid.x < 2^31); nfiles and frame indices are int / uint32 in the kernels
	// (+ one CTA per file for the headers of fb200_encode_flac_files_*)
	if(nv + (flac ? nfiles : 0) >= 0x7fffffffull || nfiles >= 0x7fffffffu) { set_error("too many frames or files in one call"); return FB200_ERR_INVALID; }

	// ---- host tables: segments, frames per file, output order, frame numbers, chunks
	std::vector<FileSeg> segs(2 * (size_t)nfiles);
	std::vector<FileFrames> ff(nfiles);
	std::vector<uint32_t> frame_no(nv);
	{
		uint64_t src = 0, fb = 0;
		for(uint32_t f = 0; f < nfiles; f++) {
			const uint64_t nfull = file_samples[f] / bs;
			segs[2 * f] = FileSeg{src, fb * bs * ch, nfull * bs * ch, 0};
			segs[2 * f + 1] = FileSeg{src + nfull * bs * ch, 0, 0, 0};
			ff[f] = FileFrames{(uint32_t)fb, (uint32_t)nfull, ~0u};
			for(uint64_t j = 0; j < nfull; j++) frame_no[fb + j] = (uint32_t)j;
			src += file_samples[f] * ch;
			fb += nfull;
		}
	}
	std::vector<PipeChunk> chunks = full_block_chunks(e, nfull_all, e->pipe_chunks, 512);
	const size_t nfull_chunks = chunks.size();
	std::vector<uint64_t> tail_pcm;  // element offset of each tail chunk in the compacted layout
	uint64_t compact = nfull_all * bs * ch;
	{
		uint64_t v = nfull_all;
		for(auto &g : groups) {
			const uint64_t t = g.first, n = g.second.size();
			compact = (compact + 3) & ~3ull;  // every group starts 16-byte aligned, as the fast kernels' bulk copies need
			for(uint64_t done = 0; done < n; done += e->max_blocks) {
				chunks.push_back(PipeChunk{v + done, (uint32_t)((n - done) < e->max_blocks ? (n - done) : e->max_blocks), (uint32_t)t, nullptr});
				tail_pcm.push_back(compact + done * t * ch);
			}
			for(uint32_t f : g.second) {
				segs[2 * f + 1].dst = compact;
				segs[2 * f + 1].n = t * ch;
				ff[f].tail = (uint32_t)v;
				frame_no[v] = ff[f].nfull;
				v++;
				compact += t * ch;
			}
		}
	}
	std::vector<RgFileDev> rgf(rg ? nfiles : 0);
	uint64_t rg_nwin = 0;
	for(uint32_t f = 0; f < rgf.size(); f++) {
		RgFileDev &R = rgf[f];
		R = RgFileDev{segs[2 * f].dst, segs[2 * f].n / ch, segs[2 * f + 1].dst, file_samples[f], rg_nwin, (uint32_t)ch, rg->bps[f], rg->ds, rg->W,
		              rg->filt, 0};
		rg_nwin += R.n / R.ds / R.W;
	}
	unsigned long long items = 0;
	for(FileSeg &s : segs) {
		s.item0 = items;
		items += (s.n + kUnpackFilesItem - 1) / kUnpackFilesItem;
	}
	std::vector<uint2> order;  // output frame -> (frame in encode order, file)
	order.reserve(nv);
	for(uint32_t f = 0; f < nfiles; f++) {
		for(uint32_t j = 0; j < ff[f].nfull; j++) order.push_back(make_uint2(ff[f].first + j, f));
		if(ff[f].tail != ~0u) order.push_back(make_uint2(ff[f].tail, f));
	}
	// the queued flips as places: a frame in encode order (what 0) or an element of the compacted input (what 1)
	std::vector<unsigned long long> flip_at(perturb.size());
	for(size_t i = 0; i < perturb.size(); i++) {
		const fb200_encoder::Perturb &p = perturb[i];
		bool ok = p.file < nfiles && p.what <= 1;
		if(ok && p.what == 0) {
			const FileFrames &F = ff[p.file];
			ok = p.a < F.nfull || (p.a == F.nfull && F.tail != ~0u);
			if(ok) flip_at[i] = p.a < F.nfull ? F.first + p.a : F.tail;
		}
		else if(ok) {
			ok = p.a < file_samples[p.file] && p.b < ch;
			const uint64_t full = (uint64_t)ff[p.file].nfull * bs;
			if(ok) flip_at[i] = p.a < full ? segs[2 * p.file].dst + p.a * ch + p.b : segs[2 * p.file + 1].dst + (p.a - full) * ch + p.b;
		}
		if(!ok) { set_error("verify perturbation %zu names no frame / sample of this call", i); return FB200_ERR_INVALID; }
	}

	// ---- device memory, all of it before the first launch
	size_t o = 0;
	const size_t o_segs = o; o = align16(o + segs.size() * sizeof(FileSeg));
	const size_t o_ff = o; o = align16(o + ff.size() * sizeof(FileFrames));
	const size_t o_order = o; o = align16(o + order.size() * sizeof(uint2));
	const size_t o_fno = o; o = align16(o + frame_no.size() * sizeof(uint32_t));
	const size_t o_pcmf = o; o = pcm_src ? align16(o + pcm_src->files.size() * sizeof(PcmFileDev)) : o;
	const size_t o_heads = o; o = align16(o + plan.heads.size() * sizeof(FlacHead));
	const size_t o_pts = o; o = align16(o + plan.pts.size() * sizeof(SeekPt));
	const size_t o_hblob = o; o = align16(o + plan.blob.size() + rg_slack + 4);  // + 4: k_files_gather reads whole words
	const size_t o_rgf = o; o = align16(o + rgf.size() * sizeof(RgFileDev));
	const size_t upload = o;
	const size_t o_si = o; o = align16(o + 34 * (size_t)nfiles);
	const size_t o_fbase = o; o = align16(o + (size_t)nfiles * sizeof(unsigned long long));
	const size_t o_voff = o; o = align16(o + (nv + 1) * sizeof(unsigned long long));
	const size_t o_foff = o; o = align16(o + (nv + 1) * sizeof(unsigned long long));
	const size_t o_md5 = o; o += 16 * (size_t)nfiles;  // digests, then the unpack error word
	const size_t o_err = o; o += 16;
	const size_t o_bad = o; o += 16;  // k_pcm_unpack's first failing value
	const size_t o_rgpk = o; o = align16(o + rgf.size() * sizeof(uint32_t));  // ReplayGain: each file's peak, every window's v
	const size_t o_rgv = o; o = align16(o + rg_nwin * sizeof(double));
	// verify: clamped frame bounds, the decoder's record and the verdict of every frame (encode order), one record per file
	const bool verify = e->verify;
	const size_t o_vb = o; o = verify ? align16(o + (nv + 1) * sizeof(unsigned long long)) : o;
	const size_t o_vmeta = o; o = verify ? align16(o + (size_t)nv * verify_meta_bytes()) : o;
	const size_t o_verd = o; o = verify ? align16(o + (size_t)nv * sizeof(DecVerdict)) : o;
	const size_t o_vinfo = o; o = verify ? align16(o + (size_t)nfiles * sizeof(fb200_file_verify_info)) : o;
	const uint64_t ntails = nv - nfull_all;  // the tails' input, one configured block per tail: one verify launch set for them all
	const size_t o_vtail = o; o = verify ? align16(o + (size_t)ntails * bs * ch * sizeof(int32_t)) : o;
	// fb200_reencode_flac_files_*: the gather's and the headers' tables over the files check() keeps
	const bool fill = pcm_src && pcm_src->fill;
	const size_t o_kff = o; o = fill ? align16(o + ff.size() * sizeof(FileFrames)) : o;
	const size_t o_korder = o; o = fill ? align16(o + order.size() * sizeof(uint2)) : o;
	const size_t o_ksegs = o; o = fill ? align16(o + segs.size() * sizeof(FileSeg)) : o;
	const size_t o_kheads = o; o = fill ? align16(o + plan.heads.size() * sizeof(FlacHead)) : o;
	const size_t o_kmd5 = o; o = fill ? align16(o + 16 * (size_t)nfiles) : o;
	std::vector<uint8_t> &blob = e->files_upload;
	if(blob.size() < upload) blob.resize(upload);
	memcpy(blob.data() + o_segs, segs.data(), segs.size() * sizeof(FileSeg));
	memcpy(blob.data() + o_ff, ff.data(), ff.size() * sizeof(FileFrames));
	memcpy(blob.data() + o_order, order.data(), order.size() * sizeof(uint2));
	memcpy(blob.data() + o_fno, frame_no.data(), frame_no.size() * sizeof(uint32_t));
	if(pcm_src) memcpy(blob.data() + o_pcmf, pcm_src->files.data(), pcm_src->files.size() * sizeof(PcmFileDev));
	if(rg) memcpy(blob.data() + o_rgf, rgf.data(), rgf.size() * sizeof(RgFileDev));
	if(flac) {
		memcpy(blob.data() + o_heads, plan.heads.data(), plan.heads.size() * sizeof(FlacHead));
		memcpy(blob.data() + o_pts, plan.pts.data(), plan.pts.size() * sizeof(SeekPt));
		memcpy(blob.data() + o_hblob, plan.blob.data(), plan.blob.size());
	}
	const size_t need_out = (size_t)nv * max_frame_bytes_for(e->cfg, (int)bs) + header_bytes + 64;
	const size_t vcap = out_capacity < need_out ? out_capacity : need_out;  // the encode-order stream is exactly as long as the output
	int rc;
	if((rc = grow((void **)&e->d_files, &e->d_files_cap, o)) != FB200_OK) return rc;
	if((rc = grow((void **)&e->d_pcm, &e->d_pcm_cap, (size_t)compact * sizeof(int32_t) + 256)) != FB200_OK) return rc;
	if((rc = grow((void **)&e->d_out, &e->d_out_cap, vcap + 64)) != FB200_OK) return rc;  // + 64: k_files_gather reads whole words
	if(!device) {
		const size_t in_bytes = pcm_src ? (size_t)pcm_src->bytes : (size_t)in_elems * bytes_per_sample;
		if((rc = grow((void **)&e->d_packed, &e->d_packed_cap, in_bytes + 256)) != FB200_OK) return rc;
		if((rc = grow((void **)&e->d_fout, &e->d_fout_cap, vcap + 64)) != FB200_OK) return rc;
	}
	if(do_md5 && !fill && !e->s_md5) {
		FB_CUDA(cudaStreamCreateWithFlags(&e->s_md5, cudaStreamNonBlocking));
		FB_CUDA(cudaEventCreateWithFlags(&e->ev_md5_fork, cudaEventDisableTiming));
		FB_CUDA(cudaEventCreateWithFlags(&e->ev_md5_done, cudaEventDisableTiming));
	}
	if(rg && !e->s_rg) {
		FB_CUDA(cudaStreamCreateWithFlags(&e->s_rg, cudaStreamNonBlocking));
		FB_CUDA(cudaEventCreateWithFlags(&e->ev_rg_fork, cudaEventDisableTiming));
	}
	// The tail lengths' geometries are built now, so that no allocation lands between launches. When the call ends (after its
	// last synchronise) the least recently used ones beyond kTailGeomCache are freed.
	struct Cleanup {
		fb200_encoder *e;
		cudaStream_t st;
		std::vector<int> used;
		~Cleanup()
		{
			cudaStreamSynchronize(st);
			for(int i = 0; i < fb200_encoder::kStageAStreams; i++) cudaStreamSynchronize(e->s_as[i]);
			if(e->s_md5) cudaStreamSynchronize(e->s_md5);
			if(e->s_rg) cudaStreamSynchronize(e->s_rg);
			e->files_frame_no = nullptr;
			const uint64_t call = ++e->files_calls;
			for(int t : used) e->tail_geom_use[t] = call;
			while(e->tail_geom_use.size() > fb200_encoder::kTailGeomCache) {
				auto lru = e->tail_geom_use.begin();
				for(auto it = e->tail_geom_use.begin(); it != e->tail_geom_use.end(); ++it)
					if(it->second < lru->second) lru = it;
				auto g = e->geoms.find(lru->first);
				if(g != e->geoms.end()) {
					cudaFree(g->second.d_windows); cudaFree(g->second.d_secs); cudaFree(g->second.d_cands); cudaFree(g->second.d_secwin);
					e->geoms.erase(g);
				}
				e->tail_geom_use.erase(lru);
			}
		}
	} cleanup{e, st, {}};
	for(auto &g : groups) {
		Geometry *geo = nullptr;
		if((rc = build_geometry(e, (int)g.first, &geo)) != FB200_OK) return rc;
		cleanup.used.push_back((int)g.first);
	}
	for(size_t i = nfull_chunks; i < chunks.size(); i++) chunks[i].pcm = e->d_pcm + tail_pcm[i - nfull_chunks];

	// ---- launches
	uint8_t *const d = e->d_files;
	const FileSeg *d_segs = reinterpret_cast<const FileSeg *>(d + o_segs);
	unsigned long long *d_voff = reinterpret_cast<unsigned long long *>(d + o_voff);
	int *d_uerr = reinterpret_cast<int *>(d + o_err);
	FB_CUDA(cudaMemcpyAsync(d, blob.data(), upload, cudaMemcpyHostToDevice, st));
	FB_CUDA(cudaMemsetAsync(d + o_md5, 0, 16 * (size_t)nfiles + 16, st));
	FB_CUDA(cudaMemsetAsync(e->d_running, 0, 2 * sizeof(unsigned long long), st));
	FB_CUDA(cudaMemsetAsync(e->d_err, 0, sizeof(int), st));
	unsigned long long *d_bad = reinterpret_cast<unsigned long long *>(d + o_bad);
	const void *in = pcm;
	if(!device && !fill) {
		FB_CUDA(cudaMemcpyAsync(e->d_packed, pcm, pcm_src ? (size_t)pcm_src->bytes : (size_t)in_elems * bytes_per_sample, cudaMemcpyHostToDevice, st));
		in = e->d_packed;
	}
	std::vector<uint8_t> keep(nfiles, 1);
	if(fill) {
		// decoded in place of the unpack; the MD5 before the encode, so that check() can drop damaged and mismatching files
		FB_CUDA(cudaMemsetAsync(d_bad, 0xFF, sizeof *d_bad, st));
		if((rc = pcm_src->fill(pcm_src->ctx, e->d_pcm, compact, d_segs, st)) != FB200_OK) return rc;
		launch_md5_files(e->d_pcm, d_segs, (int)nfiles, (int)(e->cfg.bits_per_sample + 7) / 8, d + o_md5, st);
		e->launches++;
		if((rc = pcm_src->check(pcm_src->ctx, d + o_md5, st, &keep)) != FB200_OK) return rc;
	}
	else if(pcm_src) {
		FB_CUDA(cudaMemsetAsync(d_bad, 0xFF, sizeof *d_bad, st));
		prof_mark(e, -1, st);
		launch_pcm_unpack(static_cast<const uint8_t *>(in), pcm_src->bytes, reinterpret_cast<const PcmFileDev *>(d + o_pcmf), d_segs, (int)segs.size(), items,
		                  e->d_pcm, d_bad, st);
		prof_mark(e, FB200_PROF_PREP, st);
	}
	else launch_unpack_files(in, (int)bytes_per_sample, d_segs, (int)segs.size(), items, e->d_pcm, (int)e->cfg.bits_per_sample, d_uerr, st);
	if(!fill) e->launches++;
	if(do_md5 && !fill) {  // concurrently with the encode; joined before the results are read
		FB_CUDA(cudaEventRecord(e->ev_md5_fork, st));
		FB_CUDA(cudaStreamWaitEvent(e->s_md5, e->ev_md5_fork, 0));
		launch_md5_files(e->d_pcm, d_segs, (int)nfiles, (int)(e->cfg.bits_per_sample + 7) / 8, d + o_md5, e->s_md5);
		FB_CUDA(cudaEventRecord(e->ev_md5_done, e->s_md5));
		e->launches++;
	}
	if(rg) {  // concurrently with the encode, like the MD5; the host waits for it once every chunk is queued
		FB_CUDA(cudaEventRecord(e->ev_rg_fork, st));
		FB_CUDA(cudaStreamWaitEvent(e->s_rg, e->ev_rg_fork, 0));
		launch_replaygain(e->d_pcm, reinterpret_cast<const RgFileDev *>(d + o_rgf), (int)nfiles, reinterpret_cast<double *>(d + o_rgv),
		                  reinterpret_cast<uint32_t *>(d + o_rgpk), e->s_rg);
		e->launches++;
	}
	if((rc = fork_stage_a(e, nv, st)) != FB200_OK) return rc;
	e->files_frame_no = reinterpret_cast<const uint32_t *>(d + o_fno);
	for(size_t i = 0; i < chunks.size(); i++)
		if((rc = enqueue_chunk(e, i, chunks[i], e->d_pcm, 0, e->d_out, vcap, d_voff, st)) != FB200_OK) return rc;
	if(rg) {
		// The tags, and with them each header's length, are known once the analysis is: its results come back while the encode
		// runs, and the final headers replace the planned ones before the gather lays the files out.
		std::vector<double> v(rg_nwin);
		std::vector<uint32_t> peak(nfiles), album(nfiles, 0);
		FB_CUDA(cudaMemcpyAsync(peak.data(), d + o_rgpk, peak.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->s_rg));
		if(rg_nwin) FB_CUDA(cudaMemcpyAsync(v.data(), d + o_rgv, v.size() * sizeof(double), cudaMemcpyDeviceToHost, e->s_rg));
		FB_CUDA(cudaStreamSynchronize(e->s_rg));
		std::vector<fb200_replaygain_info> info(nfiles);
		replaygain_results(rgf, album.data(), v.data(), peak.data(), info.data());
		std::vector<uint8_t> meta;
		std::vector<uint64_t> moffs;
		if((rc = rg->rebuild(rg->ctx, info.data(), &meta, &moffs)) != FB200_OK) return rc;
		const size_t npts = plan.pts.size(), nblob = plan.blob.size();
		plan.heads.clear();
		plan.pts.clear();
		plan.blob.clear();
		if((rc = plan_flac_headers(meta.data(), moffs.data(), nfiles, &plan)) != FB200_OK) return rc;
		if(plan.pts.size() != npts || plan.blob.size() > nblob + rg_slack) { set_error("internal: ReplayGain tags outgrew their header room"); return FB200_ERR_CUDA; }
		memcpy(blob.data() + o_heads, plan.heads.data(), plan.heads.size() * sizeof(FlacHead));
		memcpy(blob.data() + o_hblob, plan.blob.data(), plan.blob.size());
		FB_CUDA(cudaMemcpyAsync(d + o_heads, blob.data() + o_heads, o_rgf - o_heads, cudaMemcpyHostToDevice, st));
	}
	// the files the output keeps: all of them but those check() dropped
	uint32_t nk = 0;
	for(uint32_t f = 0; f < nfiles; f++) nk += keep[f] ? 1 : 0;
	const FileFrames *d_kff = reinterpret_cast<const FileFrames *>(d + o_ff);
	const uint2 *d_korder = reinterpret_cast<const uint2 *>(d + o_order);
	const FileSeg *d_ksegs = d_segs;
	const uint8_t *d_kmd5 = d + o_md5;
	uint64_t nvk = nv;
	std::vector<uint32_t> kept;  // output file -> file of the call
	for(uint32_t f = 0; f < nfiles; f++)
		if(keep[f]) kept.push_back(f);
	std::vector<FlacHead> kheads;
	if(nk < nfiles) {
		std::vector<FileFrames> kff;
		std::vector<uint2> korder;
		std::vector<FileSeg> ksegs;
		std::vector<uint8_t> kmd5(16 * (size_t)nfiles);
		std::vector<uint8_t> md5(16 * (size_t)nfiles);
		FB_CUDA(cudaMemcpyAsync(md5.data(), d + o_md5, md5.size(), cudaMemcpyDeviceToHost, st));
		FB_CUDA(cudaStreamSynchronize(st));
		for(uint32_t k = 0; k < nk; k++) {
			const uint32_t f = kept[k];
			kff.push_back(ff[f]);
			ksegs.push_back(segs[2 * f]);
			ksegs.push_back(segs[2 * f + 1]);
			if(flac) kheads.push_back(plan.heads[f]);
			memcpy(kmd5.data() + 16 * (size_t)k, md5.data() + 16 * (size_t)f, 16);
			for(uint32_t j = 0; j < ff[f].nfull; j++) korder.push_back(make_uint2(ff[f].first + j, k));
			if(ff[f].tail != ~0u) korder.push_back(make_uint2(ff[f].tail, k));
		}
		nvk = korder.size();
		if(nk) {
			FB_CUDA(cudaMemcpyAsync(d + o_kff, kff.data(), kff.size() * sizeof(FileFrames), cudaMemcpyHostToDevice, st));
			FB_CUDA(cudaMemcpyAsync(d + o_korder, korder.data(), korder.size() * sizeof(uint2), cudaMemcpyHostToDevice, st));
			FB_CUDA(cudaMemcpyAsync(d + o_ksegs, ksegs.data(), ksegs.size() * sizeof(FileSeg), cudaMemcpyHostToDevice, st));
			FB_CUDA(cudaMemcpyAsync(d + o_kmd5, kmd5.data(), 16 * (size_t)nk, cudaMemcpyHostToDevice, st));
			if(flac) FB_CUDA(cudaMemcpyAsync(d + o_kheads, kheads.data(), kheads.size() * sizeof(FlacHead), cudaMemcpyHostToDevice, st));
			FB_CUDA(cudaStreamSynchronize(st));  // the host tables go out of scope
		}
		d_kff = reinterpret_cast<const FileFrames *>(d + o_kff);
		d_korder = reinterpret_cast<const uint2 *>(d + o_korder);
		d_ksegs = reinterpret_cast<const FileSeg *>(d + o_ksegs);
		d_kmd5 = d + o_kmd5;
	}
	else if(flac) kheads = plan.heads;
	uint8_t *fout = device ? out : e->d_fout;
	const unsigned long long fcap = device ? out_capacity : vcap;
	unsigned long long *foff = device && frame_offsets ? reinterpret_cast<unsigned long long *>(frame_offsets) : reinterpret_cast<unsigned long long *>(d + o_foff);
	const FlacHead *d_heads = flac ? reinterpret_cast<const FlacHead *>(d + (nk < nfiles ? o_kheads : o_heads)) : nullptr;
	unsigned long long *d_fbase = reinterpret_cast<unsigned long long *>(d + o_fbase);
	if(nk) {
		launch_files_gather(e->d_out, vcap, d_voff, d_kff, (int)nk, d_korder, nvk, d_heads, d + o_hblob, d_fbase, fout, fcap, foff, e->d_err, st);
		e->launches += 2;
	}
	if(verify) {
		// every chunk's frames decoded from the encode-order scratch and compared with the chunk's input, after everything that
		// reads the input on this stream (the MD5 runs on its own, and no flip is queued when it does)
		for(size_t i = 0; i < perturb.size(); i++) {
			if(perturb[i].what == 0) launch_files_perturb(e->d_out, d_voff, vcap, flip_at[i], perturb[i].b, nullptr, 0, perturb[i].mask, st);
			else launch_files_perturb(nullptr, nullptr, 0, 0, 0, e->d_pcm, flip_at[i], perturb[i].mask, st);
			e->launches++;
		}
		unsigned long long *d_vb = reinterpret_cast<unsigned long long *>(d + o_vb);
		DecVerdict *d_verd = reinterpret_cast<DecVerdict *>(d + o_verd);
		launch_verify_bounds(d_voff, nv, vcap, d_vb, st);
		auto verify_frames = [&](uint64_t v0, uint64_t n, int32_t *pcm) {
			launch_verify_chunk((int)ch, (int)e->cfg.bits_per_sample, (int)e->cfg.sample_rate, (int)bs, e->d_out, d_vb + v0, (int)n,
			                    d + o_vmeta + (size_t)v0 * verify_meta_bytes(), d_verd + v0, pcm, e->d_vcrc_tab, st);
			e->launches += 4;
		};
		// every full block of the call in one launch set, not one per encode chunk: the decode kernels need the whole batch of
		// frames to fill the device (a chunk of 4096 stereo frames is 64 CTAs)
		if(nfull_all) verify_frames(0, nfull_all, e->d_pcm);
		if(ntails) {
			// a tail's header blocksize is checked against its own length by k_verify_files
			int32_t *d_vtail = reinterpret_cast<int32_t *>(d + o_vtail);
			launch_files_tail_slots(e->d_pcm, d_segs, reinterpret_cast<const FileFrames *>(d + o_ff), (int)nfiles, (uint32_t)nfull_all, bs * ch, d_vtail, st);
			e->launches++;
			verify_frames(nfull_all, ntails, d_vtail);
		}
		launch_verify_files(d + o_vmeta, d_verd, reinterpret_cast<const FileFrames *>(d + o_ff), d_segs, (int)nfiles, (uint32_t)ch, (uint32_t)bs,
		                    e->cfg.sample_rate, reinterpret_cast<fb200_file_verify_info *>(d + o_vinfo), st);
		e->launches += 2;
	}
	if(do_md5 && !fill) FB_CUDA(cudaStreamWaitEvent(st, e->ev_md5_done, 0));
	if(nk) {
		launch_flac_file_headers(d_voff, d_kff, d_ksegs, (int)nk, (uint32_t)bs, (uint32_t)ch, e->cfg.bits_per_sample, e->cfg.sample_rate,
		                         do_md5 ? d_kmd5 : nullptr, d + o_si, d_heads, reinterpret_cast<const SeekPt *>(d + o_pts), d_fbase, fout, fcap, st);
		e->launches++;
	}
	FB_CUDA(cudaGetLastError());

	// ---- results
	std::vector<uint64_t> offs_copy(device || !frame_offsets ? nvk + 1 : 0);
	uint64_t *offs = offs_copy.empty() ? frame_offsets : offs_copy.data();
	std::vector<uint8_t> si(34 * (size_t)nfiles);
	std::vector<fb200_file_verify_info> vinfo(verify ? nfiles : 0);
	int err = 0, uerr = 0;
	unsigned long long bad = ~0ull;
	if(pcm_src) FB_CUDA(cudaMemcpyAsync(&bad, d_bad, sizeof bad, cudaMemcpyDeviceToHost, st));
	if(nk) FB_CUDA(cudaMemcpyAsync(offs, foff, (nvk + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
	else offs[0] = 0;
	FB_CUDA(cudaMemcpyAsync(si.data(), d + o_si, 34 * (size_t)nk, cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaMemcpyAsync(&uerr, d_uerr, sizeof uerr, cudaMemcpyDeviceToHost, st));
	if(verify) FB_CUDA(cudaMemcpyAsync(vinfo.data(), d + o_vinfo, vinfo.size() * sizeof(fb200_file_verify_info), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaMemcpyAsync(&err, e->d_err, sizeof err, cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	if(uerr) { set_error("a sample does not fit bits_per_sample"); return FB200_ERR_INVALID; }
	if(bad != ~0ull) {
		uint32_t f = 0;
		while(f + 1 < nfiles && pcm_src->files[f + 1].elem0 <= bad) f++;
		const unsigned long long v = bad - pcm_src->files[f].elem0;
		set_error("file %u, sample %llu, channel %llu: non-zero bits below the %u-bit sample (shift %u; format_input rejects it)", f, v / ch, v % ch,
		          e->cfg.bits_per_sample, pcm_src->files[f].shift);
		return FB200_ERR_INVALID;
	}
	if(err == 2) { set_error("internal: frame exceeded its size bound"); return FB200_ERR_CUDA; }
	if(err) { set_error("output buffer too small"); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if(!device && nk) FB_CUDA(cudaMemcpy(out, e->d_fout, (size_t)offs[nvk], cudaMemcpyDeviceToHost));
	*nframes = nvk;
	uint64_t of = 0;
	if(flac)
		for(uint32_t f = 0; f < nfiles; f++) memset(&flac_files[f], 0, sizeof flac_files[f]);
	for(uint32_t k = 0; k < nk; k++) {
		const uint32_t f = kept[k];
		const uint32_t n = ff[f].nfull + (ff[f].tail != ~0u ? 1 : 0);
		if(flac) {
			fb200_flac_file_info &I = flac_files[f];
			I.audio_offset = kheads[k].bytes;
			I.offset = offs[of] - I.audio_offset;
			I.bytes = (k + 1 < nk ? offs[of + n] - kheads[k + 1].bytes : offs[nvk]) - I.offset;
			I.first_frame = of;
			I.nframes = n;
			I.seek_points = kheads[k].npts;
			memcpy(I.streaminfo, si.data() + 34 * (size_t)k, 34);
		}
		else {
			files[f].first_frame = of;
			files[f].nframes = n;
			memcpy(files[f].streaminfo, si.data() + 34 * (size_t)k, 34);
		}
		of += n;
	}
	if(verify) {
		e->verify_info.swap(vinfo);
		e->verify_valid = true;
		uint32_t nbad = 0, first_bad = 0;
		for(uint32_t f = nfiles; f-- > 0;)
			if(e->verify_info[f].status != FB200_VERIFY_OK) { nbad++; first_bad = f; }
		if(nbad) {
			const fb200_file_verify_info &r = e->verify_info[first_bad];
			set_error("%u file(s) failed verification; the first, file %u: %s in frame %u", nbad, first_bad,
			          r.status == FB200_VERIFY_MISMATCH ? "sample mismatch" : "decoder error", r.frame_number);
			return FB200_ERR_VERIFY;
		}
	}
	return FB200_OK;
}

int fb200_encode_files_host(fb200_encoder *e, const void *pcm_interleaved, uint32_t bytes_per_sample, const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                            uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes, fb200_file_info *files)
{
	return encode_files_impl(e, pcm_interleaved, bytes_per_sample, false, file_samples, nfiles, do_md5, nullptr, nullptr, out, out_capacity, frame_offsets,
	                         nframes, files, nullptr, e ? e->stream : nullptr);
}

int fb200_encode_files_device(fb200_encoder *e, const int32_t *d_pcm_interleaved, const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                              uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes, fb200_file_info *files, void *cuda_stream)
{
	return encode_files_impl(e, d_pcm_interleaved, 4, true, file_samples, nfiles, do_md5, nullptr, nullptr, d_out, out_capacity, d_frame_offsets, nframes,
	                         files, nullptr, (cudaStream_t)cuda_stream);
}

int fb200_encode_flac_files_host(fb200_encoder *e, const void *pcm_interleaved, uint32_t bytes_per_sample, const uint64_t *file_samples, uint32_t nfiles,
                                 int do_md5, const uint8_t *metadata, const uint64_t *metadata_offsets, uint8_t *out, size_t out_capacity,
                                 uint64_t *frame_offsets, uint64_t *nframes, fb200_flac_file_info *files)
{
	if(!files) { set_error("files is NULL"); return FB200_ERR_INVALID; }
	return encode_files_impl(e, pcm_interleaved, bytes_per_sample, false, file_samples, nfiles, do_md5, metadata, metadata_offsets, out, out_capacity,
	                         frame_offsets, nframes, nullptr, files, e ? e->stream : nullptr);
}

int fb200_encode_flac_files_device(fb200_encoder *e, const int32_t *d_pcm_interleaved, const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                                   const uint8_t *metadata, const uint64_t *metadata_offsets, uint8_t *d_out, size_t out_capacity,
                                   uint64_t *d_frame_offsets, uint64_t *nframes, fb200_flac_file_info *files, void *cuda_stream)
{
	if(!files) { set_error("files is NULL"); return FB200_ERR_INVALID; }
	return encode_files_impl(e, d_pcm_interleaved, 4, true, file_samples, nfiles, do_md5, metadata, metadata_offsets, d_out, out_capacity, d_frame_offsets,
	                         nframes, nullptr, files, (cudaStream_t)cuda_stream);
}

int fb200_encoder_set_verify(fb200_encoder *e, int on)
{
	if(!e) return FB200_ERR_INVALID;
	if(on && !e->d_vcrc_tab) {
		FB_CUDA(cudaSetDevice(e->device));
		FB_CUDA(cudaMalloc(&e->d_vcrc_tab, kVerifyCrcTabBytes));
		launch_verify_crc_tables(e->d_vcrc_tab, e->stream);
		FB_CUDA(cudaStreamSynchronize(e->stream));
	}
	e->verify = on != 0;
	return FB200_OK;
}

int fb200_encoder_get_verify(const fb200_encoder *e, fb200_file_verify_info *info, uint32_t nfiles)
{
	if(!e || !info) return FB200_ERR_INVALID;
	if(!e->verify_valid) { set_error("the last encode_files call did not verify"); return FB200_ERR_INVALID; }
	if(nfiles != e->verify_info.size()) { set_error("the last encode_files call had %zu files, not %u", e->verify_info.size(), nfiles); return FB200_ERR_INVALID; }
	memcpy(info, e->verify_info.data(), (size_t)nfiles * sizeof *info);
	return FB200_OK;
}

int fb200_debug_perturb_verify(fb200_encoder *e, uint32_t file, uint32_t what, uint32_t a, uint32_t b, uint32_t xor_mask)
{
	if(!e || what > 1) return FB200_ERR_INVALID;
	e->perturb.push_back(fb200_encoder::Perturb{file, what, a, b, xor_mask});
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

// k_lpc on caller-supplied autocorrelations (tests/test_gpu_lpc_edges.py), launched by launch_lpc as the encoder launches it
int fb200_debug_lpc(int device, const double *autoc, uint32_t nsec, uint32_t lag_stride, const int32_t *meta, const int32_t *cands,
                    uint32_t nwin, uint32_t nitems, uint32_t max_order, uint32_t qlp_precision, int prec_search, int exhaustive,
                    uint32_t blocksize, int autoc_unshifted, void *out, size_t cand_bytes, uint32_t *nslots_out)
{
	if(!autoc || !meta || !cands || !out || !nslots_out) return FB200_ERR_INVALID;
	if(cand_bytes != sizeof(CandDesc)) { set_error("candidate size mismatch %zu != %zu", cand_bytes, sizeof(CandDesc)); return FB200_ERR_INVALID; }
	if(max_order < 1 || max_order > FB200_MAX_LPC_ORDER || max_order >= blocksize || blocksize > 65535 || lag_stride < max_order + 1 ||
	   nsec == 0 || nwin == 0 || nitems == 0 || (!prec_search && (qlp_precision < kMinQlpPrecision || qlp_precision > kMaxQlpPrecision))) {
		set_error("fb200_debug_lpc: arguments out of range");
		return FB200_ERR_INVALID;
	}
	for(uint32_t i = 0; i < nitems; i++)
		if(meta[2 * i] < 0 || meta[2 * i] > 31 || meta[2 * i + 1] < 0 || meta[2 * i + 1] > 32) { set_error("fb200_debug_lpc: meta %u", i); return FB200_ERR_INVALID; }
	for(uint32_t w = 0; w < nwin; w++) {
		const int32_t *c = cands + 3 * w;
		if(c[0] < 0 || c[0] > 1 || c[1] < 0 || (uint32_t)c[1] >= nsec || c[2] < 0 || (uint32_t)c[2] >= nsec) { set_error("fb200_debug_lpc: candidate %u", w); return FB200_ERR_INVALID; }
	}
	EncK k;
	memset(&k, 0, sizeof k);
	k.bs = (int)blocksize;
	k.max_order = (int)max_order;
	k.lags = k.max_order + 1;
	k.lag_stride = (int)lag_stride;
	k.qlp_precision = (int)qlp_precision;
	k.prec_search = prec_search ? 1 : 0;
	k.exhaustive = exhaustive ? 1 : 0;
	k.nsec = (int)nsec;
	k.nwin = (int)nwin;
	k.nslots = k.nwin * (k.exhaustive ? k.max_order : 1) * (k.prec_search ? kQlpPrecisionSteps : 1);  // as the encoder sizes them
	*nslots_out = (uint32_t)k.nslots;
	const size_t nac = (size_t)nsec * nitems * lag_stride, nout = (size_t)nitems * k.nslots;
	std::vector<DevCand> hc(nwin);
	for(uint32_t w = 0; w < nwin; w++) hc[w] = DevCand{cands[3 * w], cands[3 * w + 1], cands[3 * w + 2]};
	std::vector<SigMeta> hm(nitems);
	for(uint32_t i = 0; i < nitems; i++) hm[i] = SigMeta{meta[2 * i], meta[2 * i + 1]};
	FB_CUDA(cudaSetDevice(device));
	double *d_ac = nullptr;
	DevCand *d_c = nullptr;
	SigMeta *d_m = nullptr;
	CandDesc *d_o = nullptr;
	int rc = FB200_OK;
	if(cudaMalloc(&d_ac, nac * sizeof(double)) != cudaSuccess || cudaMalloc(&d_c, nwin * sizeof(DevCand)) != cudaSuccess ||
	   cudaMalloc(&d_m, nitems * sizeof(SigMeta)) != cudaSuccess || cudaMalloc(&d_o, nout * sizeof(CandDesc)) != cudaSuccess ||
	   cudaMemcpy(d_ac, autoc, nac * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
	   cudaMemcpy(d_c, hc.data(), nwin * sizeof(DevCand), cudaMemcpyHostToDevice) != cudaSuccess ||
	   cudaMemcpy(d_m, hm.data(), nitems * sizeof(SigMeta), cudaMemcpyHostToDevice) != cudaSuccess ||
	   cudaMemset(d_o, 0xff, nout * sizeof(CandDesc)) != cudaSuccess) {
		set_error("fb200_debug_lpc: %s", cudaGetErrorString(cudaGetLastError()));
		rc = FB200_ERR_CUDA;
	}
	if(rc == FB200_OK) {
		launch_lpc(k, d_ac, d_c, d_m, nullptr, d_o, (int)nitems, autoc_unshifted ? 1 : 0, 0);
		cudaError_t err = cudaGetLastError();
		if(err == cudaSuccess) err = cudaMemcpy(out, d_o, nout * sizeof(CandDesc), cudaMemcpyDeviceToHost);
		if(err != cudaSuccess) { set_error("fb200_debug_lpc: %s", cudaGetErrorString(err)); rc = FB200_ERR_CUDA; }
	}
	cudaFree(d_ac); cudaFree(d_c); cudaFree(d_m); cudaFree(d_o);
	return rc;
}

// the general search kernel's evaluation of given LPC candidates on given signals (tests/test_gpu_lpc_edges.py)
int fb200_debug_evaluate_lpc(int device, const int32_t *signals, const int32_t *meta, const void *cands, size_t cand_bytes, uint32_t n,
                             uint32_t blocksize, uint32_t min_po, uint32_t max_po, uint32_t rice_limit, uint32_t *est)
{
	if(!signals || !meta || !cands || !est || n == 0) return FB200_ERR_INVALID;
	if(cand_bytes != sizeof(CandDesc)) { set_error("candidate size mismatch %zu != %zu", cand_bytes, sizeof(CandDesc)); return FB200_ERR_INVALID; }
	if(blocksize < 16 || blocksize > 65535 || max_po > (uint32_t)kMaxPartitionOrder || min_po > max_po || (rice_limit != 15 && rice_limit != 31)) {
		set_error("fb200_debug_evaluate_lpc: arguments out of range");
		return FB200_ERR_INVALID;
	}
	const CandDesc *hc = static_cast<const CandDesc *>(cands);
	std::vector<SigMeta> hm(n);
	for(uint32_t i = 0; i < n; i++) {
		hm[i] = SigMeta{meta[2 * i], meta[2 * i + 1]};
		if(hm[i].wasted < 0 || hm[i].wasted > 31 || hm[i].bps < 1 || hm[i].bps > 32 || hc[i].order < 1 || hc[i].order > FB200_MAX_LPC_ORDER ||
		   (uint32_t)hc[i].order >= blocksize || hc[i].shift < 0 || hc[i].shift > 15) {
			set_error("fb200_debug_evaluate_lpc: candidate %u", i);
			return FB200_ERR_INVALID;
		}
	}
	EncK k;
	memset(&k, 0, sizeof k);
	k.bs = k.bs_stride = (int)blocksize;
	k.min_po = (int)min_po;
	k.max_po = (int)max_po;
	k.rice_limit = (int)rice_limit;
	FB_CUDA(cudaSetDevice(device));
	const size_t ns = (size_t)n * blocksize;
	int32_t *d_sig = nullptr;
	SigMeta *d_m = nullptr;
	CandDesc *d_c = nullptr;
	uint32_t *d_absr = nullptr, *d_est = nullptr;
	int rc = FB200_OK;
	if(cudaMalloc(&d_sig, ns * sizeof(int32_t)) != cudaSuccess || cudaMalloc(&d_m, n * sizeof(SigMeta)) != cudaSuccess ||
	   cudaMalloc(&d_c, n * sizeof(CandDesc)) != cudaSuccess || cudaMalloc(&d_absr, ns * sizeof(uint32_t)) != cudaSuccess ||
	   cudaMalloc(&d_est, n * sizeof(uint32_t)) != cudaSuccess ||
	   cudaMemcpy(d_sig, signals, ns * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess ||
	   cudaMemcpy(d_m, hm.data(), n * sizeof(SigMeta), cudaMemcpyHostToDevice) != cudaSuccess ||
	   cudaMemcpy(d_c, hc, n * sizeof(CandDesc), cudaMemcpyHostToDevice) != cudaSuccess) {
		set_error("fb200_debug_evaluate_lpc: %s", cudaGetErrorString(cudaGetLastError()));
		rc = FB200_ERR_CUDA;
	}
	if(rc == FB200_OK) {
		launch_debug_evaluate(k, d_sig, d_m, d_c, d_absr, d_est, (int)n);
		cudaError_t err = cudaGetLastError();
		if(err == cudaSuccess) err = cudaMemcpy(est, d_est, n * sizeof(uint32_t), cudaMemcpyDeviceToHost);
		if(err != cudaSuccess) { set_error("fb200_debug_evaluate_lpc: %s", cudaGetErrorString(err)); rc = FB200_ERR_CUDA; }
	}
	cudaFree(d_sig); cudaFree(d_m); cudaFree(d_c); cudaFree(d_absr); cudaFree(d_est);
	return rc;
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

// stage A of the last call's full blocks (tests/test_gpu_autoc.py): reads the workspace slices the call's chunks left behind
int fb200_debug_copy_autoc(fb200_encoder *e, uint32_t nblocks, double *autoc, size_t autoc_doubles, int32_t *meta, uint32_t *sigor,
                           int32_t *sections, uint32_t max_sections, fb200_debug_autoc_info *info)
{
	if(!e || !info) return FB200_ERR_INVALID;
	const auto it = e->geoms.find((int)e->cfg.blocksize);
	if(nblocks == 0 || !e->slice_mode || it == e->geoms.end() || it->second.k.nwin == 0) {
		set_error("fb200_debug_copy_autoc: the last call did not fit one workspace set, or its configuration computes no autocorrelation");
		return FB200_ERR_INVALID;
	}
	const Geometry &g = it->second;
	const size_t nsig = (size_t)e->nsig, nitems = (size_t)nblocks * nsig, ls = e->lag_stride, nsec = (size_t)g.k.nsec;
	uint64_t covered = 0;
	int route = -1;
	for(const auto &c : e->chunks_a) {
		if(covered >= nblocks) break;
		if(c.first != covered || (route >= 0 && c.route != route)) {
			set_error("fb200_debug_copy_autoc: the last call's full blocks are not consecutive chunks of one route");
			return FB200_ERR_INVALID;
		}
		route = c.route;
		covered += c.nb;
	}
	if(covered < nblocks) { set_error("fb200_debug_copy_autoc: the last call encoded %llu full blocks, not %u", (unsigned long long)covered, nblocks); return FB200_ERR_INVALID; }
	info->nsec = (uint32_t)nsec; info->lags = (uint32_t)g.k.lags; info->kernel_lags = (uint32_t)autoc_kernel_lags(g.k.lags);
	info->lag_stride = (uint32_t)ls; info->route = route;
	if(!autoc) return FB200_OK;  // sizes only
	if(!meta || !sigor || !sections || autoc_doubles < nsec * nitems * ls || max_sections < nsec) return FB200_ERR_INVALID;
	static_assert(sizeof(SigMeta) == 2 * sizeof(int32_t) && sizeof(DevSection) == 5 * sizeof(int32_t), "the C ABI's layouts");
	FB_CUDA(cudaSetDevice(e->device));
	FB_CUDA(cudaDeviceSynchronize());
	const size_t slice = e->max_nsec ? e->max_nsec : 1;
	for(const auto &c : e->chunks_a) {
		if(c.first >= nblocks) break;
		const size_t n = (size_t)(c.nb < nblocks - c.first ? c.nb : nblocks - c.first) * nsig, cn = (size_t)c.nb * nsig, o = (size_t)c.first * nsig;
		// use_ws: the chunk's records start at its first item's slice, section-major over the chunk's own items
		const double *src = e->ws[0].d_autoc + o * slice * ls;
		for(size_t sec = 0; sec < nsec; sec++)
			FB_CUDA(cudaMemcpy(autoc + (sec * nitems + o) * ls, src + sec * cn * ls, n * ls * sizeof(double), cudaMemcpyDeviceToHost));
		FB_CUDA(cudaMemcpy(meta + 2 * o, e->ws[0].d_meta + o, n * sizeof(SigMeta), cudaMemcpyDeviceToHost));
		if(route == (int)StageA::fused) FB_CUDA(cudaMemcpy(sigor + o, e->ws[0].d_sigor + o, n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
	}
	FB_CUDA(cudaMemcpy(sections, g.d_secs, nsec * sizeof(DevSection), cudaMemcpyDeviceToHost));
	return FB200_OK;
}

}  // extern "C"

namespace fb200 {

void encoder_spread_verify(fb200_encoder *e, const std::vector<uint32_t> &at, uint32_t nlisted)
{
	if(!e->verify_valid) return;
	std::vector<fb200_file_verify_info> all(nlisted);
	memset(all.data(), 0, all.size() * sizeof(fb200_file_verify_info));
	for(size_t i = 0; i < at.size() && i < e->verify_info.size(); i++) all[at[i]] = e->verify_info[i];
	e->verify_info.swap(all);
}

int encoder_device(const fb200_encoder *e) { return e->device; }

// encode_files_impl is this file's; fb200_encode_pcm_files_* (pcm_container.cu) and fb200_reencode_flac_files_* (reencode.cu)
// reach it through here
int encode_pcm_files_impl(fb200_encoder *e, const PcmSource &src, bool device, const uint64_t *file_samples, uint32_t nfiles, int do_md5,
                          const uint8_t *metadata, const uint64_t *metadata_offsets, uint8_t *out, size_t out_capacity, uint64_t *frame_offsets,
                          uint64_t *nframes, fb200_flac_file_info *files, void *cuda_stream)
{
	return encode_files_impl(e, src.data, 4, device, file_samples, nfiles, do_md5, metadata, metadata_offsets, out, out_capacity, frame_offsets, nframes,
	                         nullptr, files, device ? (cudaStream_t)cuda_stream : e->stream, &src);
}

}  // namespace fb200

namespace fb200 {

int encoder_create(const fb200_encoder_config *cfg, int device, uint32_t max_blocks, bool bound_tiled, fb200_encoder **out)
{
	return create_impl(cfg, device, max_blocks, bound_tiled, out);
}

uint32_t encoder_capacity(const fb200_encoder *e) { return e ? e->max_blocks : 0; }

void put_streaminfo(uint8_t body[34], uint32_t min_blocksize, uint32_t max_blocksize, uint32_t min_framesize, uint32_t max_framesize,
                    uint32_t sample_rate, uint32_t channels, uint32_t bits_per_sample, uint64_t total_samples, const uint8_t md5[16])
{
	auto be = [&](int at, uint64_t v, int n) { for(int i = 0; i < n; i++) body[at + i] = (uint8_t)(v >> (8 * (n - 1 - i))); };
	be(0, min_blocksize, 2); be(2, max_blocksize, 2); be(4, min_framesize, 3); be(7, max_framesize, 3);
	be(10, ((uint64_t)sample_rate << 44) | ((uint64_t)(channels - 1) << 41) | ((uint64_t)(bits_per_sample - 1) << 36) | (total_samples & 0xFFFFFFFFFull), 8);
	memcpy(body + 18, md5, 16);
}

}  // namespace fb200
