// decoder.cu -- host side of the FLAC batch frame decoder + its C ABI (include/flac_b200.h).
#include <string.h>

#include <algorithm>
#include <array>
#include <map>
#include <utility>
#include <vector>

#include "decode_kernels.cuh"
#include "flac_parse.h"

using namespace fb200;

struct fb200_decoder {
	fb200_decoder_config cfg;
	int device = 0;
	uint32_t max_frames = 0;
	DecK k{};
	DecFrameMeta *d_meta = nullptr;
	uint16_t *d_crc_tab = nullptr;     // slicing tables + combine multipliers of k_dec_crc
	DecSubframeInfo *d_subinfo = nullptr;  // per (frame, channel), only when the client asked for subframe details
	size_t d_subinfo_cap = 0;
	bool want_subinfo = false;
	// staging for the host entry point
	uint8_t *d_frames = nullptr;
	size_t d_frames_cap = 0;
	unsigned long long *d_offsets = nullptr;
	size_t d_offsets_cap = 0;
	int32_t *d_pcm = nullptr;
	size_t d_pcm_cap = 0;
	uint32_t *d_status = nullptr;
	size_t d_status_cap = 0;
	cudaStream_t stream = nullptr, s_h2d = nullptr, s_d2h = nullptr;
	std::vector<cudaEvent_t> ev_in, ev_done;  // per chunk of the host path: frames arrived / decoded
	uint8_t *d_packed = nullptr;      // narrowed output of fb200_decode_host_packed
	size_t d_packed_cap = 0;
	std::vector<uint32_t> h_status;   // per-frame status words of the last host decode
	uint8_t *d_stream = nullptr;      // staging of fb200_decoder_index_host / fb200_decode_stream_host
	size_t d_stream_cap = 0;
	unsigned long long *d_cand = nullptr;
	size_t d_cand_cap = 0;
	unsigned *d_count = nullptr;
	uint32_t *d_fbytes = nullptr;
	size_t d_fbytes_cap = 0;
	uint64_t launches = 0;
	bool prof_on = false;
	std::vector<cudaEvent_t> prof_events;
	std::vector<int> prof_ids;
	double prof_ms[FB200_DPROF_KERNELS] = {0};
	uint64_t prof_launches[FB200_DPROF_KERNELS] = {0};
	// fb200_decode_files_*: the resident batch (d_fdata) and its index. Files of one (channels, bits per sample) group are
	// decoded by one launch set; the index arrays hold the candidates group by group, file by file, ascending.
	struct FilesGroup {
		uint32_t channels, bps, max_bs;
		uint64_t cand0, ncand;   // candidates [cand0, cand0 + ncand)
		uint32_t pos0, nfiles;   // files [pos0, pos0 + nfiles) of files_order / files_state0
	};
	bool files_ready = false;
	uint64_t files_values = 0, files_ncand = 0;
	std::vector<fb200_file_decode_info> files_info;  // what the index call reported
	std::vector<std::array<uint8_t, 16>> files_md5;  // STREAMINFO MD5 per file
	std::vector<FilesGroup> files_groups;
	std::vector<uint32_t> files_order;               // group order -> file
	std::vector<FileDecState> files_state0;          // group order: the state a decode call starts from
	uint8_t *d_fdata = nullptr;                      // the batch (+ 64 bytes of slack)
	size_t d_fdata_cap = 0;
	uint8_t *d_findex = nullptr;                     // begins, ends, candidates, file states
	size_t d_findex_cap = 0;
	uint8_t *d_fwork = nullptr;                      // per chunk: status, frame bytes, places; MD5 segments and digests
	size_t d_fwork_cap = 0;
	int32_t *d_fslots = nullptr;                     // decoded candidates, one slot of max_blocksize x channels each
	size_t d_fslots_cap = 0;
	uint8_t *d_rwork = nullptr;                      // fb200_decode_files_ranges_*: per range selection, count, offset, state
	size_t d_rwork_cap = 0;
	uint8_t *d_rcand = nullptr;                      // ... and the selected candidates: begins, ends, FileDecCand
	size_t d_rcand_cap = 0;
	std::vector<uint32_t> files_mask;                // fb200_decode_pcm_files_*: each file's WAVEFORMATEXTENSIBLE_CHANNEL_MASK tag (0: none)
	std::vector<uint64_t> files_start, files_audio;  // fb200_reencode_flac_files_*: each file's first byte and first frame byte in the batch
	std::vector<uint64_t> files_end;                 // fb200_add_replaygain_flac_files_*: each file's end in the batch
	std::vector<uint32_t> files_pos;                 // ... and its place in files_order (~0u: not OK)
	uint8_t *d_pwork = nullptr;                      // ... and k_pcm_pack's plan: segments, their containers, containers, headers
	size_t d_pwork_cap = 0;
	uint8_t *d_keep = nullptr;                       // fb200_decode_pcm_files_replaygain_*: every candidate's frame bytes and place
	size_t d_keep_cap = 0;
	uint8_t *d_rgswork = nullptr;                    // ... and k_rg_synth's plan
	size_t d_rgswork_cap = 0;
};

// device buffer of at least `need` bytes (contents not kept)
static int grow(void **p, size_t *cap, size_t need)
{
	if(need <= *cap) return FB200_OK;
	cudaFree(*p); *p = nullptr; *cap = 0;
	if(cudaMalloc(p, need) != cudaSuccess) {
		cudaGetLastError();
		set_error("device allocation of %zu bytes failed", need);
		return FB200_ERR_ALLOC;
	}
	*cap = need;
	return FB200_OK;
}

static size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

static void dprof_mark(fb200_decoder *d, int id, cudaStream_t st)
{
	if(!d->prof_on) return;
	cudaEvent_t ev;
	if(cudaEventCreate(&ev) != cudaSuccess) return;
	cudaEventRecord(ev, st);
	d->prof_events.push_back(ev);
	d->prof_ids.push_back(id);
}

static void dprof_resolve(fb200_decoder *d)
{
	for(size_t i = 1; i < d->prof_events.size(); i++) {
		if(d->prof_ids[i] < 0) continue;
		float ms = 0.f;
		cudaEventSynchronize(d->prof_events[i]);
		if(cudaEventElapsedTime(&ms, d->prof_events[i - 1], d->prof_events[i]) == cudaSuccess) {
			d->prof_ms[d->prof_ids[i]] += ms;
			d->prof_launches[d->prof_ids[i]]++;
		}
	}
	for(cudaEvent_t ev : d->prof_events) cudaEventDestroy(ev);
	d->prof_events.clear();
	d->prof_ids.clear();
}

extern "C" {

int fb200_decoder_create(const fb200_decoder_config *cfg, int device, uint32_t max_frames, fb200_decoder **out)
{
	if(!cfg || !out) return FB200_ERR_INVALID;
	*out = nullptr;
	if(cfg->channels == 0 || cfg->channels > FB200_MAX_CHANNELS) { set_error("invalid number of channels %u", cfg->channels); return FB200_ERR_INVALID; }
	if(cfg->bits_per_sample < 4 || cfg->bits_per_sample > 32) { set_error("invalid bits per sample %u", cfg->bits_per_sample); return FB200_ERR_INVALID; }
	if(cfg->bits_per_sample > 24) { set_error("bits_per_sample %u > 24 is outside this engine's scope", cfg->bits_per_sample); return FB200_ERR_UNSUPPORTED; }
	if(cfg->blocksize < 1 || cfg->blocksize > 65535) { set_error("invalid blocksize %u", cfg->blocksize); return FB200_ERR_INVALID; }
	int ndev = 0;
	if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
		set_error("no CUDA device: the FLAC block engine has no CPU fallback");
		return FB200_ERR_CUDA;
	}
	if(device < 0 || device >= ndev) { set_error("invalid device %d", device); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(device));
	fb200_decoder *d = new fb200_decoder();
	d->cfg = *cfg;
	d->device = device;
	d->max_frames = max_frames ? max_frames : 16384;
	d->k.channels = (int)cfg->channels; d->k.bps = (int)cfg->bits_per_sample; d->k.sample_rate = (int)cfg->sample_rate;
	d->k.blocksize = (int)cfg->blocksize;
	d->k.loose_end = 0;
	if(cudaMalloc(&d->d_crc_tab, (size_t)kDecCrcTabEntries * sizeof(uint16_t)) != cudaSuccess ||
	   cudaMalloc(&d->d_meta, (size_t)d->max_frames * sizeof(DecFrameMeta)) != cudaSuccess ||
	   cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess) {
		set_error("decoder workspace allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
		fb200_decoder_destroy(d);
		return FB200_ERR_ALLOC;
	}
	k_dec_crc_tables<<<(kDecCrcLw * 5 + 255) / 256, 256, 0, d->stream>>>(d->d_crc_tab);
	if(cudaStreamSynchronize(d->stream) != cudaSuccess) {
		set_error("decoder table kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
		fb200_decoder_destroy(d);
		return FB200_ERR_CUDA;
	}
	*out = d;
	return FB200_OK;
}

void fb200_decoder_destroy(fb200_decoder *d)
{
	if(!d) return;
	cudaSetDevice(d->device);
	cudaFree(d->d_subinfo); cudaFree(d->d_meta); cudaFree(d->d_crc_tab); cudaFree(d->d_stream); cudaFree(d->d_cand); cudaFree(d->d_count); cudaFree(d->d_fbytes); cudaFree(d->d_frames); cudaFree(d->d_offsets); cudaFree(d->d_pcm); cudaFree(d->d_status);
	if(d->stream) cudaStreamDestroy(d->stream);
	if(d->s_h2d) cudaStreamDestroy(d->s_h2d);
	if(d->s_d2h) cudaStreamDestroy(d->s_d2h);
	for(cudaEvent_t ev : d->ev_in) cudaEventDestroy(ev);
	for(cudaEvent_t ev : d->ev_done) cudaEventDestroy(ev);
	cudaFree(d->d_packed);
	cudaFree(d->d_fdata); cudaFree(d->d_findex); cudaFree(d->d_fwork); cudaFree(d->d_fslots); cudaFree(d->d_rwork); cudaFree(d->d_rcand); cudaFree(d->d_pwork);
	cudaFree(d->d_keep); cudaFree(d->d_rgswork);
	delete d;
}

uint64_t fb200_decoder_launch_count(const fb200_decoder *d) { return d ? d->launches : 0; }

int fb200_decoder_set_profiling(fb200_decoder *d, int on)
{
	if(!d) return FB200_ERR_INVALID;
	cudaSetDevice(d->device);
	dprof_resolve(d);
	d->prof_on = on != 0;
	return FB200_OK;
}

int fb200_decoder_get_profile(fb200_decoder *d, double ms[FB200_DPROF_KERNELS], uint64_t launches[FB200_DPROF_KERNELS], int reset)
{
	if(!d) return FB200_ERR_INVALID;
	cudaSetDevice(d->device);
	dprof_resolve(d);
	for(int i = 0; i < FB200_DPROF_KERNELS; i++) {
		if(ms) ms[i] = d->prof_ms[i];
		if(launches) launches[i] = d->prof_launches[i];
		if(reset) { d->prof_ms[i] = 0; d->prof_launches[i] = 0; }
	}
	return FB200_OK;
}

// frames f = 0..nframes-1 occupy [begins[f], ends[f]) of d_frames (device arrays); loose: the ends are upper bounds
// k: the stream's facts; k.blocksize is also the slot stride (frame i of the call decodes to sample i * k.blocksize);
// want_subinfo: collect subframe records (fb200_decoder_enable_subframe_info)
static int decode_ranges(fb200_decoder *d, DecK k, bool want_subinfo, const uint8_t *d_frames, const unsigned long long *begins, const unsigned long long *ends,
                         uint32_t nframes, int32_t *d_pcm, uint64_t pcm_capacity_samples, uint32_t *d_frame_status, uint32_t *d_frame_bytes, int loose,
                         cudaStream_t st, uint32_t subinfo_base = 0)
{
	const int ch = k.channels;
	const int chl = ch <= 1 ? 1 : ch <= 2 ? 2 : ch <= 4 ? 4 : 8;
	const int fpw = 32 / chl;
	k.loose_end = loose;
	// subframe records of frame i of this call go to slot subinfo_base + i (a chunked caller sized the array for all its frames)
	if(want_subinfo && (size_t)(subinfo_base + nframes) * ch > d->d_subinfo_cap) {
		if(subinfo_base) { set_error("internal: subframe info array too small"); return FB200_ERR_INVALID; }
		cudaFree(d->d_subinfo); d->d_subinfo = nullptr; d->d_subinfo_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_subinfo, (size_t)nframes * ch * sizeof(DecSubframeInfo)));
		d->d_subinfo_cap = (size_t)nframes * ch;
	}
	uint32_t done = 0;
	while(done < nframes) {
		const int nf = (int)((nframes - done) < d->max_frames ? (nframes - done) : d->max_frames);
		// frame `done + i` decodes to sample offset (done + i) * blocksize
		const unsigned long long used = (unsigned long long)done * k.blocksize;
		const unsigned long long cap_left = pcm_capacity_samples > used ? pcm_capacity_samples - used : 0ull;  // frames that do not fit are reported (DEC_LENGTH), never written
		dprof_mark(d, -1, st);
		k_dec_walk<<<(nf + 127) / 128, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta);
		dprof_mark(d, FB200_DPROF_WALK, st);
		const int warps = (nf + fpw - 1) / fpw;
		// predictors of at most 12 taps (every preset) and the rest (-l 13..32): two instantiations, each taking its frames
		k_dec_frames<12><<<(warps + 3) / 4, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta, d_pcm + (size_t)done * k.blocksize * ch, cap_left,
		                                                 d_frame_status ? d_frame_status + done : nullptr,
		                                                 want_subinfo ? d->d_subinfo + (size_t)(subinfo_base + done) * ch : nullptr);
		k_dec_frames<32><<<(warps + 3) / 4, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta, d_pcm + (size_t)done * k.blocksize * ch, cap_left,
		                                                 d_frame_status ? d_frame_status + done : nullptr,
		                                                 want_subinfo ? d->d_subinfo + (size_t)(subinfo_base + done) * ch : nullptr);
		dprof_mark(d, FB200_DPROF_FRAMES, st);
		k_dec_crc<<<(nf + 3) / 4, 128, 0, st>>>(d_frames, begins + done, nf, d->d_meta, d_frame_status ? d_frame_status + done : nullptr,
		                                       d_frame_bytes ? d_frame_bytes + done : nullptr, d->d_crc_tab);
		dprof_mark(d, FB200_DPROF_CRC, st);
		d->launches += 4;
		done += nf;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

int fb200_decode_device(fb200_decoder *d, const uint8_t *d_frames, const uint64_t *d_frame_offsets, uint32_t nframes,
                        int32_t *d_pcm, uint64_t pcm_capacity_samples, uint32_t *d_frame_status, void *cuda_stream, int sync)
{
	if(!d || !d_frames || !d_frame_offsets || !d_pcm) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(d->device));
	cudaStream_t st = (cudaStream_t)cuda_stream;
	const unsigned long long *offs = reinterpret_cast<const unsigned long long *>(d_frame_offsets);
	const int rc = decode_ranges(d, d->k, d->want_subinfo, d_frames, offs, offs + 1, nframes, d_pcm, pcm_capacity_samples, d_frame_status, nullptr, 0, st);
	if(rc != FB200_OK) return rc;
	if(sync) FB_CUDA(cudaStreamSynchronize(st));
	return FB200_OK;
}

// Host-buffer decode: the batch is cut into chunks of frames; chunk i+1's frame bytes cross PCIe while chunk i decodes and
// chunk i-1's samples go back (three streams; truly asynchronous with pinned buffers). bytes_per_sample 2 / 3 narrows the
// samples on the device to packed little-endian 16- / 24-bit PCM (what a WAV writer wants): the D2H copy is the end-to-end
// bound of a decoder, and int32 doubles it for 16-bit audio.
static int decode_host_impl(fb200_decoder *d, const uint8_t *frames, const uint64_t *frame_offsets, uint32_t nframes,
                            void *pcm_out, uint32_t bytes_per_sample, uint64_t pcm_capacity_samples, uint64_t *samples_decoded, uint32_t *bad_frames)
{
	if(!d || !frames || !frame_offsets || !pcm_out) return FB200_ERR_INVALID;
	if(bytes_per_sample != 2 && bytes_per_sample != 3 && bytes_per_sample != 4) { set_error("bytes_per_sample must be 2, 3 or 4"); return FB200_ERR_INVALID; }
	if(d->cfg.bits_per_sample > 8 * bytes_per_sample) { set_error("%u-bit samples do not fit %u bytes", d->cfg.bits_per_sample, bytes_per_sample); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(d->device));
	if(samples_decoded) *samples_decoded = 0;
	if(bad_frames) *bad_frames = 0;
	if(nframes == 0) return FB200_OK;
	const uint32_t ch = d->cfg.channels, bs = d->cfg.blocksize;
	const size_t nbytes = (size_t)frame_offsets[nframes];
	const uint64_t need_samples = (uint64_t)nframes * bs;
	const uint64_t cap = pcm_capacity_samples < need_samples ? pcm_capacity_samples : need_samples;
	const bool packed = bytes_per_sample != 4;
	if(nbytes + 64 > d->d_frames_cap) {
		cudaFree(d->d_frames); d->d_frames = nullptr; d->d_frames_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_frames, nbytes + 64));
		d->d_frames_cap = nbytes + 64;
	}
	if((size_t)nframes + 1 > d->d_offsets_cap) {
		cudaFree(d->d_offsets); d->d_offsets = nullptr; d->d_offsets_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_offsets, ((size_t)nframes + 1) * sizeof(unsigned long long)));
		d->d_offsets_cap = (size_t)nframes + 1;
	}
	if(need_samples * ch > d->d_pcm_cap) {
		cudaFree(d->d_pcm); d->d_pcm = nullptr; d->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_pcm, need_samples * ch * sizeof(int32_t)));
		d->d_pcm_cap = need_samples * ch;
	}
	if(packed && need_samples * ch * bytes_per_sample + 16 > d->d_packed_cap) {
		cudaFree(d->d_packed); d->d_packed = nullptr; d->d_packed_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_packed, need_samples * ch * bytes_per_sample + 16));
		d->d_packed_cap = need_samples * ch * bytes_per_sample + 16;
	}
	if(nframes > d->d_status_cap) {
		cudaFree(d->d_status); d->d_status = nullptr; d->d_status_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_status, (size_t)nframes * sizeof(uint32_t)));
		d->d_status_cap = nframes;
	}
	if(d->want_subinfo && (size_t)nframes * ch > d->d_subinfo_cap) {
		cudaFree(d->d_subinfo); d->d_subinfo = nullptr; d->d_subinfo_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_subinfo, (size_t)nframes * ch * sizeof(DecSubframeInfo)));
		d->d_subinfo_cap = (size_t)nframes * ch;
	}
	if(!d->s_h2d) FB_CUDA(cudaStreamCreateWithFlags(&d->s_h2d, cudaStreamNonBlocking));
	if(!d->s_d2h) FB_CUDA(cudaStreamCreateWithFlags(&d->s_d2h, cudaStreamNonBlocking));
	// chunks: 16 per call, at least 1024 frames, at most the launch capacity (chosen on a previous GPU, not re-measured on H100)
	uint32_t chunk = (nframes + 15) / 16;
	if(chunk < 1024) chunk = 1024;
	if(chunk > d->max_frames) chunk = d->max_frames;
	const uint32_t nchunks = (nframes + chunk - 1) / chunk;
	while(d->ev_in.size() < nchunks) {
		cudaEvent_t a, b;
		FB_CUDA(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
		FB_CUDA(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
		d->ev_in.push_back(a); d->ev_done.push_back(b);
	}
	FB_CUDA(cudaMemcpyAsync(d->d_offsets, frame_offsets, ((size_t)nframes + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, d->s_h2d));
	FB_CUDA(cudaMemsetAsync(d->d_frames + nbytes, 0, 64, d->s_h2d));
	const unsigned long long *offs = d->d_offsets;
	for(uint32_t c = 0; c < nchunks; c++) {
		const uint32_t f0 = c * chunk, f1 = (f0 + chunk < nframes) ? f0 + chunk : nframes;
		const size_t b0 = (size_t)frame_offsets[f0], b1 = (size_t)frame_offsets[f1];
		if(b1 > b0) FB_CUDA(cudaMemcpyAsync(d->d_frames + b0, frames + b0, b1 - b0, cudaMemcpyHostToDevice, d->s_h2d));
		FB_CUDA(cudaEventRecord(d->ev_in[c], d->s_h2d));
		FB_CUDA(cudaStreamWaitEvent(d->stream, d->ev_in[c], 0));
		const uint64_t s0 = (uint64_t)f0 * bs;  // first sample (per channel) of the chunk
		const int rc = decode_ranges(d, d->k, d->want_subinfo, d->d_frames, offs + f0, offs + f0 + 1, f1 - f0, d->d_pcm + (size_t)s0 * ch, need_samples - s0, d->d_status + f0, nullptr, 0,
		                             d->stream, f0);
		if(rc != FB200_OK) return rc;
		const uint64_t s1 = (uint64_t)f1 * bs < cap ? (uint64_t)f1 * bs : cap;  // samples of this chunk the caller has room for
		if(s1 > s0) {
			const size_t n = (size_t)(s1 - s0) * ch;
			if(packed) {
				if(bytes_per_sample == 2) k_dec_pack<2><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm + (size_t)s0 * ch, d->d_packed + (size_t)s0 * ch * 2, n);
				else k_dec_pack<3><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm + (size_t)s0 * ch, d->d_packed + (size_t)s0 * ch * 3, n);
				d->launches++;
			}
			FB_CUDA(cudaEventRecord(d->ev_done[c], d->stream));
			FB_CUDA(cudaStreamWaitEvent(d->s_d2h, d->ev_done[c], 0));
			if(packed) FB_CUDA(cudaMemcpyAsync(static_cast<uint8_t *>(pcm_out) + (size_t)s0 * ch * bytes_per_sample, d->d_packed + (size_t)s0 * ch * bytes_per_sample, n * bytes_per_sample, cudaMemcpyDeviceToHost, d->s_d2h));
			else FB_CUDA(cudaMemcpyAsync(static_cast<int32_t *>(pcm_out) + (size_t)s0 * ch, d->d_pcm + (size_t)s0 * ch, n * sizeof(int32_t), cudaMemcpyDeviceToHost, d->s_d2h));
		}
	}
	d->h_status.resize(nframes);
	uint32_t *h_status = d->h_status.data();
	cudaError_t ce = cudaMemcpyAsync(h_status, d->d_status, (size_t)nframes * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream);
	if(ce == cudaSuccess) ce = cudaStreamSynchronize(d->stream);
	if(ce == cudaSuccess) ce = cudaStreamSynchronize(d->s_d2h);
	if(ce != cudaSuccess) {
		set_error("decode: %s", cudaGetErrorString(ce));
		return FB200_ERR_CUDA;
	}
	uint32_t bad = 0, first_bad = 0, first_code = 0;
	for(uint32_t i = 0; i < nframes; i++)
		if((h_status[i] & 0xffu) != DEC_OK) {
			if(!bad) { first_bad = i; first_code = h_status[i] & 0xffu; }
			bad++;
		}
	const uint64_t last_bs = h_status[nframes - 1] >> 8;
	if(bad_frames) *bad_frames = bad;
	if(samples_decoded) {
		const uint64_t n = (uint64_t)(nframes - 1) * bs + last_bs;
		*samples_decoded = n < cap ? n : cap;
	}
	if(bad) set_error("%u of %u frames failed to decode (first: frame %u, status %u)", bad, nframes, first_bad, first_code);
	return FB200_OK;
}

int fb200_decode_host(fb200_decoder *d, const uint8_t *frames, const uint64_t *frame_offsets, uint32_t nframes,
                      int32_t *pcm, uint64_t pcm_capacity_samples, uint64_t *samples_decoded, uint32_t *bad_frames)
{
	return decode_host_impl(d, frames, frame_offsets, nframes, pcm, 4, pcm_capacity_samples, samples_decoded, bad_frames);
}

int fb200_decode_host_packed(fb200_decoder *d, const uint8_t *frames, const uint64_t *frame_offsets, uint32_t nframes,
                             void *pcm, uint32_t bytes_per_sample, uint64_t pcm_capacity_samples, uint64_t *samples_decoded, uint32_t *bad_frames)
{
	return decode_host_impl(d, frames, frame_offsets, nframes, pcm, bytes_per_sample, pcm_capacity_samples, samples_decoded, bad_frames);
}


int fb200_decoder_get_frame_status(const fb200_decoder *d, uint32_t *status, uint32_t nframes)
{
	if(!d || !status) return FB200_ERR_INVALID;
	if(nframes > d->h_status.size()) { set_error("only %zu frames were decoded by the last call", d->h_status.size()); return FB200_ERR_INVALID; }
	memcpy(status, d->h_status.data(), (size_t)nframes * sizeof(uint32_t));
	return FB200_OK;
}

int fb200_decoder_enable_subframe_info(fb200_decoder *d, int on)
{
	if(!d) return FB200_ERR_INVALID;
	d->want_subinfo = on != 0;
	return FB200_OK;
}

int fb200_decoder_get_subframe_info(fb200_decoder *d, fb200_subframe_info *info, uint32_t nframes)
{
	if(!d || !info) return FB200_ERR_INVALID;
	static_assert(sizeof(fb200_subframe_info) == sizeof(DecSubframeInfo), "public and device subframe records must match");
	if(!d->want_subinfo || (size_t)nframes * d->cfg.channels > d->d_subinfo_cap) { set_error("subframe details were not collected for %u frames", nframes); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(d->device));
	FB_CUDA(cudaMemcpy(info, d->d_subinfo, (size_t)nframes * d->cfg.channels * sizeof(DecSubframeInfo), cudaMemcpyDeviceToHost));
	return FB200_OK;
}

// The decoder front end for a whole stream (frame_sync_ + read_frame_header_ for every byte position at once): offsets of
// every position that carries a sync code and a self-consistent frame header, ascending.
int fb200_decoder_index_host(fb200_decoder *d, const uint8_t *stream, uint64_t nbytes, uint64_t *candidates, uint32_t capacity, uint32_t *ncandidates)
{
	if(!d || (!stream && nbytes) || !candidates || !ncandidates) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(d->device));
	*ncandidates = 0;
	if(nbytes < 6) return FB200_OK;
	if(nbytes + 64 > d->d_stream_cap) {
		cudaFree(d->d_stream); d->d_stream = nullptr; d->d_stream_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_stream, nbytes + 64));
		d->d_stream_cap = nbytes + 64;
	}
	if(capacity > d->d_cand_cap) {
		cudaFree(d->d_cand); d->d_cand = nullptr; d->d_cand_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_cand, (size_t)capacity * sizeof(unsigned long long)));
		d->d_cand_cap = capacity;
	}
	if(!d->d_count) FB_CUDA(cudaMalloc(&d->d_count, sizeof(unsigned)));
	FB_CUDA(cudaMemcpyAsync(d->d_stream, stream, nbytes, cudaMemcpyHostToDevice, d->stream));
	FB_CUDA(cudaMemsetAsync(d->d_stream + nbytes, 0, 64, d->stream));
	FB_CUDA(cudaMemsetAsync(d->d_count, 0, sizeof(unsigned), d->stream));
	int nsm = 0;
	FB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, d->device));
	k_dec_scan<<<nsm * 8, 256, 0, d->stream>>>(d->d_stream, nbytes, d->d_cand, capacity, d->d_count);
	d->launches++;
	unsigned n = 0;
	FB_CUDA(cudaMemcpyAsync(&n, d->d_count, sizeof n, cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaStreamSynchronize(d->stream));
	if(n > capacity) { set_error("more than %u frame header candidates", capacity); return FB200_ERR_OUTPUT_TOO_SMALL; }
	FB_CUDA(cudaMemcpy(candidates, d->d_cand, (size_t)n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
	std::sort(candidates, candidates + n);
	*ncandidates = n;
	return FB200_OK;
}

// Decode the frames that START at begins[i] of the stream last given to fb200_decoder_index_host (still resident on the
// device); frame i may extend at most to begins[i] + max_frame_bytes (or the end of the stream): its true length comes out
// of the parse (frame_bytes[i]) and its CRC-16 is checked over exactly that. Frame i lands at sample offset i * blocksize.
int fb200_decode_indexed_host(fb200_decoder *d, const uint64_t *begins, uint32_t nframes, uint32_t max_frame_bytes, uint64_t stream_bytes,
                              int32_t *pcm, uint64_t pcm_capacity_samples, uint32_t *frame_status, uint32_t *frame_bytes)
{
	if(!d || !begins || !pcm || !frame_status || !frame_bytes) return FB200_ERR_INVALID;
	if(!d->d_stream || stream_bytes + 64 > d->d_stream_cap) { set_error("no indexed stream is resident"); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(d->device));
	if(nframes == 0) return FB200_OK;
	const uint64_t need_samples = (uint64_t)nframes * d->cfg.blocksize;
	const uint64_t cap = pcm_capacity_samples < need_samples ? pcm_capacity_samples : need_samples;
	if(2 * (size_t)nframes > d->d_offsets_cap) {
		cudaFree(d->d_offsets); d->d_offsets = nullptr; d->d_offsets_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_offsets, 2 * (size_t)nframes * sizeof(unsigned long long)));
		d->d_offsets_cap = 2 * (size_t)nframes;
	}
	if(need_samples * d->cfg.channels > d->d_pcm_cap) {
		cudaFree(d->d_pcm); d->d_pcm = nullptr; d->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_pcm, need_samples * d->cfg.channels * sizeof(int32_t)));
		d->d_pcm_cap = need_samples * d->cfg.channels;
	}
	if(nframes > d->d_status_cap) {
		cudaFree(d->d_status); d->d_status = nullptr; d->d_status_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_status, (size_t)nframes * sizeof(uint32_t)));
		d->d_status_cap = nframes;
	}
	if(nframes > d->d_fbytes_cap) {
		cudaFree(d->d_fbytes); d->d_fbytes = nullptr; d->d_fbytes_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_fbytes, (size_t)nframes * sizeof(uint32_t)));
		d->d_fbytes_cap = nframes;
	}
	std::vector<unsigned long long> be(2 * (size_t)nframes);
	for(uint32_t i = 0; i < nframes; i++) {
		be[i] = begins[i];
		const unsigned long long e = begins[i] + max_frame_bytes;
		be[nframes + i] = e < stream_bytes ? e : stream_bytes;
	}
	FB_CUDA(cudaMemcpyAsync(d->d_offsets, be.data(), be.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, d->stream));
	FB_CUDA(cudaMemsetAsync(d->d_fbytes, 0, (size_t)nframes * sizeof(uint32_t), d->stream));
	const int rc = decode_ranges(d, d->k, d->want_subinfo, d->d_stream, d->d_offsets, d->d_offsets + nframes, nframes, d->d_pcm, need_samples, d->d_status, d->d_fbytes, 1, d->stream);
	if(rc != FB200_OK) return rc;
	FB_CUDA(cudaMemcpyAsync(pcm, d->d_pcm, (size_t)cap * d->cfg.channels * sizeof(int32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaMemcpyAsync(frame_status, d->d_status, (size_t)nframes * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaMemcpyAsync(frame_bytes, d->d_fbytes, (size_t)nframes * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaStreamSynchronize(d->stream));
	d->h_status.assign(frame_status, frame_status + nframes);
	return FB200_OK;
}

// ---------------------------------------------------------------- batches of whole .flac files
// Index layout in d_findex (all arrays in group order): begins[ncand], ends[ncand], FileDecCand[ncand], FileDecState[files]
struct FilesIndexLayout {
	size_t begins, ends, cands, states, bytes;
	FilesIndexLayout(uint64_t ncand, size_t nstates)
	{
		size_t o = 0;
		begins = o; o = align16(o + ncand * sizeof(unsigned long long));
		ends = o; o = align16(o + ncand * sizeof(unsigned long long));
		cands = o; o = align16(o + ncand * sizeof(FileDecCand));
		states = o; o = align16(o + nstates * sizeof(FileDecState));
		bytes = o;
	}
};

int fb200_decode_files_index(fb200_decoder *d, const uint8_t *data, uint64_t nbytes, const uint64_t *file_offsets, uint32_t nfiles,
                             fb200_file_decode_info *files, uint64_t *total_values)
{
	if(!d || !data || !file_offsets || !files || !total_values || nfiles == 0) return FB200_ERR_INVALID;
	if(nfiles >= 0x7fffffffu) { set_error("too many files in one call"); return FB200_ERR_INVALID; }
	for(uint32_t f = 0; f < nfiles; f++)
		if(file_offsets[f] > file_offsets[f + 1]) { set_error("file offsets must ascend (file %u)", f); return FB200_ERR_INVALID; }
	if(file_offsets[nfiles] > nbytes) { set_error("file %u ends past the data", nfiles - 1); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(d->device));
	d->files_ready = false;

	// ---- metadata of every file (host)
	std::vector<FLAC__StreamMetadata_StreamInfo> si(nfiles);
	std::vector<uint64_t> audio0(nfiles);
	std::vector<uint32_t> mask(nfiles, 0);
	for(uint32_t f = 0; f < nfiles; f++) {
		fb200_file_decode_info &I = files[f];
		memset(&I, 0, sizeof I);
		const uint8_t *p = data + file_offsets[f];
		const size_t n = (size_t)(file_offsets[f + 1] - file_offsets[f]);
		bool has_si = false;
		uint32_t si_len = 0;
		size_t audio = 0;
		memset(&si[f], 0, sizeof si[f]);
		if(!walk_metadata(p, n, si[f], &has_si, &si_len, &audio)) { I.status = FB200_FILE_NOT_FLAC; continue; }
		mask[f] = channel_mask_tag(p, n);
		if(!has_si) { I.status = FB200_FILE_NO_STREAMINFO; continue; }
		const FLAC__StreamMetadata_StreamInfo &s = si[f];
		I.channels = s.channels; I.bits_per_sample = s.bits_per_sample; I.sample_rate = s.sample_rate;
		I.min_blocksize = s.min_blocksize; I.max_blocksize = s.max_blocksize; I.total_samples = s.total_samples;
		if(si_len != 34 || s.min_blocksize < 16 || s.max_blocksize < s.min_blocksize || s.sample_rate == 0 || s.bits_per_sample < 4)
			I.status = FB200_FILE_BAD_STREAMINFO;
		else if(s.bits_per_sample > 24) I.status = FB200_FILE_UNSUPPORTED;
		audio0[f] = file_offsets[f] + audio;
	}

	// ---- one k_dec_scan over the whole batch
	int rc;
	if((rc = grow((void **)&d->d_fdata, &d->d_fdata_cap, (size_t)nbytes + 64)) != FB200_OK) return rc;
	if(!d->d_count) FB_CUDA(cudaMalloc(&d->d_count, sizeof(unsigned)));
	FB_CUDA(cudaMemcpyAsync(d->d_fdata, data, (size_t)nbytes, cudaMemcpyHostToDevice, d->stream));
	FB_CUDA(cudaMemsetAsync(d->d_fdata + nbytes, 0, 64, d->stream));
	int nsm = 0;
	FB_CUDA(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, d->device));
	size_t cap = std::max<size_t>(1 << 16, (size_t)nbytes / 256);
	unsigned ncand = 0;
	for(;;) {
		if(cap > d->d_cand_cap) {
			cudaFree(d->d_cand); d->d_cand = nullptr; d->d_cand_cap = 0;
			FB_CUDA(cudaMalloc(&d->d_cand, cap * sizeof(unsigned long long)));
			d->d_cand_cap = cap;
		}
		FB_CUDA(cudaMemsetAsync(d->d_count, 0, sizeof(unsigned), d->stream));
		k_dec_scan<<<nsm * 8, 256, 0, d->stream>>>(d->d_fdata, nbytes, d->d_cand, (unsigned)cap, d->d_count);
		d->launches++;
		FB_CUDA(cudaMemcpyAsync(&ncand, d->d_count, sizeof ncand, cudaMemcpyDeviceToHost, d->stream));
		FB_CUDA(cudaStreamSynchronize(d->stream));
		if(ncand <= cap) break;
		cap = ncand;  // the count goes on past the capacity: one more scan with room for all
	}
	std::vector<uint64_t> cand(ncand);
	FB_CUDA(cudaMemcpy(cand.data(), d->d_cand, (size_t)ncand * sizeof(uint64_t), cudaMemcpyDeviceToHost));
	std::sort(cand.begin(), cand.end());

	// ---- each candidate to its file, kept when its header agrees with the file's STREAMINFO (dec_build_index in stream_api.cu)
	struct Cand { uint64_t begin, end; FileDecCand c; };
	std::vector<std::vector<Cand>> per_file(nfiles);
	uint32_t f = 0;
	for(uint32_t i = 0; i < ncand; i++) {
		const uint64_t pos = cand[i];
		while(f < nfiles && pos >= file_offsets[f + 1]) f++;
		if(f == nfiles) break;
		if(files[f].status != FB200_FILE_OK || pos < audio0[f]) continue;
		const FLAC__StreamMetadata_StreamInfo &s = si[f];
		const uint64_t fend = file_offsets[f + 1];
		FrameHeader fh;
		memset(&fh, 0, sizeof fh);
		if(parse_frame_header(data + pos, (size_t)(fend - pos), s.sample_rate, s.bits_per_sample, fh).status != DEC_OK) continue;
		if(fh.channels != s.channels || fh.bps != s.bits_per_sample || fh.blocksize > s.max_blocksize) continue;
		Cand c;
		c.begin = pos;
		// how far the frame may reach: twice the verbatim worst case, and never past its own file
		const uint64_t bound = 64 + 2 * (uint64_t)s.channels * (((uint64_t)s.max_blocksize * (s.bits_per_sample + 2) + 7) / 8 + 64);
		c.end = std::min<uint64_t>(fend, pos + bound);
		c.c.blocksize = fh.blocksize;
		c.c.rate_differs = fh.sample_rate != s.sample_rate;
		// the frame's first sample (stream_decoder.c:2915-2938); a frame number in a stream of varying blocksizes is not accepted
		if(fh.variable) c.c.first_sample = fh.number;
		else if(s.min_blocksize == s.max_blocksize) c.c.first_sample = fh.number * s.max_blocksize;
		else c.c.first_sample = ~0ull;
		per_file[f].push_back(c);
	}

	// ---- lengths and places in the output
	uint64_t values = 0;
	for(f = 0; f < nfiles; f++) {
		fb200_file_decode_info &I = files[f];
		I.first_value = values;
		if(I.status != FB200_FILE_OK) continue;
		uint64_t n = I.total_samples;
		if(n == 0)
			for(auto it = per_file[f].rbegin(); it != per_file[f].rend(); ++it)
				if(it->c.first_sample != ~0ull) { n = it->c.first_sample + it->c.blocksize; break; }
		I.samples = n;
		values += n * I.channels;
	}

	// ---- groups of (channels, bits per sample), their candidates back to back
	std::map<std::pair<uint32_t, uint32_t>, std::vector<uint32_t>> groups;
	for(f = 0; f < nfiles; f++)
		if(files[f].status == FB200_FILE_OK) groups[std::make_pair(files[f].channels, files[f].bits_per_sample)].push_back(f);
	d->files_groups.clear(); d->files_order.clear(); d->files_state0.clear();
	uint64_t total = 0;
	for(uint32_t g = 0; g < nfiles; g++) total += per_file[g].size();
	std::vector<unsigned long long> h_begins, h_ends;
	std::vector<FileDecCand> h_cands;
	h_begins.reserve(total); h_ends.reserve(total); h_cands.reserve(total);
	for(auto &g : groups) {
		fb200_decoder::FilesGroup G;
		G.channels = g.first.first; G.bps = g.first.second; G.max_bs = 16;
		G.cand0 = h_begins.size(); G.pos0 = (uint32_t)d->files_order.size(); G.nfiles = (uint32_t)g.second.size();
		for(uint32_t fi : g.second) {
			FileDecState S;
			memset(&S, 0, sizeof S);
			S.cand0 = h_begins.size(); S.ncand = per_file[fi].size();
			S.first_value = files[fi].first_value; S.end_sample = files[fi].samples; S.channels = files[fi].channels;
			for(const Cand &c : per_file[fi]) { h_begins.push_back(c.begin); h_ends.push_back(c.end); h_cands.push_back(c.c); }
			G.max_bs = std::max(G.max_bs, files[fi].max_blocksize);
			d->files_order.push_back(fi);
			d->files_state0.push_back(S);
		}
		G.ncand = h_begins.size() - G.cand0;
		d->files_groups.push_back(G);
	}
	const FilesIndexLayout L(total, d->files_state0.size());
	if((rc = grow((void **)&d->d_findex, &d->d_findex_cap, L.bytes + 16)) != FB200_OK) return rc;
	if(total) {
		FB_CUDA(cudaMemcpyAsync(d->d_findex + L.begins, h_begins.data(), total * sizeof(unsigned long long), cudaMemcpyHostToDevice, d->stream));
		FB_CUDA(cudaMemcpyAsync(d->d_findex + L.ends, h_ends.data(), total * sizeof(unsigned long long), cudaMemcpyHostToDevice, d->stream));
		FB_CUDA(cudaMemcpyAsync(d->d_findex + L.cands, h_cands.data(), total * sizeof(FileDecCand), cudaMemcpyHostToDevice, d->stream));
	}
	FB_CUDA(cudaStreamSynchronize(d->stream));
	d->files_info.assign(files, files + nfiles);
	d->files_md5.resize(nfiles);
	for(f = 0; f < nfiles; f++) memcpy(d->files_md5[f].data(), si[f].md5sum, 16);
	d->files_mask.swap(mask);
	d->files_start.assign(file_offsets, file_offsets + nfiles);
	d->files_audio.swap(audio0);
	d->files_end.assign(file_offsets + 1, file_offsets + nfiles + 1);
	d->files_pos.assign(nfiles, ~0u);
	for(uint32_t i = 0; i < d->files_order.size(); i++) d->files_pos[d->files_order[i]] = i;
	d->files_values = values;
	d->files_ncand = total;
	d->files_ready = true;
	*total_values = values;
	return FB200_OK;
}

// Candidates per chunk of a group: at most max_frames, and slots for at most FB200_DECODE_FILES_SAMPLE_BUDGET samples.
static uint64_t files_chunk(const fb200_decoder *d, const fb200_decoder::FilesGroup &G)
{
	const uint64_t per = (uint64_t)G.max_bs * G.channels;
	return std::max<uint64_t>(1, std::min<uint64_t>(d->max_frames, FB200_DECODE_FILES_SAMPLE_BUDGET / per));
}

// The states of one (channels, bits per sample) group and the candidates they own: states [0, nstates) (h_states a host copy,
// d_states on the device) hold, in order and back to back, candidates [cand0, cand0 + ncand) of begins / ends / cands.
struct FilesRun {
	const fb200_decoder::FilesGroup *group;
	uint64_t cand0, ncand;
	const FileDecState *h_states;
	FileDecState *d_states;
	uint32_t nstates;
	const unsigned long long *begins, *ends;
	const FileDecCand *cands;
};

// Decodes a run chunk by chunk: the frame decoder fills a slot per candidate, k_files_accept carries the states across the
// chunks, k_files_place copies what they accepted to d_out. d_stat / d_bytes / d_place hold files_chunk() entries; with keep,
// d_bytes / d_place hold one entry per candidate of the index instead, and every chunk's entries stay there.
static int decode_files_run(fb200_decoder *d, const FilesRun &R, uint32_t *d_stat, uint32_t *d_bytes, FilePlace *d_place, int32_t *d_out, cudaStream_t st,
                            const FileSeg *d_segs = nullptr, int nsegs = 0, bool keep = false)
{
	const fb200_decoder::FilesGroup &G = *R.group;
	DecK k;
	k.channels = (int)G.channels; k.bps = (int)G.bps; k.sample_rate = 0; k.blocksize = (int)G.max_bs; k.loose_end = 1;
	const uint64_t per = (uint64_t)G.max_bs * G.channels;
	const uint64_t chunk = files_chunk(d, G);
	uint32_t fa = 0;  // first state whose candidates reach into the chunk
	for(uint64_t c0 = R.cand0; c0 < R.cand0 + R.ncand; c0 += chunk) {
		const uint64_t c1 = std::min(c0 + chunk, R.cand0 + R.ncand);
		const uint32_t n = (uint32_t)(c1 - c0);
		while(fa < R.nstates && R.h_states[fa].cand0 + R.h_states[fa].ncand <= c0) fa++;
		uint32_t fb = fa;
		while(fb < R.nstates && R.h_states[fb].cand0 < c1) fb++;
		FB_CUDA(cudaMemsetAsync(d_stat, 0xff, (size_t)n * sizeof(uint32_t), st));  // a candidate without a verdict is never accepted
		int rc;
		uint32_t *bytes = keep ? d_bytes + c0 : d_bytes;
		FilePlace *place = keep ? d_place + c0 : d_place;
		if((rc = decode_ranges(d, k, false, d->d_fdata, R.begins + c0, R.ends + c0, n, d->d_fslots, (uint64_t)n * G.max_bs, d_stat, bytes, 1, st)) != FB200_OK)
			return rc;
		launch_files_accept(R.d_states + fa, (int)(fb - fa), R.begins, R.cands, d_stat, bytes, c0, c1, place, st);
		launch_files_place(d->d_fslots, per, place, n, d_out, d_segs, nsegs, st);
		d->launches += 2;
	}
	return FB200_OK;
}

// Decodes the resident batch into d_out (int32, total values, zeroed first). skip_bps: groups deeper than this are not decoded
// (FB200_FILE_WIDTH). Returns after completion with files[] filled. With kept, every candidate's place (FilePlace, indexed as the
// resident index) is copied there too.
static int decode_files_impl(fb200_decoder *d, int32_t *d_out, uint32_t skip_bps, int do_md5, fb200_file_decode_info *files, cudaStream_t st,
                             std::vector<FilePlace> *kept = nullptr)
{
	const uint32_t nfiles = (uint32_t)d->files_info.size();
	const FilesIndexLayout L(d->files_ncand, d->files_state0.size());
	const unsigned long long *d_begins = reinterpret_cast<const unsigned long long *>(d->d_findex + L.begins);
	const unsigned long long *d_ends = reinterpret_cast<const unsigned long long *>(d->d_findex + L.ends);
	const FileDecCand *d_cands = reinterpret_cast<const FileDecCand *>(d->d_findex + L.cands);
	FileDecState *d_states = reinterpret_cast<FileDecState *>(d->d_findex + L.states);
	std::vector<fb200_file_decode_info> info(d->files_info);
	std::vector<bool> skipped(nfiles, false);
	uint64_t chunk_max = 1, slot_values_max = 0;
	for(const auto &G : d->files_groups) {
		if(G.bps > skip_bps) continue;
		const uint64_t per = (uint64_t)G.max_bs * G.channels;
		const uint64_t c = files_chunk(d, G);
		chunk_max = std::max(chunk_max, c);
		slot_values_max = std::max(slot_values_max, c * per);
	}
	// MD5 segments: one per checked file (+ an empty tail), files grouped by sample width
	std::vector<FileSeg> segs;
	std::vector<uint32_t> md5_file;
	int width_first[5] = {0}, width_count[5] = {0};
	for(uint32_t w = 1; w <= 4; w++) {
		width_first[w] = (int)md5_file.size();
		for(uint32_t i = 0; i < d->files_order.size(); i++) {
			const uint32_t f = d->files_order[i];
			const fb200_file_decode_info &I = info[f];
			if(!do_md5 || I.bits_per_sample > skip_bps || (I.bits_per_sample + 7) / 8 != w) continue;
			static const uint8_t zero[16] = {0};
			if(memcmp(d->files_md5[f].data(), zero, 16) == 0) continue;  // an all-zero STREAMINFO MD5 is not checked
			segs.push_back(FileSeg{0, I.first_value, I.samples * I.channels, 0});
			segs.push_back(FileSeg{0, 0, 0, 0});
			md5_file.push_back(f);
		}
		width_count[w] = (int)md5_file.size() - width_first[w];
	}
	const size_t o_stat = 0;
	const size_t o_bytes = align16(o_stat + chunk_max * sizeof(uint32_t));
	const size_t o_place = align16(o_bytes + chunk_max * sizeof(uint32_t));
	const size_t o_segs = align16(o_place + chunk_max * sizeof(FilePlace));
	const size_t o_md5 = align16(o_segs + segs.size() * sizeof(FileSeg));
	const size_t work = o_md5 + 16 * md5_file.size() + 16;
	int rc;
	if((rc = grow((void **)&d->d_fwork, &d->d_fwork_cap, work)) != FB200_OK) return rc;
	if((rc = grow((void **)&d->d_fslots, &d->d_fslots_cap, (size_t)slot_values_max * sizeof(int32_t) + 16)) != FB200_OK) return rc;
	uint32_t *d_stat = reinterpret_cast<uint32_t *>(d->d_fwork + o_stat);
	uint32_t *d_bytes = reinterpret_cast<uint32_t *>(d->d_fwork + o_bytes);
	FilePlace *d_place = reinterpret_cast<FilePlace *>(d->d_fwork + o_place);
	const size_t k_bytes = align16((size_t)d->files_ncand * sizeof(FilePlace));
	if(kept) {
		if((rc = grow((void **)&d->d_keep, &d->d_keep_cap, k_bytes + (size_t)d->files_ncand * sizeof(uint32_t) + 16)) != FB200_OK) return rc;
		if(d->files_ncand) FB_CUDA(cudaMemsetAsync(d->d_keep, 0, k_bytes, st));
	}

	if(!d->files_state0.empty())
		FB_CUDA(cudaMemcpyAsync(d_states, d->files_state0.data(), d->files_state0.size() * sizeof(FileDecState), cudaMemcpyHostToDevice, st));
	if(!segs.empty()) FB_CUDA(cudaMemcpyAsync(d->d_fwork + o_segs, segs.data(), segs.size() * sizeof(FileSeg), cudaMemcpyHostToDevice, st));
	if(d->files_values) FB_CUDA(cudaMemsetAsync(d_out, 0, (size_t)d->files_values * sizeof(int32_t), st));
	for(const auto &G : d->files_groups) {
		if(G.bps > skip_bps) {
			for(uint32_t i = 0; i < G.nfiles; i++) skipped[d->files_order[G.pos0 + i]] = true;
			continue;
		}
		const FilesRun R{&G, G.cand0, G.ncand, d->files_state0.data() + G.pos0, d_states + G.pos0, G.nfiles, d_begins, d_ends, d_cands};
		if(kept) rc = decode_files_run(d, R, d_stat, reinterpret_cast<uint32_t *>(d->d_keep + k_bytes), reinterpret_cast<FilePlace *>(d->d_keep), d_out, st,
		                               nullptr, 0, true);
		else rc = decode_files_run(d, R, d_stat, d_bytes, d_place, d_out, st);
		if(rc != FB200_OK) return rc;
	}
	if(kept) {
		kept->resize(d->files_ncand);
		if(d->files_ncand) FB_CUDA(cudaMemcpyAsync(kept->data(), d->d_keep, (size_t)d->files_ncand * sizeof(FilePlace), cudaMemcpyDeviceToHost, st));
	}
	uint8_t *d_digests = d->d_fwork + o_md5;
	for(int w = 1; w <= 4; w++)
		if(width_count[w]) {
			launch_md5_files(d_out, reinterpret_cast<const FileSeg *>(d->d_fwork + o_segs) + 2 * width_first[w], width_count[w], w, d_digests + 16 * (size_t)width_first[w], st);
			d->launches++;
		}
	FB_CUDA(cudaGetLastError());
	std::vector<FileDecState> states(d->files_state0.size());
	std::vector<uint8_t> digests(16 * md5_file.size());
	if(!states.empty()) FB_CUDA(cudaMemcpyAsync(states.data(), d_states, states.size() * sizeof(FileDecState), cudaMemcpyDeviceToHost, st));
	if(!digests.empty()) FB_CUDA(cudaMemcpyAsync(digests.data(), d_digests, digests.size(), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	for(uint32_t i = 0; i < d->files_order.size(); i++) {
		const uint32_t f = d->files_order[i];
		fb200_file_decode_info &I = info[f];
		if(skipped[f]) { I.status = FB200_FILE_WIDTH; I.samples_missing = I.samples; continue; }
		I.nframes = states[i].nframes;
		I.errors = states[i].errors;
		I.samples_missing = I.samples - states[i].covered;
	}
	for(size_t j = 0; j < md5_file.size(); j++) {
		fb200_file_decode_info &I = info[md5_file[j]];
		memcpy(I.md5, digests.data() + 16 * j, 16);
		I.md5_state = memcmp(I.md5, d->files_md5[md5_file[j]].data(), 16) == 0 ? 1 : 2;
	}
	memcpy(files, info.data(), info.size() * sizeof(fb200_file_decode_info));
	return FB200_OK;
}

int fb200_decode_files_device(fb200_decoder *d, int32_t *d_pcm, uint64_t pcm_capacity_values, int do_md5, fb200_file_decode_info *files, void *cuda_stream)
{
	if(!d || !d_pcm || !files) return FB200_ERR_INVALID;
	if(!d->files_ready) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	if(pcm_capacity_values < d->files_values) { set_error("output holds %llu values, the batch needs %llu", (unsigned long long)pcm_capacity_values, (unsigned long long)d->files_values); return FB200_ERR_OUTPUT_TOO_SMALL; }
	FB_CUDA(cudaSetDevice(d->device));
	return decode_files_impl(d, d_pcm, 32, do_md5, files, (cudaStream_t)cuda_stream);
}

// Decodes on the device, then narrows (k_dec_pack) and copies back; the copies do not overlap compute.
int fb200_decode_files_host(fb200_decoder *d, void *pcm, uint32_t bytes_per_sample, uint64_t pcm_capacity_values, int do_md5, fb200_file_decode_info *files)
{
	if(!d || !pcm || !files) return FB200_ERR_INVALID;
	if(bytes_per_sample != 2 && bytes_per_sample != 3 && bytes_per_sample != 4) { set_error("bytes_per_sample must be 2, 3 or 4"); return FB200_ERR_INVALID; }
	if(!d->files_ready) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	if(pcm_capacity_values < d->files_values) { set_error("output holds %llu values, the batch needs %llu", (unsigned long long)pcm_capacity_values, (unsigned long long)d->files_values); return FB200_ERR_OUTPUT_TOO_SMALL; }
	FB_CUDA(cudaSetDevice(d->device));
	const size_t n = (size_t)d->files_values;
	int rc;
	if(n + 4 > d->d_pcm_cap) {
		cudaFree(d->d_pcm); d->d_pcm = nullptr; d->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_pcm, (n + 4) * sizeof(int32_t)));
		d->d_pcm_cap = n + 4;
	}
	if(bytes_per_sample != 4 && (rc = grow((void **)&d->d_packed, &d->d_packed_cap, n * bytes_per_sample + 16)) != FB200_OK) return rc;
	if((rc = decode_files_impl(d, d->d_pcm, 8 * bytes_per_sample, do_md5, files, d->stream)) != FB200_OK) return rc;
	if(n == 0) return FB200_OK;
	if(bytes_per_sample == 4) FB_CUDA(cudaMemcpy(pcm, d->d_pcm, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
	else {
		if(bytes_per_sample == 2) k_dec_pack<2><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm, d->d_packed, n);
		else k_dec_pack<3><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm, d->d_packed, n);
		d->launches++;
		FB_CUDA(cudaGetLastError());
		FB_CUDA(cudaMemcpyAsync(pcm, d->d_packed, n * bytes_per_sample, cudaMemcpyDeviceToHost, d->stream));
		FB_CUDA(cudaStreamSynchronize(d->stream));
	}
	return FB200_OK;
}


// ---------------------------------------------------------------- sample ranges of the resident batch
// The output layout of a ranged call: info[r]'s status, format and place, *total_values. skip_bps: files deeper than this get
// FB200_FILE_WIDTH. Fails with FB200_ERR_INVALID, before any work, on a request that does not fit the batch.
static int ranges_layout(const fb200_decoder *d, const fb200_sample_range *ranges, uint32_t nranges, uint32_t skip_bps, fb200_range_decode_info *info,
                         uint64_t *total_values)
{
	if(!d->files_ready) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	if(nranges == 0 || nranges >= 0x80000000u) { set_error("invalid number of ranges %u", nranges); return FB200_ERR_INVALID; }
	const uint32_t nfiles = (uint32_t)d->files_info.size();
	for(uint32_t r = 0; r < nranges; r++) {
		const fb200_sample_range &q = ranges[r];
		if(q.file >= nfiles) { set_error("range %u: file %u of a batch of %u", r, q.file, nfiles); return FB200_ERR_INVALID; }
		if(q.samples == 0) { set_error("range %u is empty", r); return FB200_ERR_INVALID; }
		if(q.first_sample + q.samples < q.first_sample) { set_error("range %u: first_sample + samples overflows", r); return FB200_ERR_INVALID; }
		const fb200_file_decode_info &I = d->files_info[q.file];
		if(I.status == FB200_FILE_OK && q.first_sample + q.samples > I.samples) {
			set_error("range %u: samples [%llu, %llu) of file %u, which has %llu", r, (unsigned long long)q.first_sample,
			          (unsigned long long)(q.first_sample + q.samples), q.file, (unsigned long long)I.samples);
			return FB200_ERR_INVALID;
		}
	}
	uint64_t values = 0;
	for(uint32_t r = 0; r < nranges; r++) {
		const fb200_sample_range &q = ranges[r];
		const fb200_file_decode_info &I = d->files_info[q.file];
		fb200_range_decode_info &R = info[r];
		memset(&R, 0, sizeof R);
		R.status = I.status == FB200_FILE_OK && I.bits_per_sample > skip_bps ? (uint32_t)FB200_FILE_WIDTH : I.status;
		R.channels = I.channels; R.bits_per_sample = I.bits_per_sample;
		R.first_value = values;
		R.values = R.status == FB200_FILE_OK ? q.samples * I.channels : 0;
		R.samples_missing = q.samples;
		values += R.values;
	}
	*total_values = values;
	return FB200_OK;
}

// Decodes the ranges whose layout ranges_layout() gave into d_out (int32, total values, zeroed first). Returns after completion
// with nframes / samples_missing / candidates of info[] filled (and errors[r], when given, with range r's damaged stretches +
// overlapping frames). The resident index is only read. With kept, the place of every candidate selected for range r is copied to
// (*kept)[kept0[r] ..], info[r].candidates of them. With d_segs (nsegs of them, a batch's FileSeg pairs), info[r].first_value is
// a value index in the back-to-back numbering of FileSeg::src and the frames are placed through the segments into d_out, the
// compacted layout `total` values long (decoder_decode_into's placement).
static int decode_files_ranges_impl(fb200_decoder *d, const fb200_sample_range *ranges, uint32_t nranges, int32_t *d_out, uint64_t total,
                                    fb200_range_decode_info *info, cudaStream_t st, uint32_t *errors = nullptr, std::vector<FilePlace> *kept = nullptr,
                                    std::vector<uint64_t> *kept0 = nullptr, const FileSeg *d_segs = nullptr, int nsegs = 0)
{
	const uint32_t nfiles = (uint32_t)d->files_info.size(), ngroups = (uint32_t)d->files_groups.size();
	const FilesIndexLayout L(d->files_ncand, d->files_state0.size());
	const unsigned long long *d_begins = reinterpret_cast<const unsigned long long *>(d->d_findex + L.begins);
	const unsigned long long *d_ends = reinterpret_cast<const unsigned long long *>(d->d_findex + L.ends);
	const FileDecCand *d_cands = reinterpret_cast<const FileDecCand *>(d->d_findex + L.cands);
	// each file's group and place in group order
	std::vector<uint32_t> file_group(nfiles, ~0u), file_pos(nfiles, 0);
	for(uint32_t g = 0; g < ngroups; g++)
		for(uint32_t i = 0; i < d->files_groups[g].nfiles; i++) {
			const uint32_t p = d->files_groups[g].pos0 + i;
			file_group[d->files_order[p]] = g;
			file_pos[d->files_order[p]] = p;
		}
	// the ranges to decode, grouped (request order within a group): order[gfirst[g] .. gfirst[g + 1])
	std::vector<uint32_t> gfirst(ngroups + 1, 0), order;
	for(uint32_t r = 0; r < nranges; r++)
		if(info[r].status == FB200_FILE_OK) gfirst[file_group[ranges[r].file] + 1]++;
	for(uint32_t g = 0; g < ngroups; g++) gfirst[g + 1] += gfirst[g];
	order.resize(gfirst[ngroups]);
	{
		std::vector<uint32_t> fill(gfirst.begin(), gfirst.end() - 1);
		for(uint32_t r = 0; r < nranges; r++)
			if(info[r].status == FB200_FILE_OK) order[fill[file_group[ranges[r].file]]++] = r;
	}
	const uint32_t n = (uint32_t)order.size();
	int rc;
	if(total) FB_CUDA(cudaMemsetAsync(d_out, 0, (size_t)total * sizeof(int32_t), st));
	if(n == 0) {
		FB_CUDA(cudaStreamSynchronize(st));
		return FB200_OK;
	}

	// ---- selection: count, then (after an exclusive scan here) compact each range's candidates
	const size_t o_sel = 0;
	const size_t o_count = align16(o_sel + n * sizeof(RangeSel));
	const size_t o_dst = align16(o_count + n * sizeof(uint32_t));
	const size_t o_states = align16(o_dst + n * sizeof(unsigned long long));
	if((rc = grow((void **)&d->d_rwork, &d->d_rwork_cap, align16(o_states + n * sizeof(FileDecState)))) != FB200_OK) return rc;
	RangeSel *d_sel = reinterpret_cast<RangeSel *>(d->d_rwork + o_sel);
	uint32_t *d_count = reinterpret_cast<uint32_t *>(d->d_rwork + o_count);
	unsigned long long *d_dst = reinterpret_cast<unsigned long long *>(d->d_rwork + o_dst);
	FileDecState *d_states = reinterpret_cast<FileDecState *>(d->d_rwork + o_states);
	std::vector<RangeSel> sel(n);
	for(uint32_t i = 0; i < n; i++) {
		const fb200_sample_range &q = ranges[order[i]];
		const FileDecState &F = d->files_state0[file_pos[q.file]];
		sel[i] = RangeSel{F.cand0, F.ncand, q.first_sample, q.first_sample + q.samples};
	}
	std::vector<uint32_t> count(n);
	FB_CUDA(cudaMemcpyAsync(d_sel, sel.data(), n * sizeof(RangeSel), cudaMemcpyHostToDevice, st));
	launch_ranges_count(d_sel, (int)n, d_cands, d_count, st);
	d->launches++;
	FB_CUDA(cudaMemcpyAsync(count.data(), d_count, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	FB_CUDA(cudaGetLastError());
	std::vector<unsigned long long> dst(n);
	std::vector<FileDecState> states(n);
	uint64_t nsel = 0;
	for(uint32_t i = 0; i < n; i++) {
		const fb200_sample_range &q = ranges[order[i]];
		dst[i] = nsel;
		FileDecState &S = states[i];
		memset(&S, 0, sizeof S);
		S.cand0 = nsel; S.ncand = count[i];
		S.first_value = info[order[i]].first_value; S.first_sample = q.first_sample; S.end_sample = q.first_sample + q.samples;
		S.channels = info[order[i]].channels;
		nsel += count[i];
	}
	const size_t o_rbeg = 0;
	const size_t o_rend = align16(o_rbeg + nsel * sizeof(unsigned long long));
	const size_t o_rcand = align16(o_rend + nsel * sizeof(unsigned long long));
	if((rc = grow((void **)&d->d_rcand, &d->d_rcand_cap, align16(o_rcand + nsel * sizeof(FileDecCand)) + 16)) != FB200_OK) return rc;
	unsigned long long *d_rbeg = reinterpret_cast<unsigned long long *>(d->d_rcand + o_rbeg);
	unsigned long long *d_rend = reinterpret_cast<unsigned long long *>(d->d_rcand + o_rend);
	FileDecCand *d_rcands = reinterpret_cast<FileDecCand *>(d->d_rcand + o_rcand);
	FB_CUDA(cudaMemcpyAsync(d_dst, dst.data(), n * sizeof(unsigned long long), cudaMemcpyHostToDevice, st));
	FB_CUDA(cudaMemcpyAsync(d_states, states.data(), n * sizeof(FileDecState), cudaMemcpyHostToDevice, st));
	if(nsel) {
		launch_ranges_select(d_sel, (int)n, d_begins, d_ends, d_cands, d_dst, d_rbeg, d_rend, d_rcands, st);
		d->launches++;
	}

	// ---- per group and chunk: the frame decoder, k_files_accept, k_files_place over the selected candidates
	uint64_t chunk_max = 1, slot_values_max = 0;
	for(uint32_t g = 0; g < ngroups; g++) {
		if(gfirst[g] == gfirst[g + 1]) continue;
		const fb200_decoder::FilesGroup &G = d->files_groups[g];
		const uint64_t c = files_chunk(d, G);
		chunk_max = std::max(chunk_max, c);
		slot_values_max = std::max(slot_values_max, c * G.max_bs * G.channels);
	}
	const size_t o_stat = 0;
	const size_t o_bytes = align16(o_stat + chunk_max * sizeof(uint32_t));
	const size_t o_place = align16(o_bytes + chunk_max * sizeof(uint32_t));
	if((rc = grow((void **)&d->d_fwork, &d->d_fwork_cap, align16(o_place + chunk_max * sizeof(FilePlace)))) != FB200_OK) return rc;
	if((rc = grow((void **)&d->d_fslots, &d->d_fslots_cap, (size_t)slot_values_max * sizeof(int32_t) + 16)) != FB200_OK) return rc;
	uint32_t *d_stat = reinterpret_cast<uint32_t *>(d->d_fwork + o_stat);
	uint32_t *d_bytes = reinterpret_cast<uint32_t *>(d->d_fwork + o_bytes);
	FilePlace *d_place = reinterpret_cast<FilePlace *>(d->d_fwork + o_place);
	const size_t k_bytes = align16((size_t)nsel * sizeof(FilePlace));
	if(kept) {
		if((rc = grow((void **)&d->d_keep, &d->d_keep_cap, k_bytes + (size_t)nsel * sizeof(uint32_t) + 16)) != FB200_OK) return rc;
		if(nsel) FB_CUDA(cudaMemsetAsync(d->d_keep, 0, k_bytes, st));
	}
	for(uint32_t g = 0; g < ngroups; g++) {
		const uint32_t a = gfirst[g], b = gfirst[g + 1];
		if(a == b) continue;
		const uint64_t c0 = dst[a], c1 = b < n ? dst[b] : nsel;
		const FilesRun R{&d->files_groups[g], c0, c1 - c0, states.data() + a, d_states + a, b - a, d_rbeg, d_rend, d_rcands};
		if(kept) rc = decode_files_run(d, R, d_stat, reinterpret_cast<uint32_t *>(d->d_keep + k_bytes), reinterpret_cast<FilePlace *>(d->d_keep), d_out, st,
		                               nullptr, 0, true);
		else rc = decode_files_run(d, R, d_stat, d_bytes, d_place, d_out, st, d_segs, nsegs);
		if(rc != FB200_OK) return rc;
	}
	if(kept) {
		kept->resize(nsel);
		kept0->assign(nranges, 0);
		for(uint32_t i = 0; i < n; i++) (*kept0)[order[i]] = dst[i];
		if(nsel) FB_CUDA(cudaMemcpyAsync(kept->data(), d->d_keep, (size_t)nsel * sizeof(FilePlace), cudaMemcpyDeviceToHost, st));
	}
	FB_CUDA(cudaGetLastError());
	FB_CUDA(cudaMemcpyAsync(states.data(), d_states, n * sizeof(FileDecState), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	for(uint32_t i = 0; i < n; i++) {
		fb200_range_decode_info &I = info[order[i]];
		I.nframes = states[i].nframes;
		I.samples_missing = ranges[order[i]].samples - states[i].covered;
		I.candidates = count[i];
		if(errors) errors[order[i]] = states[i].errors;
	}
	return FB200_OK;
}

int fb200_decode_files_ranges_device(fb200_decoder *d, const fb200_sample_range *ranges, uint32_t nranges, int32_t *d_pcm, uint64_t pcm_capacity_values,
                                     uint64_t *total_values, fb200_range_decode_info *info, void *cuda_stream)
{
	if(!d || !ranges || !total_values || !info) return FB200_ERR_INVALID;
	int rc;
	if((rc = ranges_layout(d, ranges, nranges, 32, info, total_values)) != FB200_OK) return rc;
	const uint64_t n = *total_values;
	if(pcm_capacity_values < n) { set_error("output holds %llu values, the ranges need %llu", (unsigned long long)pcm_capacity_values, (unsigned long long)n); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if(!d_pcm && n) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(d->device));
	return decode_files_ranges_impl(d, ranges, nranges, d_pcm, n, info, (cudaStream_t)cuda_stream);
}

// Decodes on the device, then narrows (k_dec_pack) and copies back; the copies do not overlap compute.
int fb200_decode_files_ranges_host(fb200_decoder *d, const fb200_sample_range *ranges, uint32_t nranges, void *pcm, uint32_t bytes_per_sample,
                                   uint64_t pcm_capacity_values, uint64_t *total_values, fb200_range_decode_info *info)
{
	if(!d || !ranges || !total_values || !info) return FB200_ERR_INVALID;
	if(bytes_per_sample != 2 && bytes_per_sample != 3 && bytes_per_sample != 4) { set_error("bytes_per_sample must be 2, 3 or 4"); return FB200_ERR_INVALID; }
	int rc;
	if((rc = ranges_layout(d, ranges, nranges, 8 * bytes_per_sample, info, total_values)) != FB200_OK) return rc;
	const size_t n = (size_t)*total_values;
	if(pcm_capacity_values < n) { set_error("output holds %llu values, the ranges need %llu", (unsigned long long)pcm_capacity_values, (unsigned long long)n); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if(!pcm && n) return FB200_ERR_INVALID;
	FB_CUDA(cudaSetDevice(d->device));
	if(n + 4 > d->d_pcm_cap) {
		cudaFree(d->d_pcm); d->d_pcm = nullptr; d->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_pcm, (n + 4) * sizeof(int32_t)));
		d->d_pcm_cap = n + 4;
	}
	if(bytes_per_sample != 4 && (rc = grow((void **)&d->d_packed, &d->d_packed_cap, n * bytes_per_sample + 16)) != FB200_OK) return rc;
	if((rc = decode_files_ranges_impl(d, ranges, nranges, d->d_pcm, n, info, d->stream)) != FB200_OK) return rc;
	if(n == 0) return FB200_OK;
	if(bytes_per_sample == 4) FB_CUDA(cudaMemcpy(pcm, d->d_pcm, n * sizeof(int32_t), cudaMemcpyDeviceToHost));
	else {
		if(bytes_per_sample == 2) k_dec_pack<2><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm, d->d_packed, n);
		else k_dec_pack<3><<<(unsigned)((n / 4 + 256) / 256), 256, 0, d->stream>>>(d->d_pcm, d->d_packed, n);
		d->launches++;
		FB_CUDA(cudaGetLastError());
		FB_CUDA(cudaMemcpyAsync(pcm, d->d_packed, n * bytes_per_sample, cudaMemcpyDeviceToHost, d->stream));
		FB_CUDA(cudaStreamSynchronize(d->stream));
	}
	return FB200_OK;
}

// ---------------------------------------------------------------- the resident batch as container files (flac -d)
// The delivered blocks of one container (the accepted frames' parts inside it, in order, as FilePlace entries of its values from
// value v0 on) as k_rg_synth takes them: appended to blocks, gaps filled so that they tile [0, ns). Returns the samples the tool
// writes before its first error: the blocks before the first sample no frame covers.
static uint64_t rgs_blocks(const FilePlace *place, uint64_t nplace, uint64_t v0, uint32_t C, uint64_t ns, std::vector<RgsBlock> &blocks)
{
	uint64_t pos = 0, delivered = 0;
	bool whole = true;
	for(uint64_t k = 0; k < nplace; k++) {
		const FilePlace &q = place[k];
		if(q.n == 0) continue;
		const uint64_t s = (q.dst - v0) / C, m = q.n / C;
		if(s > pos) {
			blocks.push_back(RgsBlock{pos, s - pos});
			whole = false;
		}
		blocks.push_back(RgsBlock{s, m});
		pos = s + m;
		if(whole) delivered = pos;
	}
	if(pos < ns) blocks.push_back(RgsBlock{pos, ns - pos});
	return delivered;
}

// Sizes every container on the host, decodes into the int32 scratch by the whole-file or the ranged path, then packs every
// container with one k_pcm_pack launch into `out` (device memory; the caller's with _device, d_packed with _host). With rg, the
// containers the tool applies ReplayGain to get apply_gain's values (k_rg_synth, in place in the scratch) and are packed with
// shift 0; rginfo[n] receives the decisions and draw positions.
static int decode_pcm_files(fb200_decoder *d, const fb200_pcm_decode_options *opt, const fb200_sample_range *ranges, uint32_t nranges, bool host,
                            uint8_t *out, uint64_t out_capacity, uint64_t *total_bytes, fb200_pcm_decode_info *info, cudaStream_t st,
                            const fb200_replaygain_synthesis *rg = nullptr, fb200_replaygain_synthesis_info *rginfo = nullptr)
{
	if(!d || !total_bytes || !info) return FB200_ERR_INVALID;
	if(!pcm_decode_options_ok(opt)) return FB200_ERR_INVALID;
	if(!d->files_ready) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	const bool whole = ranges == nullptr;
	const uint32_t n = whole ? (uint32_t)d->files_info.size() : nranges;
	int rc;
	std::vector<fb200_range_decode_info> rinfo;
	uint64_t rvalues = 0;
	if(!whole) {
		rinfo.resize(nranges ? nranges : 1);
		if((rc = ranges_layout(d, ranges, nranges, 32, rinfo.data(), &rvalues)) != FB200_OK) return rc;
	}
	// ---- every container's header and length
	std::vector<PcmHeader> heads(n);
	uint64_t off = 0;
	for(uint32_t i = 0; i < n; i++) {
		const uint32_t f = whole ? i : ranges[i].file;
		const fb200_file_decode_info &F = d->files_info[f];
		fb200_pcm_decode_info &I = info[i];
		memset(&I, 0, sizeof I);
		I.status = whole ? F.status : rinfo[i].status;
		if(!whole && I.status == FB200_FILE_OK && F.total_samples == 0) I.status = FB200_FILE_NO_TOTAL;  // decode.c:1347-1362
		I.channels = F.channels; I.bits_per_sample = F.bits_per_sample; I.sample_rate = F.sample_rate;
		I.offset = off;
		if(I.status != FB200_FILE_OK) continue;
		I.samples = whole ? F.samples : ranges[i].samples;
		PcmHeader &h = heads[i];
		pcm_header_build(*opt, F.channels, F.bits_per_sample, F.sample_rate, d->files_mask[f], I.samples, &h);
		if(h.too_big) { I.status = FB200_FILE_TOO_BIG; I.samples = 0; continue; }
		// the pad is sized from STREAMINFO's total_samples (decode.c:551-574); with 0 there, fixup_iff_headers only rewrites the header
		if(F.total_samples == 0) h.pad = 0;
		I.container_bits = h.container_bits; I.channel_mask = h.mask; I.extensible = h.extensible; I.header_bytes = h.length;
		I.bytes = h.length + h.data_bytes + h.pad;
		off += I.bytes;
	}
	*total_bytes = off;
	if(rg) {
		// the tool's decision per container, from its file's metadata (each file read once)
		std::map<uint32_t, fb200_replaygain_synthesis_info> seen;
		FB_CUDA(cudaSetDevice(d->device));
		for(uint32_t i = 0; i < n; i++) {
			fb200_replaygain_synthesis_info &R = rginfo[i];
			memset(&R, 0, sizeof R);
			R.status = FB200_RGS_NOT_DECODED;
			if(info[i].status != FB200_FILE_OK) continue;
			const uint32_t f = whole ? i : ranges[i].file;
			auto it = seen.find(f);
			if(it == seen.end()) {
				std::vector<uint8_t> meta;
				if((rc = decoder_file_metadata(d, f, &meta)) != FB200_OK) return rc;
				fb200_replaygain_synthesis_info D;
				rgs_decide(meta.data(), meta.size(), d->files_info[f].bits_per_sample, *rg, &D);
				it = seen.emplace(f, D).first;
			}
			R = it->second;
		}
	}
	if(out_capacity < off) { set_error("output holds %llu bytes, the containers need %llu", (unsigned long long)out_capacity, (unsigned long long)off); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if(!out && off) { set_error("out is NULL"); return FB200_ERR_INVALID; }
	FB_CUDA(cudaSetDevice(d->device));

	// ---- decode into the int32 scratch
	const uint64_t values = whole ? d->files_values : rvalues;
	if(values + 4 > d->d_pcm_cap) {
		cudaFree(d->d_pcm); d->d_pcm = nullptr; d->d_pcm_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_pcm, (values + 4) * sizeof(int32_t)));
		d->d_pcm_cap = values + 4;
	}
	std::vector<fb200_file_decode_info> finfo(whole ? n : 0);
	std::vector<uint32_t> rerr(whole ? 0 : n, 0);
	bool applied = false;
	for(uint32_t i = 0; rg && i < n; i++) applied |= info[i].status == FB200_FILE_OK && rginfo[i].status == FB200_RGS_APPLIED;
	std::vector<FilePlace> kept;
	std::vector<uint64_t> kept0;
	const bool keep = applied && rg->noise_shaping != 0;
	if(whole) rc = decode_files_impl(d, d->d_pcm, 24, opt->md5 ? 1 : 0, finfo.data(), st, keep ? &kept : nullptr);
	else {
		for(uint32_t i = 0; i < n; i++)
			if(info[i].status != FB200_FILE_OK) rinfo[i].status = info[i].status;  // not decoded
		rc = decode_files_ranges_impl(d, ranges, nranges, d->d_pcm, rvalues, rinfo.data(), st, rerr.data(), keep ? &kept : nullptr, keep ? &kept0 : nullptr);
	}
	if(rc != FB200_OK) return rc;

	// ---- ReplayGain: the plan of k_rg_synth over every container the tool applies gain to
	if(applied) {
		RgsPlan plan;
		uint64_t draw = 0;  // the generator's position, running on over the containers of one invocation
		unsigned long long rg_items = 0;
		for(uint32_t i = 0; i < n; i++) {
			fb200_replaygain_synthesis_info &R = rginfo[i];
			if(info[i].status != FB200_FILE_OK || R.status != FB200_RGS_APPLIED) continue;
			const uint32_t C = info[i].channels;
			const uint64_t ns = info[i].samples, v0 = whole ? finfo[i].first_value : rinfo[i].first_value;
			const RgsParam P = rgs_param(info[i].bits_per_sample, R.scale, rg->limiter == FB200_RGS_LIMIT_HARD, rg->noise_shaping);
			R.first_draw = whole && !rg->per_file ? draw : 0;
			if(ns == 0) continue;
			if(rg->noise_shaping == 0) {
				plan.segs.push_back(RgsSeg{v0, ns * C, rg_items, P});
				rg_items += (ns * C + 1023) / 1024;
				continue;
			}
			const FilePlace *place;
			uint64_t nplace;
			if(whole) {
				const FileDecState &S = d->files_state0[d->files_pos[i]];
				place = kept.data() + S.cand0;
				nplace = S.ncand;
			}
			else {
				place = kept.data() + (kept0.empty() ? 0 : kept0[i]);
				nplace = kept.empty() ? 0 : rinfo[i].candidates;
			}
			const uint32_t b0 = (uint32_t)plan.blocks.size();
			const uint64_t delivered = rgs_blocks(place, nplace, v0, C, ns, plan.blocks);
			R.draws = 2ull * C * delivered;
			draw = R.first_draw + R.draws;
			for(uint32_t c = 0; c < C; c++)
				plan.chains.push_back(RgsChain{v0, ns, R.first_draw, C, c, b0, (uint32_t)plan.blocks.size() - b0, P});
		}
		if((rc = rgs_run(plan, rg->noise_shaping, d->d_pcm, st, &d->d_rgswork, &d->d_rgswork_cap, &d->launches)) != FB200_OK) return rc;
	}

	// ---- the pack plan: one segment per container with values, one PcmPackDev per container, the headers back to back
	std::vector<FileSeg> segs;
	std::vector<uint32_t> seg_cont;
	std::vector<PcmPackDev> conts;
	std::vector<uint8_t> blob;
	unsigned long long items = 0;
	for(uint32_t i = 0; i < n; i++) {
		fb200_pcm_decode_info &I = info[i];
		if(I.status != FB200_FILE_OK) continue;
		const PcmHeader &h = heads[i];
		uint64_t src;
		if(whole) {
			const fb200_file_decode_info &F = finfo[i];
			I.nframes = F.nframes; I.errors = F.errors; I.samples_missing = F.samples_missing; I.md5_state = F.md5_state;
			memcpy(I.md5, F.md5, 16);
			src = F.first_value;
		}
		else {
			I.nframes = rinfo[i].nframes; I.errors = rerr[i]; I.samples_missing = rinfo[i].samples_missing;
			src = rinfo[i].first_value;
		}
		// DecoderSession_finish_ok / _error: any decoder error (no -F), missing samples or an MD5 mismatch delete the file
		I.tool_ok = I.errors == 0 && I.samples_missing == 0 && I.md5_state != 2;
		const uint32_t B = h.container_bits / 8;
		PcmPackDev P;
		P.out = I.offset; P.blob = blob.size(); P.data = h.data_bytes; P.hlen = h.length; P.pad = (uint32_t)h.pad; P.bytes = B;
		P.big = opt->kind == FB200_PCM_AIFF || (opt->kind == FB200_PCM_AIFF_C && opt->subformat == FB200_PCM_SUB_AIFF_C_NONE);
		P.is_unsigned = opt->kind != FB200_PCM_AIFF && opt->kind != FB200_PCM_AIFF_C && I.bits_per_sample <= 8;
		P.shift = rg && rginfo[i].status == FB200_RGS_APPLIED ? 0 : h.container_bits - I.bits_per_sample;  // apply_gain's values are at the target width
		const uint64_t nv = I.samples * I.channels;
		if(nv) {
			segs.push_back(FileSeg{src, I.offset + h.length, nv, items});
			seg_cont.push_back((uint32_t)conts.size());
			items += (nv + kUnpackFilesItem - 1) / kUnpackFilesItem;
		}
		conts.push_back(P);
		blob.insert(blob.end(), h.bytes, h.bytes + h.length);
	}
	if(conts.empty()) {
		FB_CUDA(cudaStreamSynchronize(st));
		return FB200_OK;
	}
	const size_t o_segs = 0;
	const size_t o_cont = align16(o_segs + segs.size() * sizeof(FileSeg));
	const size_t o_sc = align16(o_cont + conts.size() * sizeof(PcmPackDev));
	const size_t o_blob = align16(o_sc + seg_cont.size() * sizeof(uint32_t));
	if((rc = grow((void **)&d->d_pwork, &d->d_pwork_cap, o_blob + blob.size() + 16)) != FB200_OK) return rc;
	if(!segs.empty()) {
		FB_CUDA(cudaMemcpyAsync(d->d_pwork + o_segs, segs.data(), segs.size() * sizeof(FileSeg), cudaMemcpyHostToDevice, st));
		FB_CUDA(cudaMemcpyAsync(d->d_pwork + o_sc, seg_cont.data(), seg_cont.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
	}
	FB_CUDA(cudaMemcpyAsync(d->d_pwork + o_cont, conts.data(), conts.size() * sizeof(PcmPackDev), cudaMemcpyHostToDevice, st));
	if(!blob.empty()) FB_CUDA(cudaMemcpyAsync(d->d_pwork + o_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
	uint8_t *d_out = out;
	if(host && (rc = grow((void **)&d->d_packed, &d->d_packed_cap, off + 16)) != FB200_OK) return rc;
	if(host) d_out = d->d_packed;
	launch_pcm_pack(d->d_pcm, reinterpret_cast<const FileSeg *>(d->d_pwork + o_segs), reinterpret_cast<const uint32_t *>(d->d_pwork + o_sc), (int)segs.size(),
	                items, reinterpret_cast<const PcmPackDev *>(d->d_pwork + o_cont), (int)conts.size(), d->d_pwork + o_blob, d_out, st);
	d->launches++;
	FB_CUDA(cudaGetLastError());
	if(host) FB_CUDA(cudaMemcpyAsync(out, d_out, off, cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	return FB200_OK;
}

int fb200_decode_pcm_files_host(fb200_decoder *d, const fb200_pcm_decode_options *opt, const fb200_sample_range *ranges, uint32_t nranges, uint8_t *out,
                                uint64_t out_capacity, uint64_t *total_bytes, fb200_pcm_decode_info *info)
{
	if(!d) return FB200_ERR_INVALID;
	return decode_pcm_files(d, opt, ranges, nranges, true, out, out_capacity, total_bytes, info, d->stream);
}

int fb200_decode_pcm_files_device(fb200_decoder *d, const fb200_pcm_decode_options *opt, const fb200_sample_range *ranges, uint32_t nranges,
                                  uint8_t *d_out, uint64_t out_capacity, uint64_t *total_bytes, fb200_pcm_decode_info *info, void *cuda_stream)
{
	return decode_pcm_files(d, opt, ranges, nranges, false, d_out, out_capacity, total_bytes, info, (cudaStream_t)cuda_stream);
}

int fb200_decode_pcm_files_replaygain_host(fb200_decoder *d, const fb200_pcm_decode_options *opt, const fb200_replaygain_synthesis *rg,
                                           const fb200_sample_range *ranges, uint32_t nranges, uint8_t *out, uint64_t out_capacity,
                                           uint64_t *total_bytes, fb200_pcm_decode_info *info, fb200_replaygain_synthesis_info *rginfo)
{
	if(!d || !rginfo) return FB200_ERR_INVALID;
	if(!rgs_spec_ok(rg)) return FB200_ERR_INVALID;
	return decode_pcm_files(d, opt, ranges, nranges, true, out, out_capacity, total_bytes, info, d->stream, rg, rginfo);
}

int fb200_decode_pcm_files_replaygain_device(fb200_decoder *d, const fb200_pcm_decode_options *opt, const fb200_replaygain_synthesis *rg,
                                             const fb200_sample_range *ranges, uint32_t nranges, uint8_t *d_out, uint64_t out_capacity,
                                             uint64_t *total_bytes, fb200_pcm_decode_info *info, fb200_replaygain_synthesis_info *rginfo,
                                             void *cuda_stream)
{
	if(!d || !rginfo) return FB200_ERR_INVALID;
	if(!rgs_spec_ok(rg)) return FB200_ERR_INVALID;
	return decode_pcm_files(d, opt, ranges, nranges, false, d_out, out_capacity, total_bytes, info, (cudaStream_t)cuda_stream, rg, rginfo);
}

}  // extern "C"

// ---- the encoder's verify (fb200_encoder_set_verify): the same walk / frame / CRC kernels, frames compared instead of stored
namespace fb200 {

static_assert(kVerifyCrcTabBytes == (size_t)kDecCrcTabEntries * sizeof(uint16_t), "k_dec_crc table size");

size_t verify_meta_bytes() { return sizeof(DecFrameMeta); }

void launch_verify_crc_tables(uint16_t *tab, cudaStream_t st) { k_dec_crc_tables<<<(kDecCrcLw * 5 + 255) / 256, 256, 0, st>>>(tab); }

void launch_verify_bounds(const unsigned long long *voff, unsigned long long nframes, unsigned long long cap, unsigned long long *vb, cudaStream_t st)
{
	k_verify_bounds<<<(unsigned)((nframes + 256) / 256), 256, 0, st>>>(voff, nframes, cap, vb);
}

void launch_verify_chunk(int channels, int bps, int sample_rate, int blocksize, const uint8_t *frames, const unsigned long long *vb, int nframes,
                         void *meta_v, DecVerdict *verdict, int32_t *pcm, const uint16_t *crc_tab, cudaStream_t st)
{
	DecK k;
	k.channels = channels; k.bps = bps; k.sample_rate = sample_rate; k.blocksize = blocksize;
	k.loose_end = 0;
	DecFrameMeta *meta = static_cast<DecFrameMeta *>(meta_v);
	const int chl = channels <= 1 ? 1 : channels <= 2 ? 2 : channels <= 4 ? 4 : 8;
	const int warps = (nframes + 32 / chl - 1) / (32 / chl);
	const unsigned long long cap = (unsigned long long)nframes * (unsigned long long)blocksize;
	k_dec_walk<<<(nframes + 127) / 128, 128, 0, st>>>(k, frames, vb, vb + 1, nframes, meta);
	k_dec_frames<12, true><<<(warps + 3) / 4, 128, 0, st>>>(k, frames, vb, vb + 1, nframes, meta, pcm, cap, nullptr, nullptr, verdict);
	k_dec_frames<32, true><<<(warps + 3) / 4, 128, 0, st>>>(k, frames, vb, vb + 1, nframes, meta, pcm, cap, nullptr, nullptr, verdict);
	k_dec_crc<<<(nframes + 3) / 4, 128, 0, st>>>(frames, vb, nframes, meta, nullptr, nullptr, crc_tab);
}

void launch_verify_files(const void *meta, const DecVerdict *verdict, const FileFrames *files, const FileSeg *segs, int nfiles, uint32_t channels,
                         uint32_t blocksize, uint32_t sample_rate, fb200_file_verify_info *info, cudaStream_t st)
{
	k_verify_files<<<(nfiles + 3) / 4, 128, 0, st>>>(static_cast<const DecFrameMeta *>(meta), verdict, files, segs, nfiles, channels, blocksize, sample_rate,
	                                                 info);
}

// ---- fb200_reencode_flac_files_* (reencode.cu): the resident batch as an encoder's input
bool decoder_files(const fb200_decoder *d, uint32_t *nfiles, int *device)
{
	if(!d || !d->files_ready) return false;
	*nfiles = (uint32_t)d->files_info.size();
	*device = d->device;
	return true;
}

const fb200_file_decode_info &decoder_file_info(const fb200_decoder *d, uint32_t f) { return d->files_info[f]; }
const uint8_t *decoder_file_md5(const fb200_decoder *d, uint32_t f) { return d->files_md5[f].data(); }
uint32_t decoder_file_mask(const fb200_decoder *d, uint32_t f) { return d->files_mask[f]; }

int decoder_file_metadata(fb200_decoder *d, uint32_t f, std::vector<uint8_t> *bytes)
{
	bytes->resize((size_t)(d->files_audio[f] - d->files_start[f]));
	if(!bytes->empty()) FB_CUDA(cudaMemcpy(bytes->data(), d->d_fdata + d->files_start[f], bytes->size(), cudaMemcpyDeviceToHost));
	return FB200_OK;
}

// The whole-file path of decode_files_impl for the listed files only. A group runs over the candidates from its first listed
// file's to its last listed file's; a file between them that is not listed is decoded too but places nothing (end_sample 0).
int decoder_decode_into(fb200_decoder *d, const uint32_t *files, const uint64_t *first_value, uint32_t n, int32_t *pcm, unsigned long long values,
                        const FileSeg *d_segs, int nsegs, cudaStream_t st, FilePlace *keep_place, uint32_t *keep_bytes)
{
	const FilesIndexLayout L(d->files_ncand, d->files_state0.size());
	const unsigned long long *d_begins = reinterpret_cast<const unsigned long long *>(d->d_findex + L.begins);
	const unsigned long long *d_ends = reinterpret_cast<const unsigned long long *>(d->d_findex + L.ends);
	const FileDecCand *d_cands = reinterpret_cast<const FileDecCand *>(d->d_findex + L.cands);
	FileDecState *d_states = reinterpret_cast<FileDecState *>(d->d_findex + L.states);
	std::vector<FileDecState> states(d->files_state0);
	for(FileDecState &S : states) S.end_sample = 0;
	for(uint32_t i = 0; i < n; i++) {
		FileDecState &S = states[d->files_pos[files[i]]];
		S.first_value = first_value[i];
		S.end_sample = d->files_info[files[i]].samples;
	}
	std::vector<std::pair<uint32_t, uint32_t>> span(d->files_groups.size(), std::make_pair(~0u, 0u));  // listed positions [first, last]
	for(uint32_t i = 0; i < n; i++) {
		const uint32_t pos = d->files_pos[files[i]];
		for(size_t g = 0; g < d->files_groups.size(); g++) {
			const auto &G = d->files_groups[g];
			if(pos < G.pos0 || pos >= G.pos0 + G.nfiles) continue;
			span[g].first = std::min(span[g].first, pos);
			span[g].second = std::max(span[g].second, pos);
		}
	}
	uint64_t chunk_max = 1, slot_values_max = 0;
	for(size_t g = 0; g < d->files_groups.size(); g++) {
		if(span[g].first == ~0u) continue;
		const auto &G = d->files_groups[g];
		const uint64_t c = files_chunk(d, G);
		chunk_max = std::max(chunk_max, c);
		slot_values_max = std::max(slot_values_max, c * G.max_bs * G.channels);
	}
	const size_t o_stat = 0;
	const size_t o_bytes = align16(o_stat + chunk_max * sizeof(uint32_t));
	const size_t o_place = align16(o_bytes + chunk_max * sizeof(uint32_t));
	int rc;
	if((rc = grow((void **)&d->d_fwork, &d->d_fwork_cap, o_place + chunk_max * sizeof(FilePlace))) != FB200_OK) return rc;
	if((rc = grow((void **)&d->d_fslots, &d->d_fslots_cap, (size_t)slot_values_max * sizeof(int32_t) + 16)) != FB200_OK) return rc;
	uint32_t *d_stat = reinterpret_cast<uint32_t *>(d->d_fwork + o_stat);
	uint32_t *d_bytes = reinterpret_cast<uint32_t *>(d->d_fwork + o_bytes);
	FilePlace *d_place = reinterpret_cast<FilePlace *>(d->d_fwork + o_place);
	if(!states.empty()) FB_CUDA(cudaMemcpyAsync(d_states, states.data(), states.size() * sizeof(FileDecState), cudaMemcpyHostToDevice, st));
	FB_CUDA(cudaMemsetAsync(pcm, 0, (size_t)values * sizeof(int32_t), st));
	for(size_t g = 0; g < d->files_groups.size(); g++) {
		if(span[g].first == ~0u) continue;
		const uint32_t lo = span[g].first, hi = span[g].second;
		const FilesRun R{&d->files_groups[g], states[lo].cand0, states[hi].cand0 + states[hi].ncand - states[lo].cand0, states.data() + lo, d_states + lo,
		                 hi - lo + 1, d_begins, d_ends, d_cands};
		const bool keep = keep_place != nullptr;
		if((rc = decode_files_run(d, R, d_stat, keep ? keep_bytes : d_bytes, keep ? keep_place : d_place, pcm, st, d_segs, nsegs, keep)) != FB200_OK) return rc;
	}
	FB_CUDA(cudaGetLastError());
	return FB200_OK;
}

int decoder_decode_ranges_into(fb200_decoder *d, const fb200_sample_range *ranges, const uint64_t *first_value, uint32_t n, int32_t *pcm,
                               unsigned long long values, const FileSeg *d_segs, int nsegs, cudaStream_t st, uint32_t *errors, uint64_t *missing)
{
	std::vector<fb200_range_decode_info> info(n);
	for(uint32_t i = 0; i < n; i++) {
		const fb200_file_decode_info &I = d->files_info[ranges[i].file];
		memset(&info[i], 0, sizeof info[i]);
		info[i].status = FB200_FILE_OK;
		info[i].channels = I.channels;
		info[i].bits_per_sample = I.bits_per_sample;
		info[i].first_value = first_value[i];
		info[i].values = ranges[i].samples * I.channels;
	}
	const int rc = decode_files_ranges_impl(d, ranges, n, pcm, values, info.data(), st, errors, nullptr, nullptr, d_segs, nsegs);
	if(rc != FB200_OK) return rc;
	for(uint32_t i = 0; i < n; i++) missing[i] = info[i].samples_missing;
	return FB200_OK;
}

DecoderFilesView decoder_files_view(const fb200_decoder *d)
{
	const FilesIndexLayout L(d->files_ncand, d->files_state0.size());
	DecoderFilesView v;
	v.data = d->d_fdata;
	v.begins = reinterpret_cast<const unsigned long long *>(d->d_findex + L.begins);
	v.cands = reinterpret_cast<const FileDecCand *>(d->d_findex + L.cands);
	v.states = reinterpret_cast<const FileDecState *>(d->d_findex + L.states);
	v.ncand = d->files_ncand;
	return v;
}

DecoderFileSpan decoder_file_span(const fb200_decoder *d, uint32_t f)
{
	const FileDecState &S = d->files_state0[d->files_pos[f]];
	return DecoderFileSpan{d->files_start[f], d->files_audio[f], d->files_end[f], S.cand0, S.ncand, d->files_pos[f]};
}

void decoder_count_launches(fb200_decoder *d, uint64_t n) { d->launches += n; }

int decoder_decode_verdicts(fb200_decoder *d, const uint32_t *files, uint32_t n, cudaStream_t st, uint32_t *errors, uint64_t *missing)
{
	const FilesIndexLayout L(d->files_ncand, d->files_state0.size());
	std::vector<FileDecState> states(d->files_state0.size());
	if(!states.empty()) FB_CUDA(cudaMemcpyAsync(states.data(), d->d_findex + L.states, states.size() * sizeof(FileDecState), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	for(uint32_t i = 0; i < n; i++) {
		const FileDecState &S = states[d->files_pos[files[i]]];
		errors[i] = S.errors;
		missing[i] = d->files_info[files[i]].samples - S.covered;
	}
	return FB200_OK;
}

}  // namespace fb200
