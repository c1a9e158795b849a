// decoder.cu -- host side of the FLAC batch frame decoder + its C ABI (include/flac_b200.h).
#include <string.h>

#include <algorithm>
#include <vector>

#include "decode_kernels.cuh"

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
};

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
static int decode_ranges(fb200_decoder *d, const uint8_t *d_frames, const unsigned long long *begins, const unsigned long long *ends, uint32_t nframes,
                         int32_t *d_pcm, uint64_t pcm_capacity_samples, uint32_t *d_frame_status, uint32_t *d_frame_bytes, int loose, cudaStream_t st,
                         uint32_t subinfo_base = 0)
{
	const int ch = (int)d->cfg.channels;
	const int chl = ch <= 1 ? 1 : ch <= 2 ? 2 : ch <= 4 ? 4 : 8;
	const int fpw = 32 / chl;
	DecK k = d->k;
	k.loose_end = loose;
	// subframe records of frame i of this call go to slot subinfo_base + i (a chunked caller sized the array for all its frames)
	if(d->want_subinfo && (size_t)(subinfo_base + nframes) * ch > d->d_subinfo_cap) {
		if(subinfo_base) { set_error("internal: subframe info array too small"); return FB200_ERR_INVALID; }
		cudaFree(d->d_subinfo); d->d_subinfo = nullptr; d->d_subinfo_cap = 0;
		FB_CUDA(cudaMalloc(&d->d_subinfo, (size_t)nframes * ch * sizeof(DecSubframeInfo)));
		d->d_subinfo_cap = (size_t)nframes * ch;
	}
	uint32_t done = 0;
	while(done < nframes) {
		const int nf = (int)((nframes - done) < d->max_frames ? (nframes - done) : d->max_frames);
		// frame `done + i` decodes to sample offset (done + i) * blocksize
		const unsigned long long used = (unsigned long long)done * d->cfg.blocksize;
		const unsigned long long cap_left = pcm_capacity_samples > used ? pcm_capacity_samples - used : 0ull;  // frames that do not fit are reported (DEC_LENGTH), never written
		dprof_mark(d, -1, st);
		k_dec_walk<<<(nf + 127) / 128, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta);
		dprof_mark(d, FB200_DPROF_WALK, st);
		const int warps = (nf + fpw - 1) / fpw;
		// predictors of at most 12 taps (every preset) and the rest (-l 13..32): two instantiations, each taking its frames
		k_dec_frames<12><<<(warps + 3) / 4, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta, d_pcm + (size_t)done * d->cfg.blocksize * ch, cap_left,
		                                                 d_frame_status ? d_frame_status + done : nullptr,
		                                                 d->want_subinfo ? d->d_subinfo + (size_t)(subinfo_base + done) * ch : nullptr);
		k_dec_frames<32><<<(warps + 3) / 4, 128, 0, st>>>(k, d_frames, begins + done, ends + done, nf, d->d_meta, d_pcm + (size_t)done * d->cfg.blocksize * ch, cap_left,
		                                                 d_frame_status ? d_frame_status + done : nullptr,
		                                                 d->want_subinfo ? d->d_subinfo + (size_t)(subinfo_base + done) * ch : nullptr);
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
	const int rc = decode_ranges(d, d_frames, offs, offs + 1, nframes, d_pcm, pcm_capacity_samples, d_frame_status, nullptr, 0, st);
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
		const int rc = decode_ranges(d, d->d_frames, offs + f0, offs + f0 + 1, f1 - f0, d->d_pcm + (size_t)s0 * ch, need_samples - s0, d->d_status + f0, nullptr, 0,
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
	const int rc = decode_ranges(d, d->d_stream, d->d_offsets, d->d_offsets + nframes, nframes, d->d_pcm, need_samples, d->d_status, d->d_fbytes, 1, d->stream);
	if(rc != FB200_OK) return rc;
	FB_CUDA(cudaMemcpyAsync(pcm, d->d_pcm, (size_t)cap * d->cfg.channels * sizeof(int32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaMemcpyAsync(frame_status, d->d_status, (size_t)nframes * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaMemcpyAsync(frame_bytes, d->d_fbytes, (size_t)nframes * sizeof(uint32_t), cudaMemcpyDeviceToHost, d->stream));
	FB_CUDA(cudaStreamSynchronize(d->stream));
	d->h_status.assign(frame_status, frame_status + nframes);
	return FB200_OK;
}

}  // extern "C"
