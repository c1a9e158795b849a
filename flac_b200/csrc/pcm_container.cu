// pcm_container.cu -- fb200_pcm_files_probe and fb200_encode_pcm_files_*: WAV / RF64 / Wave64 / AIFF / AIFF-C files in, the
// .flac files the flac tool writes out. The host parses each container as the tool does (encode.c:192-803) and builds the
// metadata list EncoderSession_init_encoder makes for a non-FLAC input; k_pcm_unpack restates format_input (encode.c:2352-2505)
// over the whole batch in one launch; the rest is fb200_encode_flac_files_*'s machinery.
// The other direction (fb200_decode_pcm_files_*, decoder.cu; fb200_pcm_header): the header write_iff_headers writes
// (decode.c:718-989), built on the host, and k_pcm_pack, which restates write_callback (decode.c:1245-1632) in one launch.
#include <stdarg.h>
#include <string.h>

#include "fb200_internal.h"
#include "flac_metadata.h"

namespace fb200 {

// ---- device: k_pcm_unpack

// One CTA per work item of kUnpackFilesItem values of one segment (the segments and items of k_unpack_files). Each thread widens
// runs of 4 values: the aligned 32-bit words under the run's bytes are loaded (only words that hold a byte of the input, so a
// file's tail never reads past the batch) and funnel-shifted into place, then each value is taken out, byte-swapped for big-endian
// data, offset for unsigned data, checked and shifted down as format_input does. The lowest failing element of the back-to-back
// numbering (file, then sample, then channel) is kept with one atomicMin per thread that saw one.
template <int B>
__device__ __forceinline__ void pcm_run(const uint32_t *__restrict__ words, unsigned long long lim, unsigned long long byte, int n, const PcmFileDev &F,
                                        int32_t *__restrict__ dst, unsigned long long elem, unsigned long long *bad)
{
	const unsigned long long w0 = byte >> 2;
	const uint32_t sh = (uint32_t)(byte & 3) * 8;
	uint32_t raw[B + 1], u[B + 1];
#pragma unroll
	for(int j = 0; j <= B; j++) raw[j] = (w0 + j) * 4 < lim ? __ldg(words + w0 + j) : 0u;
#pragma unroll
	for(int j = 0; j < B; j++) u[j] = __funnelshift_r(raw[j], raw[j + 1], sh);
	u[B] = 0;
	const uint32_t mask = (1u << F.shift) - 1u;
#pragma unroll
	for(int s = 0; s < 4; s++) {
		if(s >= n) break;
		const int off = s * B;
		const unsigned long long x = ((unsigned long long)u[(off >> 2) + 1] << 32) | u[off >> 2];
		uint32_t v = (uint32_t)(x >> ((off & 3) * 8));
		if(B < 4) v &= (1u << (8 * B)) - 1u;
		if(F.big && B > 1) v = __byte_perm(v, 0, 0x0123) >> (32 - 8 * B);
		int32_t val = F.is_unsigned ? (int32_t)(v - (1u << (8 * B - 1))) : (int32_t)(v << (32 - 8 * B)) >> (32 - 8 * B);
		if((uint32_t)val & mask) *bad = min(*bad, elem + s);
		dst[s] = val >> F.shift;
	}
}

__global__ void __launch_bounds__(256) k_pcm_unpack(const uint8_t *__restrict__ in, unsigned long long in_bytes, const PcmFileDev *__restrict__ files,
                                                   const FileSeg *__restrict__ segs, int nsegs, int32_t *__restrict__ pcm,
                                                   unsigned long long *__restrict__ first_bad)
{
	const unsigned long long item = blockIdx.x;
	int lo = 0, hi = nsegs - 1;  // the last segment whose first item is <= item (empty segments own no item)
	while(lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if(segs[mid].item0 <= item) lo = mid;
		else hi = mid - 1;
	}
	const FileSeg S = segs[lo];
	const PcmFileDev F = files[lo >> 1];
	const uint32_t mis = (uint32_t)((uintptr_t)in & 3u);
	const uint32_t *words = reinterpret_cast<const uint32_t *>(in - mis);
	const unsigned long long lim = in_bytes + mis;  // byte offsets from `words`: the input is [mis, lim)
	const unsigned long long base = (item - S.item0) * kUnpackFilesItem;
	unsigned long long bad = ~0ull;
	for(int k = 0; k < kUnpackFilesItem / 1024; k++) {
		const unsigned long long e0 = base + 4ull * (threadIdx.x + 256u * k);
		if(e0 >= S.n) break;
		const int n = (int)min(4ull, S.n - e0);
		const unsigned long long elem = S.src + e0;  // in the back-to-back numbering of every file's values
		const unsigned long long byte = mis + F.data + (elem - F.elem0) * F.bytes;
		int32_t *dst = pcm + S.dst + e0;
		switch(F.bytes) {
		case 1: pcm_run<1>(words, lim, byte, n, F, dst, elem, &bad); break;
		case 2: pcm_run<2>(words, lim, byte, n, F, dst, elem, &bad); break;
		case 3: pcm_run<3>(words, lim, byte, n, F, dst, elem, &bad); break;
		default: pcm_run<4>(words, lim, byte, n, F, dst, elem, &bad); break;
		}
	}
	if(bad != ~0ull) atomicMin(first_bad, bad);
}

void launch_pcm_unpack(const uint8_t *in, unsigned long long in_bytes, const PcmFileDev *files, const FileSeg *segs, int nsegs, unsigned long long items,
                       int32_t *pcm, unsigned long long *first_bad, cudaStream_t st)
{
	if(items) k_pcm_unpack<<<(unsigned)items, 256, 0, st>>>(in, in_bytes, files, segs, nsegs, pcm, first_bad);
}

// ---- device: k_pcm_pack

// The mirror of k_pcm_unpack: write_callback (decode.c:1245-1632) over every container of a fb200_decode_pcm_files_* call. One
// CTA per work item of kUnpackFilesItem values of one container's data region. Each thread reads runs of 4 values (one 16-byte
// load when the run is aligned), shifts each left into its container, offsets unsigned 8-bit data, and stores its 1-4 bytes in
// either byte order into shared memory at the destination's byte phase. The CTA then writes the aligned 16-byte chunks inside its
// byte range with 16-byte stores and only its own bytes of the two ragged chunks with byte stores, so items that share a chunk
// (neighbouring items, a header, a container starting at any byte) never race. The last ncont CTAs each copy one container's
// header from the blob and write its pad bytes.
__global__ void __launch_bounds__(256) k_pcm_pack(const int32_t *__restrict__ pcm, const FileSeg *__restrict__ segs, const uint32_t *__restrict__ seg_cont,
                                                 int nsegs, unsigned long long items, const PcmPackDev *__restrict__ conts, const uint8_t *__restrict__ blob,
                                                 uint8_t *__restrict__ out)
{
	__shared__ __align__(16) uint8_t stage[kUnpackFilesItem * 4 + 16];
	const unsigned long long item = blockIdx.x;
	if(item >= items) {
		const PcmPackDev P = conts[item - items];
		for(uint32_t i = threadIdx.x; i < P.hlen; i += 256) out[P.out + i] = blob[P.blob + i];
		for(uint32_t i = threadIdx.x; i < P.pad; i += 256) out[P.out + P.hlen + P.data + i] = 0;
		return;
	}
	int lo = 0, hi = nsegs - 1;  // the last segment whose first item is <= item (every segment owns an item)
	while(lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if(segs[mid].item0 <= item) lo = mid;
		else hi = mid - 1;
	}
	const FileSeg S = segs[lo];
	const PcmPackDev P = conts[seg_cont[lo]];
	const unsigned long long base = (item - S.item0) * kUnpackFilesItem;
	const int n = (int)min((unsigned long long)kUnpackFilesItem, S.n - base);
	const uint32_t B = P.bytes;
	const uintptr_t dst = (uintptr_t)(out + S.dst + base * B);
	const uint32_t phase = (uint32_t)(dst & 15u);
	const int32_t *src = pcm + S.src + base;
	const bool vec = ((uintptr_t)src & 15u) == 0;
	for(int k = 0; k < kUnpackFilesItem / 1024; k++) {
		const int j = 4 * (threadIdx.x + 256 * k);
		if(j >= n) break;
		int32_t v[4];
		if(vec && j + 4 <= n) {
			const int4 q = __ldg(reinterpret_cast<const int4 *>(src + j));
			v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
		}
		else {
#pragma unroll
			for(int i = 0; i < 4; i++) v[i] = j + i < n ? __ldg(src + j + i) : 0;
		}
		const int m = min(4, n - j);
#pragma unroll
		for(int i = 0; i < 4; i++) {
			if(i >= m) break;
			uint32_t u = (uint32_t)v[i] << P.shift;
			if(P.is_unsigned) u += 0x80u;
			uint8_t *s = stage + phase + (uint32_t)(j + i) * B;
			for(uint32_t b = 0; b < B; b++) s[b] = (uint8_t)(u >> (8 * (P.big ? B - 1 - b : b)));
		}
	}
	__syncthreads();
	const uint32_t end = phase + (uint32_t)n * B;  // staged bytes [phase, end) go to [dst - phase + phase, ...)
	uint8_t *a0 = reinterpret_cast<uint8_t *>(dst - phase);
	for(uint32_t c = threadIdx.x; c < (end + 15) / 16; c += 256) {
		const uint32_t c0 = 16 * c, c1 = c0 + 16;
		if(c0 >= phase && c1 <= end) *reinterpret_cast<uint4 *>(a0 + c0) = *reinterpret_cast<const uint4 *>(stage + c0);
		else
			for(uint32_t b = max(c0, phase); b < min(c1, end); b++) a0[b] = stage[b];
	}
}

void launch_pcm_pack(const int32_t *pcm, const FileSeg *segs, const uint32_t *seg_cont, int nsegs, unsigned long long items, const PcmPackDev *conts,
                     int ncont, const uint8_t *blob, uint8_t *out, cudaStream_t st)
{
	if(items + ncont) k_pcm_pack<<<(unsigned)(items + ncont), 256, 0, st>>>(pcm, segs, seg_cont, nsegs, items, conts, blob, out);
}

// ---- host: the header of fb200_decode_pcm_files_* and fb200_pcm_header

namespace {

void put_le(uint8_t *&p, uint64_t v, int n)
{
	for(int i = 0; i < n; i++) *p++ = (uint8_t)(v >> (8 * i));
}

void put_be(uint8_t *&p, uint64_t v, int n)
{
	for(int i = 0; i < n; i++) *p++ = (uint8_t)(v >> (8 * (n - 1 - i)));
}

void put_id(uint8_t *&p, const char *s, int n)
{
	memcpy(p, s, n);
	p += n;
}

// write_sane_extended (decode.c:1185-1220)
void put_sane_extended(uint8_t *&p, uint32_t val)
{
	if(val == 0) {
		put_be(p, 0, 2); put_be(p, 0, 4); put_be(p, 0, 4);
		return;
	}
	uint32_t shift = 0;
	while((val >> (31 - shift)) == 0) shift++;
	val <<= shift;
	put_be(p, 63 - (shift + 32) + 0x3FFF, 2);
	put_be(p, val, 4);
	put_be(p, 0, 4);
}

}  // namespace

bool pcm_decode_options_ok(const fb200_pcm_decode_options *opt)
{
	if(!opt) { set_error("options are NULL"); return false; }
	const uint32_t k = opt->kind, s = opt->subformat;
	bool ok;
	if(k == FB200_PCM_WAVE) ok = s == FB200_PCM_SUB_AUTO || s == FB200_PCM_SUB_WAVE_PCM || s == FB200_PCM_SUB_WAVE_EXTENSIBLE;
	else if(k == FB200_PCM_AIFF_C) ok = s == FB200_PCM_SUB_AIFF_C_NONE || s == FB200_PCM_SUB_AIFF_C_SOWT;
	else ok = (k == FB200_PCM_RF64 || k == FB200_PCM_WAVE64 || k == FB200_PCM_AIFF) && s == FB200_PCM_SUB_AUTO;
	if(!ok) set_error("kind %u with subformat %u is not an output format of the flac tool", k, s);
	return ok;
}

// write_iff_headers (decode.c:718-989) without foreign metadata, with the fmt sizes of :991-1036, the fmt body of :1038-1078 and
// the COMM chunk of :1080-1128; the channel mask as metadata_callback (:1820) and the defaults (:429-454) leave it.
void pcm_header_build(const fb200_pcm_decode_options &opt, uint32_t channels, uint32_t bps, uint32_t rate, uint32_t tag_mask, uint64_t samples, PcmHeader *h)
{
	static const uint32_t kDefaultMask[9] = {0, 0x0004, 0x0003, 0x0007, 0x0033, 0x0607, 0x060f, 0x070f, 0x063f};
	memset(h, 0, sizeof *h);
	const uint32_t kind = opt.kind, sub = opt.subformat;
	uint32_t mask = opt.channel_map_none ? 0 : tag_mask;
	if(!opt.channel_map_none && mask == 0 && channels <= 8) mask = kDefaultMask[channels];
	const bool wave = kind == FB200_PCM_WAVE || kind == FB200_PCM_WAVE64 || kind == FB200_PCM_RF64;
	const bool ext = sub == FB200_PCM_SUB_WAVE_EXTENSIBLE ||
	                 (wave && sub != FB200_PCM_SUB_WAVE_PCM && ((mask != 0 && mask != 0x0004 && mask != 0x0003) || (bps != 8 && bps != 16) || channels > 2));
	const uint32_t B = (bps + 7) / 8;
	const uint64_t data = samples * channels * B;
	const uint64_t aligned = kind == FB200_PCM_WAVE64 ? (data + 7) & ~7ull : (data + 1) & ~1ull;
	const uint64_t fmt_field = ext ? 16 + 2 + 22 : 16;  // calculate_riff_wave_fmt_chunk_size_field
	const uint64_t w64_fmt_field = 16 + 8 + fmt_field;  // calculate_wave64_fmt_chunk_size_field
	uint64_t iff;
	if(samples == 0) iff = 0;
	else if(kind == FB200_PCM_WAVE || kind == FB200_PCM_RF64) iff = 4 + (kind == FB200_PCM_RF64 ? 36 : 0) + (8 + fmt_field) + 8 + aligned;
	else if(kind == FB200_PCM_WAVE64) iff = 16 + 8 + 16 + ((w64_fmt_field + 7) & ~7ull) + 16 + 8 + aligned;
	else if(kind == FB200_PCM_AIFF) iff = 46 + aligned;
	else iff = 16 + aligned + 36;
	h->container_bits = 8 * B;
	h->extensible = ext;
	h->mask = mask;
	h->data_bytes = data;
	h->pad = kind == FB200_PCM_WAVE64 ? (8 - (data & 7)) & 7 : data & 1;
	if(kind != FB200_PCM_WAVE64 && kind != FB200_PCM_RF64 && iff >= 0xFFFFFFF4ull) {
		h->too_big = true;
		return;
	}
	uint8_t *p = h->bytes;
	if(wave) {
		if(kind == FB200_PCM_WAVE) { put_id(p, "RIFF", 4); put_le(p, (uint32_t)iff, 4); put_id(p, "WAVE", 4); }
		else if(kind == FB200_PCM_WAVE64) {
			put_id(p, "\x72\x69\x66\x66\x2E\x91\xCF\x11\xA5\xD6\x28\xDB\x04\xC1\x00\x00", 16);
			put_le(p, iff, 8);
			put_id(p, "\x77\x61\x76\x65\xF3\xAC\xD3\x11\x8C\xD1\x00\xC0\x4F\x8E\xDB\x8A", 16);
		}
		else {
			put_id(p, "RF64", 4); put_le(p, 0xffffffffu, 4); put_id(p, "WAVE", 4);
			put_id(p, "ds64", 4); put_le(p, 28, 4); put_le(p, iff, 8); put_le(p, data, 8); put_le(p, samples, 8); put_le(p, 0, 4);
		}
		if(kind != FB200_PCM_WAVE64) { put_id(p, "fmt ", 4); put_le(p, fmt_field, 4); }
		else { put_id(p, "\x66\x6D\x74\x20\xF3\xAC\xD3\x11\x8C\xD1\x00\xC0\x4F\x8E\xDB\x8A", 16); put_le(p, w64_fmt_field, 8); }
		put_le(p, ext ? 65534 : 1, 2);
		put_le(p, channels, 2);
		put_le(p, rate, 4);
		put_le(p, (uint32_t)(rate * channels * B), 4);  // 32-bit arithmetic, as the tool's
		put_le(p, channels * B, 2);
		put_le(p, 8 * B, 2);
		if(ext) {
			put_le(p, 22, 2);
			put_le(p, bps, 2);
			put_le(p, mask, 4);
			put_id(p, "\x01\x00\x00\x00\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71", 16);
		}
		if(kind == FB200_PCM_WAVE64)
			while((p - h->bytes) % 8) *p++ = 0;
		if(kind != FB200_PCM_WAVE64) { put_id(p, "data", 4); put_le(p, kind == FB200_PCM_RF64 ? 0xffffffffu : (uint32_t)data, 4); }
		else { put_id(p, "\x64\x61\x74\x61\xF3\xAC\xD3\x11\x8C\xD1\x00\xC0\x4F\x8E\xDB\x8A", 16); put_le(p, 16 + 8 + data, 8); }
	}
	else {
		const uint32_t comm_length = kind == FB200_PCM_AIFF ? 30 : 36;
		put_id(p, "FORM", 4); put_be(p, (uint32_t)iff, 4); put_id(p, kind == FB200_PCM_AIFF ? "AIFF" : "AIFC", 4);
		put_id(p, "COMM", 4);
		put_be(p, comm_length - 12, 4);
		put_be(p, channels, 2);
		put_be(p, (uint32_t)samples, 4);
		put_be(p, bps, 2);
		put_sane_extended(p, rate);
		if(kind == FB200_PCM_AIFF_C) {
			put_id(p, sub == FB200_PCM_SUB_AIFF_C_NONE ? "NONE" : "sowt", 4);
			for(uint32_t i = 34; i < comm_length; i++) *p++ = 0;
		}
		put_id(p, "SSND", 4);
		put_be(p, (uint32_t)data + 8, 4);
		put_be(p, 0, 4);
		put_be(p, 0, 4);
	}
	h->length = (uint32_t)(p - h->bytes);
}

// ---- host: the container probe

namespace {

struct Reader {
	const uint8_t *p;
	uint64_t n, pos;
	const char *err = nullptr;
	bool take(uint64_t k, const uint8_t **out)
	{
		if(pos > n || n - pos < k) { err = "unexpected EOF"; return false; }
		*out = p + pos;
		pos += k;
		return true;
	}
	bool u16(bool big, uint32_t *v)
	{
		const uint8_t *b;
		if(!take(2, &b)) return false;
		*v = big ? ((uint32_t)b[0] << 8 | b[1]) : ((uint32_t)b[1] << 8 | b[0]);
		return true;
	}
	bool u32(bool big, uint32_t *v)
	{
		const uint8_t *b;
		if(!take(4, &b)) return false;
		*v = big ? ((uint32_t)b[0] << 24 | (uint32_t)b[1] << 16 | (uint32_t)b[2] << 8 | b[3])
		         : ((uint32_t)b[3] << 24 | (uint32_t)b[2] << 16 | (uint32_t)b[1] << 8 | b[0]);
		return true;
	}
	bool u64le(uint64_t *v)
	{
		uint32_t lo, hi;
		if(!u32(false, &lo) || !u32(false, &hi)) return false;
		*v = (uint64_t)hi << 32 | lo;
		return true;
	}
	// fskip_ahead (encode.c:2935): a seek on a regular file, which succeeds past the end; fails only beyond the largest off_t
	bool skip(uint64_t k)
	{
		if(k > (uint64_t)INT64_MAX) { err = "chunk too large to skip"; return false; }
		pos = k > UINT64_MAX - pos ? UINT64_MAX : pos + k;
		return true;
	}
};

const uint8_t kW64Guid[12] = {0xF3, 0xAC, 0xD3, 0x11, 0x8C, 0xD1, 0x00, 0xC0, 0x4F, 0x8E, 0xDB, 0x8A};  // the tail every Wave64 GUID id shares here

struct Probed {
	uint32_t channels = 0, bps = 0, shift = 0, rate = 0, channel_mask = 0;
	bool is_unsigned = false, big = false;
	uint64_t data_bytes = 0, data_pos = 0;
	bool has_data = false;
};

// get_sample_info_wave (encode.c:192-576) for WAVE, RF64 and Wave64; nullptr or the tool's error
const char *probe_wave(Reader &r, uint32_t kind, Probed *o)
{
	const bool w64 = kind == FB200_PCM_WAVE64;
	bool got_fmt = false, got_data = false, got_ds64 = false;
	uint64_t ds64_data = 0;
	r.pos = w64 ? 40 : 12;
	while(!got_data) {
		const uint32_t idlen = w64 ? 16 : 4;
		if(r.pos >= r.n) break;
		if(r.n - r.pos < idlen) return "incomplete chunk identifier";
		const uint8_t *id = r.p + r.pos;
		r.pos += idlen;
		const bool guid_ok = !w64 || !memcmp(id + 4, kW64Guid, 12);
		if(kind == FB200_PCM_RF64 && !memcmp(id, "ds64", 4)) {
			uint32_t sz, x;
			if(got_ds64) return "file has multiple 'ds64' chunks";
			if(got_fmt) return "'ds64' chunk appears after 'fmt ' or 'data' chunk";
			if(!r.u32(false, &sz)) return r.err;
			if(sz < 28) return "non-standard 'ds64' chunk";
			if(sz & 1) sz++;
			if(!r.u32(false, &x) || !r.u32(false, &x) || !r.u64le(&ds64_data)) return r.err;
			if(!r.skip(sz - 16)) return r.err;
			got_ds64 = true;
		}
		else if(!memcmp(id, "fmt ", 4) && guid_ok) {
			uint32_t sz, hi, tag, ch, rate, x, ba, bps;
			if(got_fmt) return "file has multiple 'fmt ' chunks";
			if(!r.u32(false, &sz)) return r.err;
			if(w64) {
				if(!r.u32(false, &hi)) return r.err;
				if(hi) return "freakishly large Wave64 'fmt ' chunk";
				if(sz < 24) return "freakishly small Wave64 'fmt ' chunk";
				sz -= 24;
			}
			if(sz < 16 || sz > UINT32_MAX - 8) return "non-standard 'fmt ' chunk";
			if(!w64) sz += sz & 1;
			else sz = (sz + 7) & ~7u;
			if(!r.u16(false, &tag)) return r.err;
			if(tag != 1 && tag != 65534) return "unsupported format type (not PCM or WAVE_FORMAT_EXTENSIBLE)";
			if(!r.u16(false, &ch) || !r.u32(false, &rate) || !r.u32(false, &x) || !r.u16(false, &ba) || !r.u16(false, &bps)) return r.err;
			o->is_unsigned = bps <= 8;
			if(tag == 1) {
				if(bps != 8 && bps != 16 && bps != 24 && bps != 32) return "legacy WAVE file has format type 1 but bits-per-sample not 8/16/24/32";
				if((bps + 7) / 8 * ch != ba) return "legacy WAVE file has a block alignment that disagrees with bits-per-sample and channels";
				if(ch > 2) return "WAVE has >2 channels but is not WAVE_FORMAT_EXTENSIBLE; cannot assign channels";
				sz -= 16;
			}
			else {
				uint32_t cb, valid, guid;
				if(sz < 40) return "invalid WAVEFORMATEXTENSIBLE chunk size";
				if(!r.u16(false, &cb)) return r.err;
				if(cb < 22) return "invalid WAVEFORMATEXTENSIBLE chunk with cbSize < 22";
				if(!r.u16(false, &valid)) return r.err;
				if(valid > bps) return "WAVEFORMATEXTENSIBLE wValidBitsPerSample > wBitsPerSample";
				o->shift = bps - valid;
				if(!r.u32(false, &o->channel_mask) || !r.u16(false, &guid)) return r.err;
				if(guid != 1) return "unsupported WAVEFORMATEXTENSIBLE chunk with non-PCM format";
				sz -= 26;
			}
			o->channels = ch;
			o->rate = rate;
			o->bps = bps;
			if(!r.skip(sz)) return r.err;
			got_fmt = true;
		}
		else if(!memcmp(id, "data", 4) && guid_ok) {
			uint64_t d;
			if(!got_fmt) return "got 'data' chunk before 'fmt' chunk";
			if(!w64) {
				uint32_t x;
				if(!r.u32(false, &x)) return r.err;
				d = x;
			}
			else {
				if(!r.u64le(&d)) return r.err;
				if(d < 24) return "freakishly small Wave64 'data' chunk";
				d -= 24;
			}
			if(kind == FB200_PCM_RF64) {
				if(!got_ds64) return "RF64 file has no 'ds64' chunk before 'data' chunk";
				if(d == 0xffffffffull) d = ds64_data;
			}
			if(d == 0) return "'data' chunk has size of 0";
			o->data_bytes = d;
			o->data_pos = r.pos;
			got_data = true;
		}
		else {
			uint64_t sk;
			if(!w64) {
				uint32_t x;
				if(!r.u32(false, &x)) return r.err;
				sk = (uint64_t)x + (x & 1);
			}
			else {
				if(!r.u64le(&sk)) return r.err;
				sk = (sk + 7) & ~7ull;
				if(sk < 24) return "freakishly small Wave64 chunk";
				sk -= 24;
			}
			if(!r.skip(sk)) return r.err;
		}
	}
	if(!got_fmt) return "didn't find fmt chunk";
	if(!got_data) return "didn't find data chunk";
	o->has_data = true;
	return nullptr;
}

// read_sane_extended (encode.c:2905)
bool sane_extended(Reader &r, uint32_t *v)
{
	const uint8_t *b;
	if(!r.take(10, &b)) return false;
	const int e = (int)(int16_t)(uint16_t)(((uint32_t)b[0] << 8 | b[1]) - 0x3FFF);
	if((b[0] >> 7) == 1 || e < 0 || e >= 63) { r.err = "invalid floating-point sample rate"; return false; }
	uint64_t p = 0;
	for(int i = 0; i < 8; i++) p |= (uint64_t)b[i + 2] << (56 - i * 8);
	const int shift = 63 - e;
	*v = (uint32_t)((p >> shift) + (p >> (shift - 1) & 1));
	return true;
}

// get_sample_info_aiff (encode.c:578-803) for AIFF and AIFF-C
const char *probe_aiff(Reader &r, uint32_t kind, Probed *o)
{
	bool got_comm = false, got_ssnd = false;
	uint32_t frames = 0;
	o->big = true;
	r.pos = 12;
	while(!got_ssnd) {
		if(r.pos >= r.n) break;
		if(r.n - r.pos < 4) return "incomplete chunk identifier";
		const uint8_t *id = r.p + r.pos;
		r.pos += 4;
		if(!memcmp(id, "COMM", 4)) {
			const bool aifc = kind == FB200_PCM_AIFF_C;
			const uint32_t min_size = aifc ? 22 : 18;
			uint32_t xx, ch, bps, rate;
			if(got_comm) return "file has multiple 'COMM' chunks";
			if(!r.u32(true, &xx)) return r.err;
			if(xx < min_size) return "non-standard 'COMM' chunk";
			const uint64_t sk = (uint64_t)(xx - min_size) + (xx & 1);
			if(!r.u16(true, &ch)) return r.err;
			if(ch > 2) return "unsupported number of channels for AIFF";
			if(!r.u32(true, &frames) || !r.u16(true, &bps)) return r.err;
			o->shift = (bps % 8) ? 8 - (bps % 8) : 0;
			bps += o->shift;
			if(!sane_extended(r, &rate)) return r.err;
			if(aifc) {
				uint32_t ct;
				if(!r.u32(true, &ct)) return r.err;
				if(ct == 0x736F7774) o->big = false;  // "sowt"
				else if(ct != 0x4E4F4E45) return "can't handle AIFF-C compression type (not NONE or sowt)";
			}
			if(ch != 1 && ch != 2 && ch != 3 && ch != 5) return "unsupported number of channels for AIFF";
			o->channels = ch;
			o->bps = bps;
			o->rate = rate;
			if(!r.skip(sk)) return r.err;
			got_comm = true;
		}
		else if(!memcmp(id, "SSND", 4)) {
			uint32_t xx, off, bsz;
			if(!got_comm) return "got 'SSND' chunk before 'COMM' chunk";
			if(!r.u32(true, &xx)) return r.err;
			if(xx <= 8) return "'SSND' chunk has size <= 8";
			uint64_t d = (uint64_t)xx - 8;
			if(!r.u32(true, &off)) return r.err;
			d -= off;
			if(!r.u32(true, &bsz)) return r.err;
			if(bsz) d -= (bsz - (d % bsz));
			if(!r.skip(off)) return r.err;
			o->data_bytes = d;
			o->data_pos = r.pos;
			got_ssnd = true;
		}
		else {
			uint32_t xx;
			if(!r.u32(true, &xx)) return r.err;
			if(!r.skip((uint64_t)xx + (xx & 1))) return r.err;
		}
	}
	if(!got_comm) return "didn't find COMM chunk";
	if(!got_ssnd && frames) return "didn't find SSND chunk";
	o->has_data = got_ssnd;
	return nullptr;
}

void fail(fb200_pcm_file_info *I, uint32_t status, const char *fmt, ...)
{
	I->status = status;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(I->error, sizeof I->error, fmt, ap);
	va_end(ap);
}

void probe_one(const uint8_t *p, uint64_t n, uint64_t base, fb200_pcm_file_info *I)
{
	memset(I, 0, sizeof *I);
	// main.c:1510-1556: the kind from the first 12 bytes
	uint32_t kind = 0;
	if(n >= 12) {
		if(!memcmp(p, "RIFF", 4) && !memcmp(p + 8, "WAVE", 4)) kind = FB200_PCM_WAVE;
		else if(!memcmp(p, "RF64", 4) && !memcmp(p + 8, "WAVE", 4)) kind = FB200_PCM_RF64;
		else if(!memcmp(p, "riff\x2E\x91\xCF\x11\xA5\xD6\x28\xDB", 12)) kind = FB200_PCM_WAVE64;
		else if(!memcmp(p, "FORM", 4) && !memcmp(p + 8, "AIFF", 4)) kind = FB200_PCM_AIFF;
		else if(!memcmp(p, "FORM", 4) && !memcmp(p + 8, "AIFC", 4)) kind = FB200_PCM_AIFF_C;
	}
	if(!kind) return fail(I, FB200_PCM_NOT_CONTAINER, "not a WAVE, RF64, Wave64, AIFF or AIFF-C file");
	I->kind = kind;
	Reader r{p, n, 0};
	Probed o;
	const char *err = kind >= FB200_PCM_AIFF ? probe_aiff(r, kind, &o) : probe_wave(r, kind, &o);
	if(err) return fail(I, FB200_PCM_MALFORMED, "%s", err);
	I->channels = o.channels;
	I->container_bits = o.bps;
	I->shift = o.shift;
	I->bits_per_sample = o.bps - o.shift;
	I->sample_rate = o.rate;
	I->is_unsigned = o.is_unsigned;
	I->is_big_endian = o.big;
	I->channel_mask = o.channel_mask;
	// flac__encode_file (encode.c:934-946)
	if(o.channels == 0 || o.channels > 8) return fail(I, FB200_PCM_MALFORMED, "unsupported number of channels %u", o.channels);
	if(o.rate > 1048575) return fail(I, FB200_PCM_MALFORMED, "unsupported sample rate %u", o.rate);
	if(o.bps - o.shift < 4 || o.bps - o.shift > 32) return fail(I, FB200_PCM_MALFORMED, "unsupported bits-per-sample %u", o.bps - o.shift);
	const uint64_t bpws = (uint64_t)o.channels * (o.bps / 8);
	if(bpws == 0) return fail(I, FB200_PCM_MALFORMED, "container of %u bits holds no whole byte", o.bps);
	I->data_offset = base + o.data_pos;
	I->declared = o.data_bytes / bpws;
	// the read loop (encode.c:1305-1345): chunks of whole samples until the declared bytes or the file run out; a short last read
	// that is not whole samples fails, and format_input knows 8, 16, 24 and 32-bit containers only
	const uint64_t avail = o.data_pos < n ? n - o.data_pos : 0;
	const uint64_t present = o.has_data ? (avail < o.data_bytes ? avail : o.data_bytes) : 0;
	if(present % bpws) return fail(I, FB200_PCM_MALFORMED, "got partial sample");
	I->samples = present / bpws;
	if(I->samples && o.bps != 8 && o.bps != 16 && o.bps != 24 && o.bps != 32)
		return fail(I, FB200_PCM_MALFORMED, "unsupported input format (%u-bit container)", o.bps);
	if(I->samples == 0) return fail(I, FB200_PCM_UNSUPPORTED, "no sample present");
	if(o.rate == 0) return fail(I, FB200_PCM_UNSUPPORTED, "sample rate 0");
	if(I->bits_per_sample == 32) return fail(I, FB200_PCM_UNSUPPORTED, "32-bit samples");
	I->status = FB200_PCM_OK;
}

// One file's blocks after STREAMINFO, as EncoderSession_init_encoder lists them for a non-FLAC input (encode.c:1945-2020):
// SEEKTABLE template (when there is one), VORBIS_COMMENT (entries; the vendor is the encoder's), PADDING (padding >= 0). length is
// total_samples_to_encode: the declared count, or the --skip / --until range's length (encode.c:2010, 2226)
void file_metadata(const fb200_pcm_file_info &I, uint64_t length, const fb200_pcm_encode_options &opt, const char *tags, size_t tags_len, FileMeta *M)
{
	const std::vector<uint8_t> st = seek_template(opt.seek_spacing_s, length, I.sample_rate);
	if(!st.empty()) put_block(M->before, 3, st);
	std::vector<std::string> &ent = M->ent;
	for(size_t p = 0; p < tags_len;) {
		const size_t e = strnlen(tags + p, tags_len - p);
		ent.emplace_back(tags + p, e);
		p += e + 1;
	}
	if(I.channel_mask) set_channel_mask_tag(ent, I.channel_mask);
	if(opt.padding != 0) {
		// with --replay-gain, room for its tags (GRABBAG__REPLAYGAIN_MAX_TAG_SPACE_REQUIRED, encode.c:2004-2011)
		uint64_t len = (opt.padding > 0 ? (uint64_t)opt.padding : (length / I.sample_rate < 20 * 60 ? 8192 : 65536)) + (opt.replay_gain ? 190 : 0);
		if(len > (1u << 24) - 1) len = (1u << 24) - 1;
		M->padding = (int64_t)len;
	}
}

// ranges == nullptr: every file whole (flac *.wav); else one output per range (flac --skip=first --until=first+samples)
int encode_pcm_files(fb200_encoder *e, const uint8_t *data, bool device, const uint64_t *file_offsets, uint32_t nfiles, const fb200_pcm_file_info *info,
                     const fb200_pcm_encode_options *opt, const fb200_sample_range *ranges, uint32_t nranges, const uint8_t *tags,
                     const uint64_t *tag_offsets, uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                     fb200_flac_file_info *files, void *cuda_stream)
{
	if(!e || !data || !file_offsets || !info || !opt || !files) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	if(nfiles == 0) { set_error("no files"); return FB200_ERR_INVALID; }
	if(!tags != !tag_offsets) { set_error("tags and tag_offsets must both be given or both be NULL"); return FB200_ERR_INVALID; }
	if(ranges && (nranges == 0 || nranges >= 0x80000000u)) { set_error("invalid number of ranges %u", nranges); return FB200_ERR_INVALID; }
	const uint32_t nout = ranges ? nranges : nfiles;
	const char *unit = ranges ? "range" : "file";
	std::vector<uint8_t> used(nfiles, ranges ? 0 : 1);
	for(uint32_t r = 0; ranges && r < nranges; r++) {
		const fb200_sample_range &q = ranges[r];
		if(q.file >= nfiles) { set_error("range %u: file %u of a batch of %u", r, q.file, nfiles); return FB200_ERR_INVALID; }
		if(q.samples == 0) { set_error("range %u is empty", r); return FB200_ERR_INVALID; }
		if(q.first_sample + q.samples < q.first_sample) { set_error("range %u: first_sample + samples overflows", r); return FB200_ERR_INVALID; }
		used[q.file] = 1;
	}
	fb200_encoder_config cfg;
	fb200_encoder_get_config(e, &cfg);
	const uint64_t begin = file_offsets[0], end = file_offsets[nfiles];
	if(end < begin) { set_error("file_offsets decrease"); return FB200_ERR_INVALID; }
	PcmSource src;
	src.data = data + begin;
	src.bytes = end - begin;
	src.files.resize(nout);
	std::vector<uint64_t> samples(nout), moffs(nout + 1, 0);
	std::vector<uint8_t> meta;
	RgRebuild rgr;
	rgr.files.resize(opt->replay_gain ? nout : 0);
	ReplayGainJob rg{0, 0, 0, {}, rg_rebuild, &rgr};
	if(opt->replay_gain) src.rg = &rg;
	for(uint32_t f = 0; f < nfiles; f++) {
		const fb200_pcm_file_info &I = info[f];
		if(file_offsets[f + 1] < file_offsets[f]) { set_error("file_offsets decrease at file %u", f); return FB200_ERR_INVALID; }
		if(!used[f]) continue;
		if(I.status != FB200_PCM_OK) { set_error("file %u was not probed OK: %s", f, I.error); return FB200_ERR_INVALID; }
		if(I.channels != cfg.channels || I.bits_per_sample != cfg.bits_per_sample || I.sample_rate != cfg.sample_rate) {
			set_error("file %u is %u ch / %u bits / %u Hz, the encoder %u / %u / %u", f, I.channels, I.bits_per_sample, I.sample_rate, cfg.channels,
			          cfg.bits_per_sample, cfg.sample_rate);
			return FB200_ERR_INVALID;
		}
		// encode.c:1684-1692
		if(opt->replay_gain && (I.channels < 1 || I.channels > 2)) { set_error("file %u: %u channels; --replay-gain takes 1 or 2", f, I.channels); return FB200_ERR_INVALID; }
		if(opt->replay_gain && !replaygain_rate(I.sample_rate, &rg.ds, &rg.W, &rg.filt)) {
			set_error("file %u: invalid sample rate %u for --replay-gain", f, I.sample_rate);
			return FB200_ERR_INVALID;
		}
		const uint32_t B = I.container_bits / 8;
		if(B < 1 || B > 4 || I.shift >= I.container_bits || I.data_offset < file_offsets[f] || I.data_offset > file_offsets[f + 1] ||
		   I.samples > I.declared || I.samples * I.channels * B > file_offsets[f + 1] - I.data_offset) {
			set_error("info of file %u does not describe this batch's file %u", f, f);
			return FB200_ERR_INVALID;
		}
	}
	uint64_t elem = 0;
	for(uint32_t r = 0; r < nout; r++) {
		const uint32_t f = ranges ? ranges[r].file : r;
		const fb200_pcm_file_info &I = info[f];
		// the tool's checks after canonicalising --skip / --until against the declared count (encode.c:1043, 2296); a range past the
		// samples present is refused here, where the tool writes an empty stream
		const uint64_t first = ranges ? ranges[r].first_sample : 0, length = ranges ? ranges[r].samples : I.declared;
		if(first > I.declared) { set_error("range %u of file %u: value of --skip exceeds input size", r, f); return FB200_ERR_INVALID; }
		if(first + length > I.declared) { set_error("range %u of file %u: --until value is after end of input", r, f); return FB200_ERR_INVALID; }
		if(first >= I.samples) { set_error("range %u of file %u starts at sample %llu, past the %llu samples present", r, f, (unsigned long long)first, (unsigned long long)I.samples); return FB200_ERR_INVALID; }
		if(tags && (tag_offsets[r + 1] < tag_offsets[r] || (tag_offsets[r + 1] > tag_offsets[r] && tags[tag_offsets[r + 1] - 1] != 0))) {
			set_error("tags of %s %u do not end in a NUL", unit, r);
			return FB200_ERR_INVALID;
		}
		const uint32_t B = I.container_bits / 8;
		const uint64_t present = (first + length < I.samples ? first + length : I.samples) - first;
		src.files[r] = PcmFileDev{elem, I.data_offset - begin + first * I.channels * B, B, I.is_big_endian ? 1u : 0u, I.is_unsigned ? 1u : 0u, I.shift};
		samples[r] = present;
		elem += present * I.channels;
		FileMeta M;
		file_metadata(I, length, *opt, tags ? reinterpret_cast<const char *>(tags) + tag_offsets[r] : nullptr, tags ? tag_offsets[r + 1] - tag_offsets[r] : 0, &M);
		put_file_metadata(M, meta);
		moffs[r + 1] = meta.size();
		if(opt->replay_gain) {
			// EncoderSession_process analyses the values format_input shifted down, scaled by the container's bits
			rg.bps.push_back(I.container_bits);
			rgr.files[r] = std::move(M);
		}
	}
	meta.push_back(0);
	return encode_pcm_files_impl(e, src, device, samples.data(), nout, opt->md5 ? 1 : 0, meta.data(), moffs.data(), out, out_capacity, frame_offsets, nframes,
	                             files, cuda_stream);
}

}  // namespace

}  // namespace fb200

using namespace fb200;

int fb200_pcm_files_probe(const uint8_t *data, uint64_t nbytes, const uint64_t *file_offsets, uint32_t nfiles, fb200_pcm_file_info *info)
{
	if(!file_offsets || !info || (!data && nfiles)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	for(uint32_t f = 0; f < nfiles; f++)
		if(file_offsets[f + 1] < file_offsets[f] || file_offsets[f + 1] > nbytes) { set_error("file %u lies outside the %llu bytes", f, (unsigned long long)nbytes); return FB200_ERR_INVALID; }
	for(uint32_t f = 0; f < nfiles; f++) probe_one(data + file_offsets[f], file_offsets[f + 1] - file_offsets[f], file_offsets[f], &info[f]);
	return FB200_OK;
}

int fb200_encode_pcm_files_host(fb200_encoder *e, const uint8_t *data, const uint64_t *file_offsets, uint32_t nfiles, const fb200_pcm_file_info *info,
                                const fb200_pcm_encode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *out, size_t out_capacity,
                                uint64_t *frame_offsets, uint64_t *nframes, fb200_flac_file_info *files)
{
	return encode_pcm_files(e, data, false, file_offsets, nfiles, info, opt, nullptr, 0, tags, tag_offsets, out, out_capacity, frame_offsets, nframes, files,
	                        nullptr);
}

int fb200_encode_pcm_files_device(fb200_encoder *e, const uint8_t *d_data, const uint64_t *file_offsets, uint32_t nfiles, const fb200_pcm_file_info *info,
                                  const fb200_pcm_encode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *d_out, size_t out_capacity,
                                  uint64_t *d_frame_offsets, uint64_t *nframes, fb200_flac_file_info *files, void *cuda_stream)
{
	return encode_pcm_files(e, d_data, true, file_offsets, nfiles, info, opt, nullptr, 0, tags, tag_offsets, d_out, out_capacity, d_frame_offsets, nframes,
	                        files, cuda_stream);
}

int fb200_encode_pcm_files_ranges_host(fb200_encoder *e, const uint8_t *data, const uint64_t *file_offsets, uint32_t nfiles, const fb200_pcm_file_info *info,
                                       const fb200_pcm_encode_options *opt, const fb200_sample_range *ranges, uint32_t nranges, const uint8_t *tags,
                                       const uint64_t *tag_offsets, uint8_t *out, size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes,
                                       fb200_flac_file_info *files)
{
	if(!ranges) { set_error("ranges is NULL"); return FB200_ERR_INVALID; }
	return encode_pcm_files(e, data, false, file_offsets, nfiles, info, opt, ranges, nranges, tags, tag_offsets, out, out_capacity, frame_offsets, nframes,
	                        files, nullptr);
}

int fb200_encode_pcm_files_ranges_device(fb200_encoder *e, const uint8_t *d_data, const uint64_t *file_offsets, uint32_t nfiles,
                                         const fb200_pcm_file_info *info, const fb200_pcm_encode_options *opt, const fb200_sample_range *ranges,
                                         uint32_t nranges, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *d_out, size_t out_capacity,
                                         uint64_t *d_frame_offsets, uint64_t *nframes, fb200_flac_file_info *files, void *cuda_stream)
{
	if(!ranges) { set_error("ranges is NULL"); return FB200_ERR_INVALID; }
	return encode_pcm_files(e, d_data, true, file_offsets, nfiles, info, opt, ranges, nranges, tags, tag_offsets, d_out, out_capacity, d_frame_offsets,
	                        nframes, files, cuda_stream);
}

// ---- flac [--skip] [--until]: the tool's arithmetic (utils.c:50-107, 326-398; main.c:1659-1670; encode.c:1003-1081, 2257-2303)

namespace {

// local__parse_uint64_
bool parse_u64(const char *s, uint64_t *v)
{
	uint64_t r = 0;
	if(!*s) return false;
	for(char c; (c = *s++) != '\0';) {
		if(c < '0' || c > '9') return false;
		if(r > UINT64_MAX / 10) return false;
		const uint64_t t = r * 10 + (uint64_t)(c - '0');
		if(r == UINT64_MAX / 10 && t < r) return false;
		r = t;
	}
	*v = r;
	return true;
}

// local__parse_timecode_: [0-9]+:[0-9.,]* read by strtod in the C locale
bool parse_timecode(const char *s, double *v)
{
	char c = *s++;
	if(c < '0' || c > '9') return false;
	uint32_t i = (uint32_t)(c - '0');
	while((c = *s++) != ':') {
		if(c < '0' || c > '9') return false;
		i = i * 10 + (uint32_t)(c - '0');
	}
	if(strspn(s, "1234567890.,") != strlen(s)) return false;
	char *end;
	const double d = strtod(s, &end);
	if(end == s || *end) return false;
	*v = (double)i * 60. + d;
	return true;
}

struct SkipUntil {
	bool relative = false, is_samples = true;
	int64_t samples = 0;
	double seconds = 0;
};

// flac__utils_parse_skip_until_specification
bool parse_spec(const char *s, SkipUntil *o)
{
	*o = SkipUntil{};
	if(!s) return true;
	bool neg = false;
	if(s[0] == '-') { neg = o->relative = true; s++; }
	else if(s[0] == '+') { o->relative = true; s++; }
	uint64_t v;
	if(parse_u64(s, &v)) {
		if(v > (uint64_t)INT64_MAX) return false;
		o->samples = neg ? -(int64_t)v : (int64_t)v;
		return true;
	}
	double d;
	if(!parse_timecode(s, &d)) return false;
	o->is_samples = false;
	o->seconds = neg ? -d : d;
	return true;
}

// flac__utils_canonicalize_skip_until_specification: seconds to samples, truncated
bool canonicalize(SkipUntil *o, uint32_t rate)
{
	if(o->is_samples) return true;
	const double x = o->seconds * (double)rate;
	if(x >= (double)INT64_MAX || x <= (double)INT64_MIN) return false;
	o->samples = (int64_t)x;
	o->is_samples = true;
	return true;
}

}  // namespace

int fb200_skip_until(const char *skip, const char *until, uint32_t sample_rate, uint64_t total_samples, uint64_t *first_sample, uint64_t *samples)
{
	if(!first_sample || !samples) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	*first_sample = *samples = 0;
	SkipUntil S, U;
	if(!parse_spec(skip, &S) || S.relative) { set_error("invalid value for --skip"); return FB200_ERR_INVALID; }
	if(!parse_spec(until, &U)) { set_error("invalid value for --until"); return FB200_ERR_INVALID; }
	if(!until) U.relative = true;  // no --until is --until=-0
	if(!canonicalize(&S, sample_rate)) { set_error("value of --skip is too large"); return FB200_ERR_INVALID; }
	const uint64_t s = (uint64_t)S.samples;
	// canonicalize_until_specification; 0 means end of stream
	uint64_t u = 0;
	if(!canonicalize(&U, sample_rate)) { set_error("value of --until is too large"); return FB200_ERR_INVALID; }
	if(!(U.relative && U.samples == 0)) {
		if(total_samples == 0) { set_error("cannot use --until when input length is unknown"); return FB200_ERR_INVALID; }
		int64_t v = U.samples;
		if(U.relative) v = (int64_t)((uint64_t)v + (U.samples <= 0 ? total_samples : s));  // two's complement, as the tool's int64 sum
		if(v < 0) { set_error("--until value is before beginning of input"); return FB200_ERR_INVALID; }
		if((uint64_t)v <= s) { set_error("--until value is before --skip point"); return FB200_ERR_INVALID; }
		if((uint64_t)v > total_samples) { set_error("--until value is after end of input"); return FB200_ERR_INVALID; }
		u = (uint64_t)v;
	}
	if(s > total_samples) { set_error("value of --skip exceeds input size"); return FB200_ERR_INVALID; }
	const uint64_t n = (u ? u : total_samples) - s;
	// the tool writes a stream without frames here; this engine encodes no empty file
	if(n == 0) { set_error("--skip leaves no samples to encode"); return FB200_ERR_INVALID; }
	*first_sample = s;
	*samples = n;
	return FB200_OK;
}

int fb200_pcm_header(const fb200_pcm_decode_options *opt, uint32_t channels, uint32_t bits_per_sample, uint32_t sample_rate, uint32_t channel_mask,
                     uint64_t samples, uint8_t *out, uint32_t capacity, uint32_t *length)
{
	if(!length || (!out && capacity)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	*length = 0;
	if(!pcm_decode_options_ok(opt)) return FB200_ERR_INVALID;
	if(channels < 1 || channels > 8 || bits_per_sample < 4 || bits_per_sample > 32) {
		set_error("%u channels of %u bits", channels, bits_per_sample);
		return FB200_ERR_INVALID;
	}
	PcmHeader h;
	pcm_header_build(*opt, channels, bits_per_sample, sample_rate, channel_mask, samples, &h);
	if(h.too_big) { set_error("stream is too big to fit in a single file of this kind"); return FB200_ERR_UNSUPPORTED; }
	*length = h.length;
	if(capacity < h.length) { set_error("the header needs %u bytes", h.length); return FB200_ERR_OUTPUT_TOO_SMALL; }
	memcpy(out, h.bytes, h.length);
	return FB200_OK;
}
