// add_replaygain.cu -- fb200_add_replaygain_flac_files_*: ReplayGain tags on files of the batch fb200_decode_files_index left
// resident, as metaflac --add-replay-gain writes them (src/metaflac/operations.c:557-650). Per album: the STREAMINFO pre-checks on
// the host; the whole-file decode of the listed files with every accepted frame's placement kept on the device; k_replaygain_frames
// (replaygain_kernel.cu), which checks that the frames tile each file and analyses them frame by frame as metaflac's write callback
// feeds them; the metadata chain rules on the host (fb200_replaygain_rewrite_head); and k_files_splice, which puts each new head in
// front of the input's audio bytes.
#include <stdarg.h>
#include <string.h>

#include <map>

#include "fb200_internal.h"
#include "flac_metadata.h"
#include "flac_parse.h"

extern "C" const char *FLAC__VENDOR_STRING;

namespace fb200 {

namespace {

// ---- the metadata chain (src/libFLAC/metadata_iterators.c)

// A block of the chain: its type and body as the chain writes it (the VORBIS_COMMENT's is rebuilt from vendor and entries,
// PADDING's is `length` zero bytes).
struct ChainBlock {
	uint32_t type;
	uint64_t length;
	std::vector<uint8_t> body;
	std::string vendor;
	std::vector<std::string> ent;
};

// A PICTURE whose body is exactly its fields (big-endian lengths)
bool read_picture(const std::vector<uint8_t> &b)
{
	auto be32 = [&](size_t at) { return be(b.data() + at, 4); };
	const size_t n = b.size();
	size_t pos = 4;
	if(n < pos) return false;
	for(int s = 0; s < 2; s++) {  // MIME type, description
		if(n - pos < 4 || n - pos - 4 < be32(pos)) return false;
		pos += 4 + (size_t)be32(pos);
	}
	if(n - pos < 20 || n - pos - 20 < be32(pos + 16)) return false;
	return pos + 20 + (size_t)be32(pos + 16) == n;
}

uint64_t chain_length(const std::vector<ChainBlock> &L)
{
	uint64_t n = 0;
	for(const ChainBlock &b : L) n += 4 + b.length;
	return n;
}

}  // namespace

const char kBlockTooLong[] = "a metadata block is too long for its length field";  // the one refusal of the chain write

// metaflac's store_to_file_pre_ / grabbag__replaygain_store_to_vorbiscomment / store_to_file_post_ on one file: nullptr and the
// new head, or the reason the chain read refuses the file, or kBlockTooLong when the chain write does.
const char *rg_rewrite_head(const uint8_t *m, uint64_t n, const float v[4], std::vector<uint8_t> *head, uint64_t *audio_in, bool *in_place)
{
	// FLAC__metadata_chain_read: an ID3v2 tag, "fLaC", the blocks (STREAMINFO first)
	const MetaRegion r = read_metadata_region(m, n);
	if(r.end == MetaRegion::NO_MARKER) return "not a FLAC file";
	std::vector<ChainBlock> L;
	for(const MetaBlock &h : r.blocks) {
		ChainBlock b{h.type, h.length, std::vector<uint8_t>(m + h.body, m + h.body + h.length), {}, {}};
		switch(h.type) {
			case 0: if(h.length != 34) return "STREAMINFO is not 34 bytes"; break;
			case 1: b.body.clear(); break;
			case 2: if(h.length < 4) return "APPLICATION block shorter than 4 bytes"; break;
			case 3: if(h.length % 18) return "SEEKTABLE length is not a multiple of 18"; break;
			case 4:
				if(!read_metadata_block_data_vorbis_comment(b.body.data(), h.length, &b.vendor, &b.ent)) return "VORBIS_COMMENT fields run past the block";
				break;
			case 5: if(!cuesheet_zero_reserved(b.body.data(), b.body.size())) return "CUESHEET body is not exactly its fields"; break;
			case 6: if(!read_picture(b.body)) return "PICTURE body is not exactly its fields"; break;
			default: break;
		}
		L.push_back(std::move(b));
	}
	if(r.end == MetaRegion::SHORT) return "metadata runs past the file";
	if(L.front().type != 0) return "first metadata block is not STREAMINFO";
	const uint64_t initial = chain_length(L);
	*audio_in = r.audio;

	// the first VORBIS_COMMENT, or a new one after the last block; the three edits (grabbag__replaygain_store_to_vorbiscomment)
	size_t vc = 0;
	while(vc < L.size() && L[vc].type != 4) vc++;
	if(vc == L.size()) L.push_back(ChainBlock{4, 0, {}, FLAC__VENDOR_STRING, {}});
	ChainBlock &V = L[vc];
	rg_edit(V.ent, RG_REFERENCE, 0.f, 0.f);
	rg_edit(V.ent, RG_TRACK_GAIN, v[0], v[1]);
	rg_edit(V.ent, RG_ALBUM_GAIN, v[2], v[3]);
	V.body.clear();
	put_vorbis_comment(V.body, V.vendor, V.ent);
	V.length = V.body.size();

	// FLAC__metadata_chain_sort_padding: every PADDING to the end, in order, then merged (4 + length per merged block)
	{
		std::vector<ChainBlock> kept, pads;
		for(ChainBlock &b : L) (b.type == 1 ? pads : kept).push_back(std::move(b));
		if(!pads.empty()) {
			ChainBlock p = std::move(pads[0]);
			for(size_t i = 1; i < pads.size(); i++) p.length += 4 + pads[i].length;
			kept.push_back(std::move(p));
		}
		L.swap(kept);
	}

	// chain_prepare_for_write_ with use_padding
	const int64_t pad = chain_padding(initial, chain_length(L), L.back().type == 1 ? (int64_t)L.back().length : -1);
	if(L.back().type == 1) L.pop_back();
	if(pad >= 0) L.push_back(ChainBlock{1, (uint64_t)pad, {}, {}, {}});
	for(ChainBlock &b : L)
		if(b.length >= (1u << 24)) {
			if(b.type != 1) return kBlockTooLong;
			b.length = (1u << 24) - 1;
		}
	*in_place = chain_length(L) == initial;

	head->assign(m, m + r.marker + 4);
	for(size_t i = 0; i < L.size(); i++) {
		const ChainBlock &b = L[i];
		put_block_header(*head, i + 1 == L.size(), b.type, (uint32_t)b.length);
		if(b.type == 1) head->insert(head->end(), (size_t)b.length, 0);
		else head->insert(head->end(), b.body.begin(), b.body.end());
	}
	return nullptr;
}

namespace {

// The most a file's metadata can grow by: a new VORBIS_COMMENT (header, vendor length, this library's vendor string, entry count)
// with the five longest entries: the reference loudness "...=89.0 dB" (37 bytes), "..._GAIN=-24601.00 dB" (34) and
// "..._PEAK=1.00000000" (32) twice. FB200_ADD_REPLAYGAIN_GROWTH is documented as at least this; a vendor string that outgrew it
// would raise the bound the call checks, never let it write past out_capacity.
uint64_t growth_bound()
{
	const uint64_t g = 4 + 4 + strlen(FLAC__VENDOR_STRING) + 4 + 5 * 4 + 37 + 2 * (34 + 32);
	return g > FB200_ADD_REPLAYGAIN_GROWTH ? g : FB200_ADD_REPLAYGAIN_GROWTH;
}

void fail(fb200_add_replaygain_info &I, uint32_t status, const char *fmt, ...)
{
	I.status = status;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(I.error, sizeof I.error, fmt, ap);
	va_end(ap);
}

// ---- k_files_splice: segments of bytes, from the resident batch or the heads blob, to the output at any byte phase

struct SpliceSeg { unsigned long long src, dst, n, item0; uint32_t from_blob, pad; };
constexpr unsigned kSpliceItem = 1u << 16;  // bytes per CTA

// One CTA per kSpliceItem bytes of a segment. The destination's aligned 16-byte words are stored whole, each built from five
// aligned 4-byte source words and a funnel shift; the ragged bytes at either end are stored one by one. Both sources are read at
// most 4 bytes past a segment's end (the batch has 64 bytes of slack behind it, the blob 16).
__global__ void __launch_bounds__(256) k_files_splice(const uint8_t *__restrict__ batch, const uint8_t *__restrict__ blob, const SpliceSeg *__restrict__ segs,
                                                     int nsegs, uint8_t *__restrict__ out)
{
	int lo = 0, hi = nsegs - 1;
	while(lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		if(segs[mid].item0 <= blockIdx.x) lo = mid;
		else hi = mid - 1;
	}
	const SpliceSeg S = segs[lo];
	const unsigned long long b0 = (blockIdx.x - S.item0) * (unsigned long long)kSpliceItem;
	const unsigned long long b1 = min(S.n, b0 + kSpliceItem);
	if(b0 >= b1) return;
	const uint8_t *src = (S.from_blob ? blob : batch) + S.src;
	uint8_t *dst = out + S.dst;
	const uintptr_t d0 = (uintptr_t)(dst + b0), d1 = (uintptr_t)(dst + b1);
	const uintptr_t a0 = (d0 + 15) & ~(uintptr_t)15, a1 = d1 & ~(uintptr_t)15;
	if(a0 >= a1) {
		for(unsigned long long i = b0 + threadIdx.x; i < b1; i += blockDim.x) dst[i] = src[i];
		return;
	}
	for(uintptr_t a = d0 + threadIdx.x; a < a0; a += blockDim.x) *(uint8_t *)a = src[a - (uintptr_t)dst];
	for(uintptr_t a = a1 + threadIdx.x; a < d1; a += blockDim.x) *(uint8_t *)a = src[a - (uintptr_t)dst];
	for(uintptr_t a = a0 + 16 * (uintptr_t)threadIdx.x; a < a1; a += 16 * (uintptr_t)blockDim.x) {
		const uintptr_t s = (uintptr_t)src + (a - (uintptr_t)dst);
		const uint32_t *w = reinterpret_cast<const uint32_t *>(s & ~(uintptr_t)3);
		const unsigned sh = 8u * (unsigned)(s & 3);
		uint32_t x[5];
#pragma unroll
		for(int k = 0; k < 5; k++) x[k] = __ldg(w + k);
		uint4 o;
		o.x = __funnelshift_r(x[0], x[1], sh);
		o.y = __funnelshift_r(x[1], x[2], sh);
		o.z = __funnelshift_r(x[2], x[3], sh);
		o.w = __funnelshift_r(x[3], x[4], sh);
		*reinterpret_cast<uint4 *>(a) = o;
	}
}

// One album: its files' places in the list, in list order.
struct Album { std::vector<uint32_t> at; bool ok = true; };

// Steps 1 and 2 of the call for the listed files: info[] status, album and rg filled for each file; *windows (when not null)
// gets every window of the files that pass, file after file. *launches: kernels launched.
int analyse(fb200_decoder *dec, int device, const uint32_t *files, const uint32_t *albums, uint32_t nfiles, fb200_add_replaygain_info *info,
            std::vector<double> *windows, std::map<uint32_t, Album> *out_albums, std::vector<std::vector<uint8_t>> *regions, cudaStream_t st)
{
	std::map<uint32_t, Album> &A = *out_albums;
	for(uint32_t i = 0; i < nfiles; i++) {
		fb200_add_replaygain_info &O = info[i];
		memset(&O, 0, sizeof O);
		O.album = albums ? albums[i] : 0;
		A[O.album].at.push_back(i);
	}
	auto album_fails = [&](Album &al, uint32_t bad) {
		al.ok = false;
		for(uint32_t i : al.at)
			if(i != bad && info[i].status == FB200_ADD_RG_OK) fail(info[i], FB200_ADD_RG_ALBUM, "files[%u] of this album failed", bad);
	};
	// metaflac reads every file's metadata chain before anything else (do_shorthand_operations_on_file): a file the chain read
	// refuses fails the invocation, and nothing is written
	regions->assign(nfiles, {});
	for(auto &kv : A) {
		Album &al = kv.second;
		int64_t bad = -1;
		for(uint32_t i : al.at) {
			if(decoder_file_info(dec, files[i]).status != FB200_FILE_OK) continue;
			int rc;
			if((rc = decoder_file_metadata(dec, files[i], &(*regions)[i])) != FB200_OK) return rc;
			const float zero[4] = {0.f, 0.f, 0.f, 0.f};
			std::vector<uint8_t> head;
			uint64_t audio_in;
			bool in_place;
			const char *why = rg_rewrite_head((*regions)[i].data(), (*regions)[i].size(), zero, &head, &audio_in, &in_place);
			if(why && why != kBlockTooLong) {  // a chain write that fails is step 3's
				fail(info[i], FB200_ADD_RG_METADATA, "%s", why);
				if(bad < 0) bad = i;
			}
		}
		if(bad >= 0) album_fails(al, (uint32_t)bad);
	}
	for(auto &kv : A) {
		Album &al = kv.second;
		if(!al.ok) continue;
		// step 1: STREAMINFO pre-checks, in list order, against the album's first file
		const fb200_file_decode_info *first = nullptr;
		for(uint32_t i : al.at) {
			const fb200_file_decode_info &I = decoder_file_info(dec, files[i]);
			uint32_t ds, W, filt;
			if(I.status != FB200_FILE_OK) fail(info[i], FB200_ADD_RG_INPUT, "index status %u", I.status);
			else if(first && I.sample_rate != first->sample_rate) fail(info[i], FB200_ADD_RG_FORMAT, "%u Hz, the album's first file %u Hz", I.sample_rate, first->sample_rate);
			else if(first && I.bits_per_sample != first->bits_per_sample) fail(info[i], FB200_ADD_RG_FORMAT, "%u bits, the album's first file %u", I.bits_per_sample, first->bits_per_sample);
			else if(first && I.channels != first->channels) fail(info[i], FB200_ADD_RG_FORMAT, "%u channels, the album's first file %u", I.channels, first->channels);
			else if(!replaygain_rate(I.sample_rate, &ds, &W, &filt)) fail(info[i], FB200_ADD_RG_FORMAT, "sample rate %u Hz is not supported", I.sample_rate);
			else if(I.channels > 2) fail(info[i], FB200_ADD_RG_FORMAT, "%u channels; ReplayGain takes 1 or 2", I.channels);
			if(info[i].status != FB200_ADD_RG_OK) { album_fails(al, i); break; }
			if(!first) first = &I;
		}
	}

	// step 2: decode the files of the albums that passed, their placements kept; one analysis launch
	const DecoderFilesView V = decoder_files_view(dec);
	std::vector<uint32_t> batch, place_of;  // decoded files (batch index) and their places in files[]
	std::vector<uint64_t> first_value;
	std::vector<RgFramesFileDev> dev;
	uint64_t values = 0, nwin_cap = 0;
	for(auto &kv : A) {
		if(!kv.second.ok) continue;
		for(uint32_t i : kv.second.at) {
			const uint32_t f = files[i];
			const fb200_file_decode_info &I = decoder_file_info(dec, f);
			const DecoderFileSpan sp = decoder_file_span(dec, f);
			RgFramesFileDev D{};
			replaygain_rate(I.sample_rate, &D.ds, &D.W, &D.filt);
			D.cand0 = sp.cand0; D.ncand = sp.ncand; D.audio = sp.audio; D.end = sp.end;
			D.win = nwin_cap;
			D.nwin_cap = I.samples / D.ds / D.W;
			D.state = sp.state; D.channels = I.channels; D.bps = I.bits_per_sample;
			nwin_cap += D.nwin_cap;
			dev.push_back(D);
			batch.push_back(f);
			place_of.push_back(i);
			first_value.push_back(values);
			values += I.samples * I.channels;
		}
	}
	const size_t nf = dev.size();
	std::vector<RgFramesOut> res(nf);
	std::vector<double> v(nwin_cap);
	if(nf) {
		const size_t o_place = 0, o_bytes = (o_place + V.ncand * sizeof(FilePlace) + 15) & ~(size_t)15;
		const size_t o_dev = (o_bytes + V.ncand * sizeof(uint32_t) + 15) & ~(size_t)15, o_out = (o_dev + nf * sizeof(RgFramesFileDev) + 15) & ~(size_t)15;
		const size_t o_v = (o_out + nf * sizeof(RgFramesOut) + 15) & ~(size_t)15, o_pcm = (o_v + nwin_cap * sizeof(double) + 15) & ~(size_t)15;
		uint8_t *d = nullptr;
		FB_CUDA(cudaMalloc(&d, o_pcm + values * sizeof(int32_t) + 16));
		struct Free { uint8_t *p; ~Free() { cudaFree(p); } } hold{d};
		FilePlace *d_place = reinterpret_cast<FilePlace *>(d + o_place);
		uint32_t *d_bytes = reinterpret_cast<uint32_t *>(d + o_bytes);
		int32_t *d_pcm = reinterpret_cast<int32_t *>(d + o_pcm);
		FB_CUDA(cudaMemcpyAsync(d + o_dev, dev.data(), nf * sizeof(RgFramesFileDev), cudaMemcpyHostToDevice, st));
		int rc = decoder_decode_into(dec, batch.data(), first_value.data(), (uint32_t)nf, d_pcm, values, nullptr, 0, st, d_place, d_bytes);
		if(rc != FB200_OK) return rc;
		launch_replaygain_frames(d_pcm, reinterpret_cast<const RgFramesFileDev *>(d + o_dev), (int)nf, d_place, V.begins, d_bytes, V.cands, V.states,
		                         reinterpret_cast<double *>(d + o_v), reinterpret_cast<RgFramesOut *>(d + o_out), st);
		decoder_count_launches(dec, 1);
		FB_CUDA(cudaGetLastError());
		FB_CUDA(cudaMemcpyAsync(res.data(), d + o_out, nf * sizeof(RgFramesOut), cudaMemcpyDeviceToHost, st));
		if(nwin_cap) FB_CUDA(cudaMemcpyAsync(v.data(), d + o_v, nwin_cap * sizeof(double), cudaMemcpyDeviceToHost, st));
		FB_CUDA(cudaStreamSynchronize(st));
	}
	(void)device;

	// the first file of an album that did not decode cleanly fails it; the others get their values
	std::vector<RgFileDev> rf;
	std::vector<uint32_t> ralbum, rpeak, rat;
	std::vector<uint64_t> rnwin;
	for(size_t k = 0; k < nf; k++) {
		const uint32_t i = place_of[k];
		Album &al = A[info[i].album];
		if(!al.ok) continue;
		if(!res[k].ok) {
			fail(info[i], FB200_ADD_RG_DECODE, "a decode error: a damaged or missing frame, or bytes no frame covers");
			album_fails(al, i);
		}
	}
	for(size_t k = 0; k < nf; k++) {
		const uint32_t i = place_of[k];
		if(!A[info[i].album].ok) continue;
		RgFileDev F{};
		F.win = dev[k].win; F.ds = dev[k].ds; F.W = dev[k].W; F.bps = dev[k].bps;
		rf.push_back(F);
		ralbum.push_back(info[i].album);
		rpeak.push_back(res[k].peak);
		rnwin.push_back(res[k].nwin);
		rat.push_back(i);
		if(windows) windows->insert(windows->end(), v.begin() + dev[k].win, v.begin() + dev[k].win + res[k].nwin);
	}
	std::vector<fb200_replaygain_info> ri(rf.size());
	if(!rf.empty()) replaygain_results(rf, ralbum.data(), v.data(), rpeak.data(), ri.data(), rnwin.data());
	for(size_t k = 0; k < rf.size(); k++) info[rat[k]].rg = ri[k];
	return FB200_OK;
}

// checks of both entry points and the hook; *nbatch the batch's size and *device the decoder's
int check_call(fb200_decoder *dec, const uint32_t *files, uint32_t nfiles, int *device)
{
	uint32_t nbatch = 0;
	if(!decoder_files(dec, &nbatch, device)) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	std::vector<uint8_t> seen(nbatch, 0);
	for(uint32_t i = 0; i < nfiles; i++) {
		const uint32_t f = files[i];
		if(f >= nbatch) { set_error("files[%u] = %u, the batch has %u files", i, f, nbatch); return FB200_ERR_INVALID; }
		if(seen[f]) { set_error("file %u is listed twice", f); return FB200_ERR_INVALID; }
		seen[f] = 1;
	}
	return FB200_OK;
}

int add_replaygain(fb200_decoder *dec, bool device_out, const uint32_t *files, const uint32_t *albums, uint32_t nfiles, const fb200_add_replaygain_options *opt,
                   uint8_t *out, size_t out_capacity, fb200_add_replaygain_info *info, cudaStream_t st)
{
	if(!dec || !files || !opt || !info || (!out && out_capacity)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	if(opt->reserved != 0) { set_error("fb200_add_replaygain_options.reserved must be 0"); return FB200_ERR_INVALID; }
	int device = 0, rc;
	if((rc = check_call(dec, files, nfiles, &device)) != FB200_OK) return rc;
	const bool whole = opt->whole_files != 0;
	if(!opt->scan_only) {
		uint64_t need = 0;
		for(uint32_t i = 0; i < nfiles; i++) {
			if(decoder_file_info(dec, files[i]).status != FB200_FILE_OK) continue;
			const DecoderFileSpan sp = decoder_file_span(dec, files[i]);
			need += (whole ? sp.end : sp.audio) - sp.start + growth_bound();
		}
		if(need > out_capacity) {
			set_error("out holds %llu bytes, the call may need %llu", (unsigned long long)out_capacity, (unsigned long long)need);
			return FB200_ERR_OUTPUT_TOO_SMALL;
		}
	}
	FB_CUDA(cudaSetDevice(device));
	std::map<uint32_t, Album> A;
	std::vector<std::vector<uint8_t>> regions;
	if((rc = analyse(dec, device, files, albums, nfiles, info, nullptr, &A, &regions, st)) != FB200_OK) return rc;
	if(opt->scan_only) return FB200_OK;

	// step 3: each album's files in list order; a chain write that fails stops its album
	std::vector<uint8_t> blob;
	std::vector<std::vector<uint8_t>> heads(nfiles);
	std::vector<uint8_t> written(nfiles, 0);
	for(auto &kv : A) {
		if(!kv.second.ok) continue;
		bool stopped = false;
		for(uint32_t i : kv.second.at) {
			fb200_add_replaygain_info &O = info[i];
			if(stopped) { fail(O, FB200_ADD_RG_NOT_WRITTEN, "an earlier file's chain write failed"); continue; }
			const float vals[4] = {O.rg.track_gain, O.rg.track_peak, O.rg.album_gain, O.rg.album_peak};
			uint64_t audio_in = 0;
			bool in_place = false;
			if(const char *why = rg_rewrite_head(regions[i].data(), regions[i].size(), vals, &heads[i], &audio_in, &in_place)) {
				fail(O, FB200_ADD_RG_METADATA, "%s", why);
				stopped = true;
				continue;
			}
			O.head_bytes = heads[i].size();
			O.audio_offset_in = audio_in;
			O.in_place = in_place ? 1 : 0;
			written[i] = 1;
		}
	}
	// output offsets in list order; the heads back to back in the blob, in the same order
	std::vector<SpliceSeg> segs;
	uint64_t off = 0, items = 0;
	for(uint32_t i = 0; i < nfiles; i++) {
		if(!written[i]) continue;
		fb200_add_replaygain_info &O = info[i];
		const std::vector<uint8_t> &head = heads[i];
		const DecoderFileSpan sp = decoder_file_span(dec, files[i]);
		const uint64_t audio = sp.end - sp.audio;
		O.offset = off;
		O.bytes = O.head_bytes + (whole ? audio : 0);
		if(whole) {
			segs.push_back(SpliceSeg{blob.size(), off, head.size(), items, 1, 0});
			items += (head.size() + kSpliceItem - 1) / kSpliceItem;
			if(audio) {
				segs.push_back(SpliceSeg{sp.audio, off + head.size(), audio, items, 0, 0});
				items += (audio + kSpliceItem - 1) / kSpliceItem;
			}
		}
		blob.insert(blob.end(), head.begin(), head.end());
		off += O.bytes;
	}
	if(off == 0) return FB200_OK;
	if(off > out_capacity) {  // the bound checked above holds; this keeps a miscount from writing past the caller's buffer
		set_error("the files take %llu bytes, out holds %llu", (unsigned long long)off, (unsigned long long)out_capacity);
		return FB200_ERR_OUTPUT_TOO_SMALL;
	}
	if(!whole) {
		// the heads are the output
		if(device_out) {
			FB_CUDA(cudaMemcpyAsync(out, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
			FB_CUDA(cudaStreamSynchronize(st));
		}
		else memcpy(out, blob.data(), blob.size());
		return FB200_OK;
	}
	const size_t o_segs = (blob.size() + 16 + 15) & ~(size_t)15, o_out = (o_segs + segs.size() * sizeof(SpliceSeg) + 15) & ~(size_t)15;
	uint8_t *d = nullptr;
	FB_CUDA(cudaMalloc(&d, device_out ? o_out : o_out + off));
	struct Free { uint8_t *p; ~Free() { cudaFree(p); } } hold{d};
	blob.resize(blob.size() + 16, 0);
	FB_CUDA(cudaMemcpyAsync(d, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
	FB_CUDA(cudaMemcpyAsync(d + o_segs, segs.data(), segs.size() * sizeof(SpliceSeg), cudaMemcpyHostToDevice, st));
	uint8_t *d_out = device_out ? out : d + o_out;
	k_files_splice<<<(unsigned)items, 256, 0, st>>>(decoder_files_view(dec).data, d, reinterpret_cast<const SpliceSeg *>(d + o_segs), (int)segs.size(), d_out);
	decoder_count_launches(dec, 1);
	FB_CUDA(cudaGetLastError());
	if(!device_out) FB_CUDA(cudaMemcpyAsync(out, d_out, off, cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	return FB200_OK;
}

}  // namespace

}  // namespace fb200

using namespace fb200;

int fb200_add_replaygain_flac_files_host(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles,
                                         const fb200_add_replaygain_options *opt, uint8_t *out, size_t out_capacity, fb200_add_replaygain_info *info)
{
	return add_replaygain(dec, false, files, albums, nfiles, opt, out, out_capacity, info, nullptr);
}

int fb200_add_replaygain_flac_files_device(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles,
                                           const fb200_add_replaygain_options *opt, uint8_t *d_out, size_t out_capacity,
                                           fb200_add_replaygain_info *info, void *cuda_stream)
{
	return add_replaygain(dec, true, files, albums, nfiles, opt, d_out, out_capacity, info, static_cast<cudaStream_t>(cuda_stream));
}

int fb200_replaygain_rewrite_head(const uint8_t *file, uint64_t nbytes, float track_gain, float track_peak, float album_gain, float album_peak,
                                  uint8_t *head, uint64_t head_capacity, uint64_t *head_bytes, uint64_t *audio_offset_in, uint32_t *in_place)
{
	if(!file || !head_bytes || !audio_offset_in || !in_place || (!head && head_capacity)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	const float v[4] = {track_gain, track_peak, album_gain, album_peak};
	std::vector<uint8_t> h;
	bool ip = false;
	if(const char *why = rg_rewrite_head(file, nbytes, v, &h, audio_offset_in, &ip)) { set_error("%s", why); return FB200_ERR_INVALID; }
	*head_bytes = h.size();
	*in_place = ip ? 1 : 0;
	if(h.size() > head_capacity) { set_error("the head is %zu bytes, room for %llu", h.size(), (unsigned long long)head_capacity); return FB200_ERR_OUTPUT_TOO_SMALL; }
	memcpy(head, h.data(), h.size());
	return FB200_OK;
}

int fb200_debug_add_replaygain_windows(fb200_decoder *dec, const uint32_t *files, const uint32_t *albums, uint32_t nfiles, double *windows,
                                       uint64_t capacity, uint64_t *nwindows)
{
	if(!dec || !files || !nwindows || (!windows && capacity)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	int device = 0, rc;
	if((rc = check_call(dec, files, nfiles, &device)) != FB200_OK) return rc;
	FB_CUDA(cudaSetDevice(device));
	std::vector<fb200_add_replaygain_info> info(nfiles);
	std::vector<double> w;
	std::map<uint32_t, Album> A;
	std::vector<std::vector<uint8_t>> regions;
	if((rc = analyse(dec, device, files, albums, nfiles, info.data(), &w, &A, &regions, nullptr)) != FB200_OK) return rc;
	*nwindows = w.size();
	if(w.size() > capacity) { set_error("%zu windows, room for %llu", w.size(), (unsigned long long)capacity); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if(!w.empty()) memcpy(windows, w.data(), w.size() * sizeof(double));
	return FB200_OK;
}
