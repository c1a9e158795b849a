// reencode.cu -- fb200_reencode_flac_files_*: files of the batch fb200_decode_files_index left resident, re-encoded into the .flac
// files the flac tool writes from FLAC input (src/flac/encode.c). The host builds each file's metadata list with the tool's policy
// for FLAC input (EncoderSession_init_encoder, :1710-1939) and checks it as the encoder would; the decoder then places every
// accepted frame straight into the encoder's compacted input (k_files_place_segs), the MD5 runs once over that copy, and the
// complete-file machinery of fb200_encode_flac_files_* encodes and writes the files that decoded cleanly.
#include <stdarg.h>
#include <string.h>

#include "fb200_internal.h"
#include "flac_metadata.h"
#include "flac_parse.h"

namespace fb200 {

namespace {

// One metadata block as it stands in the file: the 4-byte header (last flag cleared) and the body.
struct Block {
	uint32_t type;
	std::vector<uint8_t> bytes;
	uint32_t length() const { return (uint32_t)bytes.size() - 4; }
	const uint8_t *body() const { return bytes.data() + 4; }
};

// The blocks of a file's metadata region (an optional ID3v2 tag, "fLaC", the blocks), STREAMINFO first. The index call has
// parsed the same bytes, so this fails only on a region that is not that file's.
const char *input_blocks(const std::vector<uint8_t> &m, std::vector<Block> *out)
{
	const MetaRegion r = read_metadata_region(m.data(), m.size());
	if(r.end == MetaRegion::NO_MARKER) return "no fLaC marker";
	if(r.end == MetaRegion::SHORT) return "metadata runs past the file";
	for(const MetaBlock &h : r.blocks) {
		Block b{h.type, std::vector<uint8_t>(m.data() + h.body - 4, m.data() + h.body + h.length)};
		b.bytes[0] &= 0x7f;
		out->push_back(std::move(b));
	}
	if(out->empty() || out->front().type != 0) return "first metadata block is not STREAMINFO";  // get_sample_info_flac
	out->erase(out->begin());
	return nullptr;
}

// encode.c:1782-1795: a CUESHEET with tracks whose lead-out (the last track's offset) is not the input's length is dropped. A
// body too short to hold its tracks is kept, for the encoder's check to reject.
bool cuesheet_lead_out_wrong(const Block &b, uint64_t total)
{
	const uint8_t *p = b.body();
	const size_t n = b.length();
	if(n < 396) return false;
	const uint32_t ntracks = p[395];
	if(ntracks == 0) return false;
	size_t pos = 396, last = 0;
	for(uint32_t t = 0; t < ntracks; t++) {
		if(n - pos < 36) return false;
		last = pos;
		pos += 36 + 12 * (size_t)p[pos + 35];
		if(pos > n) return false;
	}
	return be64(p + last) != total;
}

// EncoderSession_init_encoder's list for a FLAC input (encode.c:1710-1939) into M; nullptr or why the list cannot be written
// around a single VORBIS_COMMENT (a second one, or one whose fields disagree with its length: the encoder rejects both).
// length is total_samples_to_encode (the input's total_samples, or the --skip / --until range's length); whole says it equals
// the input's total_samples, the one case an input SEEKTABLE can be kept in.
const char *flac_input_metadata(std::vector<Block> L, const fb200_flac_reencode_options &opt, const std::vector<std::string> &tags, uint32_t mask_tag,
                                uint64_t length, bool whole, uint32_t rate, FileMeta *M)
{
	const Block kNewVc{4, {}}, kNewSt{3, {}};  // markers: the VORBIS_COMMENT and SEEKTABLE this policy makes
	// VORBIS_COMMENT (:1730-1770): with tags, the input's go and their channel mask tag carries over
	bool vc_found = false;
	for(const Block &b : L) vc_found |= b.type == 4;
	if(!tags.empty()) {
		std::vector<Block> kept;
		for(Block &b : L)
			if(b.type != 4) kept.push_back(std::move(b));
		L.swap(kept);
	}
	if(!vc_found || !tags.empty()) {
		L.insert(L.begin(), kNewVc);
		M->ent = tags;
		if(!tags.empty() && mask_tag) set_channel_mask_tag(M->ent, mask_tag);
	}
	// CUESHEET (:1772-1822): the lead-out is compared with the length encoded; track offsets are not moved
	{
		std::vector<Block> kept;
		for(Block &b : L)
			if(!(b.type == 5 && cuesheet_lead_out_wrong(b, length))) kept.push_back(std::move(b));
		L.swap(kept);
	}
	// SEEKTABLE (:1824-1880): the input's goes with any -S or when the length changes; a template goes first with -S <n>s, or when
	// none is left
	bool st_found = false;
	for(const Block &b : L) st_found |= b.type == 3 && !b.bytes.empty();
	if(opt.seek_spacing_s >= 0 || !whole) {
		st_found = false;
		std::vector<Block> kept;
		for(Block &b : L)
			if(!(b.type == 3 && !b.bytes.empty())) kept.push_back(std::move(b));
		L.swap(kept);
	}
	if(opt.seek_spacing_s > 0 || (opt.seek_spacing_s < 0 && !st_found)) L.insert(L.begin(), kNewSt);
	// PADDING (:1882-1930): every input PADDING goes; their sum, -P or the default as one block at the end
	int64_t p = -1;
	{
		std::vector<Block> kept;
		for(Block &b : L) {
			if(b.type == 1) p = (p < 0 ? 0 : p) + b.length();
			else kept.push_back(std::move(b));
		}
		L.swap(kept);
	}
	if(opt.padding > 0) p = opt.padding;
	if(p < 0) p = length / rate < 20 * 60 ? 8192 : 65536;
	if(p > 0 && opt.replay_gain) p += 190;  // GRABBAG__REPLAYGAIN_MAX_TAG_SPACE_REQUIRED
	if(p > (1 << 24) - 1) p = (1 << 24) - 1;
	M->padding = opt.padding != 0 && p > 0 ? p : -1;
	// around the one VORBIS_COMMENT
	bool at_vc = false;
	for(const Block &b : L) {
		if(b.type == 4) {
			if(at_vc) return "a second VORBIS_COMMENT";
			at_vc = true;
			if(!b.bytes.empty() && vorbis_comment_exact(b.body(), b.length(), &M->ent)) return "VORBIS_COMMENT fields disagree with the block length";
			continue;
		}
		std::vector<uint8_t> &to = at_vc ? M->after : M->before;
		if(b.type == 3 && b.bytes.empty()) put_block(to, 3, seek_template(opt.seek_spacing_s > 0 ? opt.seek_spacing_s : 10, length, rate));
		else to.insert(to.end(), b.bytes.begin(), b.bytes.end());
	}
	return nullptr;
}

void fail(fb200_flac_reencode_info &I, uint32_t status, const char *fmt, ...)
{
	I.status = status;
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(I.error, sizeof I.error, fmt, ap);
	va_end(ap);
}

// What the encode's hooks share: the files it encodes (batch index, back-to-back first value, STREAMINFO MD5) and their verdicts.
// With ranges (fb200_reencode_flac_files_ranges_*), what is encoded is range[i] of file batch[i]: the ranged decode fills it and
// leaves its verdicts in errors / missing, and no input MD5 is compared (the tool zeroes it with --skip or --until, encode.c:1130).
struct Reencode {
	fb200_decoder *dec;
	std::vector<uint32_t> batch;
	std::vector<uint64_t> first_value;
	std::vector<uint32_t> status;  // FB200_REENCODE_* after check()
	RgRebuild *rg = nullptr;
	bool all_ok = true;            // every listed file passed the host plan
	bool ranged = false;
	std::vector<fb200_sample_range> range;
	std::vector<uint32_t> errors;
	std::vector<uint64_t> missing;
};

int reencode_fill(void *ctx, int32_t *pcm, unsigned long long values, const FileSeg *d_segs, cudaStream_t st)
{
	Reencode &R = *static_cast<Reencode *>(ctx);
	const uint32_t n = (uint32_t)R.batch.size();
	if(!R.ranged) return decoder_decode_into(R.dec, R.batch.data(), R.first_value.data(), n, pcm, values, d_segs, 2 * (int)n, st);
	R.errors.resize(n);
	R.missing.resize(n);
	return decoder_decode_ranges_into(R.dec, R.range.data(), R.first_value.data(), n, pcm, values, d_segs, 2 * (int)n, st, R.errors.data(), R.missing.data());
}

int reencode_check(void *ctx, const uint8_t *d_md5, cudaStream_t st, std::vector<uint8_t> *keep)
{
	Reencode &R = *static_cast<Reencode *>(ctx);
	const uint32_t n = (uint32_t)R.batch.size();
	std::vector<uint8_t> md5(16 * (size_t)n);
	if(!R.ranged) {
		R.errors.resize(n);
		R.missing.resize(n);
		FB_CUDA(cudaMemcpyAsync(md5.data(), d_md5, md5.size(), cudaMemcpyDeviceToHost, st));
		const int rc = decoder_decode_verdicts(R.dec, R.batch.data(), n, st, R.errors.data(), R.missing.data());
		if(rc != FB200_OK) return rc;
	}
	static const uint8_t zero[16] = {0};
	R.status.assign(n, FB200_REENCODE_OK);
	bool album = R.all_ok;
	for(uint32_t i = 0; i < n; i++) {
		const uint8_t *want = R.ranged ? zero : decoder_file_md5(R.dec, R.batch[i]);
		if(R.errors[i] || R.missing[i]) R.status[i] = FB200_REENCODE_DAMAGED;
		else if(memcmp(want, zero, 16) != 0 && memcmp(want, md5.data() + 16 * (size_t)i, 16) != 0) R.status[i] = FB200_REENCODE_MD5_MISMATCH;
		(*keep)[i] = R.status[i] == FB200_REENCODE_OK;
		album &= R.status[i] == FB200_REENCODE_OK;
	}
	if(R.rg) R.rg->album = album;
	return FB200_OK;
}

// files[0 .. nfiles) whole (flac -f *.flac), or with ranges (files NULL), ranges[0 .. nfiles) (flac -f --skip --until *.flac)
int reencode(fb200_encoder *e, fb200_decoder *dec, bool device, const uint32_t *files, const fb200_sample_range *ranges, uint32_t nfiles,
             const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *out, size_t out_capacity,
             uint64_t *frame_offsets, uint64_t *nframes, fb200_flac_reencode_info *info, void *cuda_stream)
{
	if(!e || !dec || (!files && !ranges) || !opt || !out || !nframes || !info) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	if(opt->reserved != 0) { set_error("fb200_flac_reencode_options.reserved must be 0"); return FB200_ERR_INVALID; }
	if(nfiles == 0 && !ranges) { set_error("no files"); return FB200_ERR_INVALID; }
	if(ranges && (nfiles == 0 || nfiles >= 0x80000000u)) { set_error("invalid number of ranges %u", nfiles); return FB200_ERR_INVALID; }
	if(!tags != !tag_offsets) { set_error("tags and tag_offsets must both be given or both be NULL"); return FB200_ERR_INVALID; }
	uint32_t nbatch = 0;
	int ddev = 0;
	if(!decoder_files(dec, &nbatch, &ddev)) { set_error("no batch of files is indexed"); return FB200_ERR_INVALID; }
	if(ddev != encoder_device(e)) { set_error("the decoder is on device %d, the encoder on %d", ddev, encoder_device(e)); return FB200_ERR_INVALID; }
	fb200_encoder_config cfg;
	fb200_encoder_get_config(e, &cfg);
	ReplayGainJob rg{0, 0, 0, {}, rg_rebuild, nullptr};
	if(opt->replay_gain) {
		// encode.c:1684-1692
		if(cfg.channels > 2) { set_error("%u channels; --replay-gain takes 1 or 2", cfg.channels); return FB200_ERR_INVALID; }
		if(!replaygain_rate(cfg.sample_rate, &rg.ds, &rg.W, &rg.filt)) { set_error("invalid sample rate %u for --replay-gain", cfg.sample_rate); return FB200_ERR_INVALID; }
	}
	std::vector<uint8_t> seen(nbatch, 0);
	for(uint32_t i = 0; i < nfiles; i++) {
		const uint32_t f = ranges ? ranges[i].file : files[i];
		if(ranges) {
			// the checks of fb200_decode_files_ranges_*; a range past total_samples is the tool's "--until value is after end of input"
			const fb200_sample_range &q = ranges[i];
			if(f >= nbatch) { set_error("range %u: file %u of a batch of %u", i, f, nbatch); return FB200_ERR_INVALID; }
			if(q.samples == 0) { set_error("range %u is empty", i); return FB200_ERR_INVALID; }
			if(q.first_sample + q.samples < q.first_sample) { set_error("range %u: first_sample + samples overflows", i); return FB200_ERR_INVALID; }
			const fb200_file_decode_info &I = decoder_file_info(dec, f);
			if(I.status == FB200_FILE_OK && I.total_samples && q.first_sample + q.samples > I.total_samples) {
				set_error("range %u: samples [%llu, %llu) of file %u, which has %llu", i, (unsigned long long)q.first_sample,
				          (unsigned long long)(q.first_sample + q.samples), f, (unsigned long long)I.total_samples);
				return FB200_ERR_INVALID;
			}
		}
		else {
			if(f >= nbatch) { set_error("files[%u] = %u, the batch has %u files", i, f, nbatch); return FB200_ERR_INVALID; }
			if(seen[f]) { set_error("file %u is listed twice", f); return FB200_ERR_INVALID; }
			seen[f] = 1;
		}
		const fb200_file_decode_info &I = decoder_file_info(dec, f);
		if(I.status == FB200_FILE_OK && (I.channels != cfg.channels || I.bits_per_sample != cfg.bits_per_sample || I.sample_rate != cfg.sample_rate)) {
			set_error("file %u is %u ch / %u bits / %u Hz, the encoder %u / %u / %u", f, I.channels, I.bits_per_sample, I.sample_rate, cfg.channels,
			          cfg.bits_per_sample, cfg.sample_rate);
			return FB200_ERR_INVALID;
		}
		if(I.status == FB200_FILE_OK && opt->replay_gain && rg.ds > 1 && (I.min_blocksize != I.max_blocksize || I.max_blocksize % rg.ds)) {
			set_error("file %u: blocksizes %u-%u at %u Hz; --replay-gain above 48 kHz needs one fixed blocksize that is a multiple of %u", f, I.min_blocksize,
			          I.max_blocksize, I.sample_rate, rg.ds);
			return FB200_ERR_INVALID;
		}
		if(tags && (tag_offsets[i + 1] < tag_offsets[i] || (tag_offsets[i + 1] > tag_offsets[i] && tags[tag_offsets[i + 1] - 1] != 0))) {
			set_error("tags of file %u do not end in a NUL", i);
			return FB200_ERR_INVALID;
		}
	}

	// ---- the host plan: each file's list, checked as the encoder checks it
	Reencode R;
	R.dec = dec;
	R.ranged = ranges != nullptr;
	RgRebuild rgr;
	if(opt->replay_gain) {
		R.rg = &rgr;
		rg.ctx = &rgr;
	}
	std::vector<uint32_t> listed;  // encoded file -> its place in files[]
	std::vector<uint64_t> samples, moffs(1, 0);
	std::vector<uint8_t> meta, region;
	uint32_t region_of = ~0u;
	uint64_t values = 0;
	for(uint32_t i = 0; i < nfiles; i++) {
		fb200_flac_reencode_info &O = info[i];
		memset(&O, 0, sizeof O);
		const uint32_t f = ranges ? ranges[i].file : files[i];
		const fb200_file_decode_info &I = decoder_file_info(dec, f);
		if(I.status != FB200_FILE_OK) { fail(O, FB200_REENCODE_INPUT, "index status %u", I.status); continue; }
		if(I.total_samples == 0) { fail(O, FB200_REENCODE_NO_TOTAL, "STREAMINFO has unknown total samples"); continue; }
		const uint64_t length = ranges ? ranges[i].samples : I.samples;
		int rc;
		if(region_of != f) {  // consecutive ranges of one file read its metadata once
			if((rc = decoder_file_metadata(dec, f, &region)) != FB200_OK) return rc;
			region_of = f;
		}
		if(region.size() >= 3 && memcmp(region.data(), "ID3", 3) == 0) { fail(O, FB200_REENCODE_INPUT, "input file has an ID3v2 tag"); continue; }  // main.c:1524
		std::vector<Block> blocks;
		std::vector<std::string> ent;
		if(tags) {
			const char *t = reinterpret_cast<const char *>(tags) + tag_offsets[i];
			const size_t len = (size_t)(tag_offsets[i + 1] - tag_offsets[i]);
			for(size_t p = 0; p < len;) {
				const size_t k = strnlen(t + p, len - p);
				ent.emplace_back(t + p, k);
				p += k + 1;
			}
		}
		FileMeta M;
		const char *why = input_blocks(region, &blocks);
		if(!why) why = flac_input_metadata(std::move(blocks), *opt, ent, decoder_file_mask(dec, f), length, length == I.total_samples, I.sample_rate, &M);
		if(why) { fail(O, FB200_REENCODE_METADATA, "%s", why); continue; }
		std::vector<uint8_t> one;
		put_file_metadata(M, one);
		const uint64_t one_offs[2] = {0, one.size()};
		one.push_back(0);
		FlacHeaderPlan plan;
		if(plan_flac_headers(one.data(), one_offs, 1, &plan) != FB200_OK) { fail(O, FB200_REENCODE_METADATA, "%s", get_error()); continue; }
		meta.insert(meta.end(), one.begin(), one.end() - 1);
		moffs.push_back(meta.size());
		listed.push_back(i);
		R.batch.push_back(f);
		if(ranges) R.range.push_back(ranges[i]);
		R.first_value.push_back(values);
		samples.push_back(length);
		values += length * I.channels;
		if(opt->replay_gain) {
			rg.bps.push_back(I.bits_per_sample);
			rgr.files.push_back(std::move(M));
		}
	}
	R.all_ok = listed.size() == nfiles;
	*nframes = 0;
	if(listed.empty()) {
		if(!device && frame_offsets) frame_offsets[0] = 0;
		return FB200_OK;
	}
	meta.push_back(0);

	// ---- decode, MD5, verdicts and encode
	PcmSource src;
	src.data = reinterpret_cast<const uint8_t *>(info);  // not read: fill() provides the samples
	src.bytes = 0;
	src.rg = opt->replay_gain ? &rg : nullptr;
	src.fill = reencode_fill;
	src.check = reencode_check;
	src.ctx = &R;
	std::vector<fb200_flac_file_info> fi(listed.size());
	const int rc = encode_pcm_files_impl(e, src, device, samples.data(), (uint32_t)listed.size(), 1, meta.data(), moffs.data(), out, out_capacity,
	                                     frame_offsets, nframes, fi.data(), cuda_stream);
	if(rc != FB200_OK && rc != FB200_ERR_VERIFY) return rc;
	for(size_t k = 0; k < listed.size(); k++) {
		fb200_flac_reencode_info &O = info[listed[k]];
		if(R.status[k] == FB200_REENCODE_DAMAGED) fail(O, FB200_REENCODE_DAMAGED, "a decode error: a damaged frame, lost sync or missing samples");
		else if(R.status[k] == FB200_REENCODE_MD5_MISMATCH) fail(O, FB200_REENCODE_MD5_MISMATCH, "MD5 of the decoded samples differs from STREAMINFO's");
		else O.file = fi[k];
	}
	encoder_spread_verify(e, listed, nfiles);
	if(rc == FB200_ERR_VERIFY) {
		// the encoder's message counts the encoded files; name the failing file by its place in files[]
		std::vector<fb200_file_verify_info> v(nfiles);
		fb200_encoder_get_verify(e, v.data(), nfiles);
		uint32_t nbad = 0, first = 0;
		for(uint32_t i = nfiles; i-- > 0;)
			if(v[i].status != FB200_VERIFY_OK) { nbad++; first = i; }
		if(ranges)
			set_error("%u range(s) failed verification; the first, range %u of file %u: %s in frame %u", nbad, first, ranges[first].file,
			          v[first].status == FB200_VERIFY_MISMATCH ? "sample mismatch" : "decoder error", v[first].frame_number);
		else
			set_error("%u file(s) failed verification; the first, files[%u] = %u: %s in frame %u", nbad, first, files[first],
			          v[first].status == FB200_VERIFY_MISMATCH ? "sample mismatch" : "decoder error", v[first].frame_number);
	}
	return rc;
}

}  // namespace

}  // namespace fb200

using namespace fb200;

int fb200_reencode_flac_files_host(fb200_encoder *e, fb200_decoder *dec, const uint32_t *files, uint32_t nfiles, const fb200_flac_reencode_options *opt,
                                   const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *out, size_t out_capacity, uint64_t *frame_offsets,
                                   uint64_t *nframes, fb200_flac_reencode_info *info)
{
	if(!files) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	return reencode(e, dec, false, files, nullptr, nfiles, opt, tags, tag_offsets, out, out_capacity, frame_offsets, nframes, info, nullptr);
}

int fb200_reencode_flac_files_device(fb200_encoder *e, fb200_decoder *dec, const uint32_t *files, uint32_t nfiles, const fb200_flac_reencode_options *opt,
                                     const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *d_out, size_t out_capacity, uint64_t *d_frame_offsets,
                                     uint64_t *nframes, fb200_flac_reencode_info *info, void *cuda_stream)
{
	if(!files) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	return reencode(e, dec, true, files, nullptr, nfiles, opt, tags, tag_offsets, d_out, out_capacity, d_frame_offsets, nframes, info, cuda_stream);
}

int fb200_reencode_flac_files_ranges_host(fb200_encoder *e, fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                          const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *out,
                                          size_t out_capacity, uint64_t *frame_offsets, uint64_t *nframes, fb200_flac_reencode_info *info)
{
	if(!ranges) { set_error("ranges is NULL"); return FB200_ERR_INVALID; }
	return reencode(e, dec, false, nullptr, ranges, nranges, opt, tags, tag_offsets, out, out_capacity, frame_offsets, nframes, info, nullptr);
}

int fb200_reencode_flac_files_ranges_device(fb200_encoder *e, fb200_decoder *dec, const fb200_sample_range *ranges, uint32_t nranges,
                                            const fb200_flac_reencode_options *opt, const uint8_t *tags, const uint64_t *tag_offsets, uint8_t *d_out,
                                            size_t out_capacity, uint64_t *d_frame_offsets, uint64_t *nframes, fb200_flac_reencode_info *info,
                                            void *cuda_stream)
{
	if(!ranges) { set_error("ranges is NULL"); return FB200_ERR_INVALID; }
	return reencode(e, dec, true, nullptr, ranges, nranges, opt, tags, tag_offsets, d_out, out_capacity, d_frame_offsets, nframes, info, cuda_stream);
}
