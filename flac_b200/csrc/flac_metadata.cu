// flac_metadata.cu -- the host half of fb200_encode_flac_files_*: every file's client metadata blocks are checked as
// init_stream_internal_ checks a set_metadata list (stream_encoder.c:869-920) and serialised as FLAC__add_metadata_block writes
// them (stream_encoder_framing.c:47-243), into one header blob per call. The STREAMINFO body and the SEEKTABLE body are left
// for k_flac_file_headers, which knows the frame sizes, the MD5 and where each frame landed.
// It also holds the other host writers of metadata blocks: the lists the batch encoders build for WAV / AIFF and FLAC input, the
// padding rule of the metadata chain, and the ReplayGain tag edits of flac --replay-gain and metaflac --add-replay-gain.
#include <locale.h>
#include <string.h>
#include <strings.h>

#include "flac_metadata.h"
#include "flac_parse.h"

extern "C" const char *FLAC__VENDOR_STRING;

namespace fb200 {

namespace {

constexpr unsigned long long kPlaceholder = ~0ull;  // FLAC__STREAM_METADATA_SEEKPOINT_PLACEHOLDER

// utf8len_ (format.c:322-360) over a bounded string: bytes past the end read as the terminating NUL
uint32_t utf8len(const uint8_t *s, size_t n, size_t i)
{
	auto b = [&](size_t k) -> uint32_t { return i + k < n ? s[i + k] : 0u; };
	if((b(0) & 0x80) == 0) return 1;
	if((b(0) & 0xE0) == 0xC0 && (b(1) & 0xC0) == 0x80) return (b(0) & 0xFE) == 0xC0 ? 0 : 2;
	if((b(0) & 0xF0) == 0xE0 && (b(1) & 0xC0) == 0x80 && (b(2) & 0xC0) == 0x80) {
		if(b(0) == 0xE0 && (b(1) & 0xE0) == 0x80) return 0;
		if(b(0) == 0xED && (b(1) & 0xE0) == 0xA0) return 0;
		if(b(0) == 0xEF && b(1) == 0xBF && (b(2) & 0xFE) == 0xBE) return 0;
		return 3;
	}
	if((b(0) & 0xF8) == 0xF0 && (b(1) & 0xC0) == 0x80 && (b(2) & 0xC0) == 0x80 && (b(3) & 0xC0) == 0x80)
		return (b(0) == 0xF0 && (b(1) & 0xF0) == 0x80) ? 0 : 4;
	if((b(0) & 0xFC) == 0xF8 && (b(1) & 0xC0) == 0x80 && (b(2) & 0xC0) == 0x80 && (b(3) & 0xC0) == 0x80 && (b(4) & 0xC0) == 0x80)
		return (b(0) == 0xF8 && (b(1) & 0xF8) == 0x80) ? 0 : 5;
	if((b(0) & 0xFE) == 0xFC && (b(1) & 0xC0) == 0x80 && (b(2) & 0xC0) == 0x80 && (b(3) & 0xC0) == 0x80 && (b(4) & 0xC0) == 0x80 &&
	   (b(5) & 0xC0) == 0x80)
		return (b(0) == 0xFC && (b(1) & 0xFC) == 0x80) ? 0 : 6;
	return 0;
}

// A CUESHEET body: its length must be exactly what its fields say; the rules of FLAC__format_cuesheet_is_legal (format.c:422-498)
// with the CD-DA subset checked when is_cd is set, as the encoder calls it. Returns the violated rule, or nullptr.
const char *check_cuesheet(const uint8_t *b, uint32_t len)
{
	if(len < 396) return "CUESHEET shorter than its fixed fields";
	const unsigned long long lead_in = be64(b + 128);
	const bool is_cd = (b[136] & 0x80) != 0;
	const uint32_t ntracks = b[395];
	if(is_cd && lead_in < 2 * 44100) return "CD-DA cue sheet lead-in shorter than 2 seconds";
	if(is_cd && lead_in % 588) return "CD-DA cue sheet lead-in not a multiple of 588 samples";
	if(ntracks == 0) return "cue sheet without tracks";
	size_t p = 396;
	for(uint32_t t = 0; t < ntracks; t++) {
		if(p + 36 > len) return "CUESHEET track runs past the block";
		const unsigned long long off = be64(b + p);
		const uint32_t number = b[p + 8], nidx = b[p + 35];
		if(number == 0) return "cue sheet track number 0";
		if(is_cd && !((number >= 1 && number <= 99) || number == 170)) return "CD-DA cue sheet track number not 1-99 or 170";
		if(is_cd && off % 588) return "CD-DA cue sheet track offset not a multiple of 588 samples";
		if(t + 1 == ntracks && is_cd && number != 170) return "CD-DA cue sheet lead-out track number not 170";
		p += 36;
		if(p + 12ull * nidx > len) return "CUESHEET index runs past the block";
		if(t + 1 < ntracks) {
			if(nidx == 0) return "cue sheet track without index points";
			if(b[p + 8] > 1) return "cue sheet track's first index number not 0 or 1";
		}
		for(uint32_t k = 0; k < nidx; k++) {
			if(is_cd && be64(b + p + 12 * k) % 588) return "CD-DA cue sheet index offset not a multiple of 588 samples";
			if(k > 0 && (uint32_t)b[p + 12 * k + 8] != (uint32_t)b[p + 12 * (k - 1) + 8] + 1) return "cue sheet index numbers do not increase by 1";
		}
		p += 12ull * nidx;
	}
	if(p != len) return "CUESHEET length differs from its fields";
	return nullptr;
}

}  // namespace

int plan_flac_headers(const uint8_t *metadata, const uint64_t *metadata_offsets, uint32_t nfiles, FlacHeaderPlan *plan)
{
	const uint32_t vlen = (uint32_t)strlen(FLAC__VENDOR_STRING);
	plan->heads.assign(nfiles, FlacHead{});
	plan->blob.clear();
	plan->pts.clear();
	for(uint32_t f = 0; metadata && f < nfiles; f++)
		if(metadata_offsets[f + 1] < metadata_offsets[f]) { set_error("file %u: metadata offsets decrease", f); return FB200_ERR_INVALID; }
	// every file's header is at most its blocks, "fLaC" + STREAMINFO and a VORBIS_COMMENT's vendor string and fixed fields
	plan->blob.reserve((metadata ? metadata_offsets[nfiles] - metadata_offsets[0] : 0) + (size_t)nfiles * (42 + 12 + vlen));
	for(uint32_t f = 0; f < nfiles; f++) {
		const uint8_t *m = metadata ? metadata + metadata_offsets[f] : nullptr;
		const uint64_t mlen = metadata ? metadata_offsets[f + 1] - metadata_offsets[f] : 0;
		// the blocks: (type, body, length)
		struct Blk { uint32_t type, len; const uint8_t *body; };
		std::vector<Blk> blks;
		bool has_st = false, has_vc = false, icon1 = false, icon2 = false;
		for(uint64_t p = 0; p < mlen;) {
			const uint32_t i = (uint32_t)blks.size();
			auto bad = [&](const char *why) { set_error("file %u, metadata block %u: %s", f, i, why); return FB200_ERR_INVALID; };
			if(p + 4 > mlen) return bad("block header runs past the file's metadata");
			const uint32_t type = m[p] & 0x7f, len = be(m + p + 1, 3);
			const uint8_t *b = m + p + 4;
			if(p + 4 + len > mlen) return bad("block runs past the file's metadata");
			p += 4 + len;
			switch(type) {
				case 0: return bad("a STREAMINFO block (the encoder writes its own)");
				case 127: return bad("type 127 is invalid");
				case 2: if(len < 4) return bad("APPLICATION shorter than its 4-byte id"); break;
				case 3: {
					if(has_st) return bad("a second SEEKTABLE");
					has_st = true;
					if(len % 18) return bad("SEEKTABLE length not a multiple of 18");
					unsigned long long prev = 0;
					for(uint32_t k = 0; k < len / 18; k++) {  // FLAC__format_seektable_is_legal (format.c:242-266)
						const unsigned long long s = be64(b + 18 * k);
						if(k > 0 && s != kPlaceholder && s <= prev) return bad("illegal seek table: points not ascending");
						prev = s;
					}
					break;
				}
				case 4: {
					if(has_vc) return bad("a second VORBIS_COMMENT");
					has_vc = true;
					if(const char *why = vorbis_comment_exact(b, len, nullptr)) return bad(why);
					if(len - le32(b) + vlen >= (1u << 24)) return bad("VORBIS_COMMENT too long with this library's vendor string");
					break;
				}
				case 5: {
					const char *why = check_cuesheet(b, len);
					if(why) return bad(why);
					break;
				}
				case 6: {
					if(len < 32) return bad("PICTURE shorter than its fixed fields");
					const uint32_t ptype = be(b, 4), ml = be(b + 4, 4);
					if(8ull + ml + 4 > len) return bad("PICTURE MIME type runs past the block");
					const uint8_t *mime = b + 8;
					const uint32_t dl = be(b + 8 + ml, 4);
					if(12ull + ml + dl + 20 > len) return bad("PICTURE description runs past the block");
					const uint8_t *desc = b + 12 + ml;
					const uint32_t w = be(desc + dl, 4), h = be(desc + dl + 4, 4), n = be(desc + dl + 16, 4);
					if(32ull + ml + dl + n != len) return bad("PICTURE length differs from its fields");
					// FLAC__format_picture_is_legal (format.c:501-524); a NUL would end the reference's C strings early
					for(uint32_t k = 0; k < ml; k++)
						if(mime[k] < 0x20 || mime[k] > 0x7e) return bad("PICTURE MIME type not printable ASCII");
					for(uint32_t k = 0; k < dl;) {
						const uint32_t u = desc[k] ? utf8len(desc, dl, k) : 0;
						if(u == 0) return bad("PICTURE description not valid UTF-8");
						k += u;
					}
					if(ptype == 1) {  // FLAC__STREAM_METADATA_PICTURE_TYPE_FILE_ICON_STANDARD (stream_encoder.c:899-913)
						if(icon1) return bad("a second 32x32 file icon (picture type 1)");
						icon1 = true;
						const bool png = (ml == 9 && !memcmp(mime, "image/png", 9)) || (ml == 3 && !memcmp(mime, "-->", 3));
						if(!png || w != 32 || h != 32) return bad("picture type 1 is not a 32x32 PNG");
					}
					else if(ptype == 2) {
						if(icon2) return bad("a second file icon (picture type 2)");
						icon2 = true;
					}
					break;
				}
				default: break;
			}
			blks.push_back(Blk{type, len, b});
		}

		// ---- the header: "fLaC", STREAMINFO (body by the device), [empty VORBIS_COMMENT], the client blocks (stream_encoder.c:1336-1428)
		FlacHead &H = plan->heads[f];
		std::vector<uint8_t> &o = plan->blob;
		const size_t h0 = o.size();
		H.blob = h0;
		o.insert(o.end(), {'f', 'L', 'a', 'C'});
		put_block_header(o, false, 0, 34);
		o.insert(o.end(), 34, 0);
		if(!has_vc) {
			put_block_header(o, blks.empty(), 4, 8 + vlen);
			put_vorbis_comment(o, FLAC__VENDOR_STRING, {});
		}
		for(size_t i = 0; i < blks.size(); i++) {
			const Blk &B = blks[i];
			const bool last = i + 1 == blks.size();
			const size_t body = o.size() + 4;
			switch(B.type) {
				case 1:  // PADDING: zeros, whatever the caller passed (stream_encoder_framing.c:97-100)
					put_block_header(o, last, 1, B.len);
					o.insert(o.end(), B.len, 0);
					break;
				case 3:  // SEEKTABLE: the template's points; the body is written by the device once the frames are placed
					put_block_header(o, last, 3, B.len);
					o.insert(o.end(), B.len, 0);
					H.st_body = (uint32_t)(body - h0);
					H.npts = B.len / 18;
					H.pts = plan->pts.size();
					for(uint32_t k = 0; k < H.npts; k++)
						plan->pts.push_back(SeekPt{be64(B.body + 18 * k), be64(B.body + 18 * k + 8), be(B.body + 18 * k + 16, 2), 0});
					break;
				case 4: {  // VORBIS_COMMENT: this library's vendor string (stream_encoder_framing.c:66-77, 118-133)
					const uint32_t old = le32(B.body);
					put_block_header(o, last, 4, B.len - old + vlen);
					put_le32(o, vlen);
					o.insert(o.end(), FLAC__VENDOR_STRING, FLAC__VENDOR_STRING + vlen);
					o.insert(o.end(), B.body + 4 + old, B.body + B.len);
					break;
				}
				case 5: {  // CUESHEET: reserved fields as zeros (stream_encoder_framing.c:162-191)
					put_block_header(o, last, 5, B.len);
					o.insert(o.end(), B.body, B.body + B.len);
					cuesheet_zero_reserved(o.data() + o.size() - B.len, B.len);  // check_cuesheet has passed: the walk is whole
					break;
				}
				default:  // APPLICATION, PICTURE and unknown types: their fields re-serialise to the same bytes
					put_block_header(o, last, B.type, B.len);
					o.insert(o.end(), B.body, B.body + B.len);
					break;
			}
		}
		const size_t hb = o.size() - h0;
		if(hb >= (1ull << 31)) { set_error("file %u: metadata too large", f); return FB200_ERR_INVALID; }
		H.bytes = (uint32_t)hb;
	}
	return FB200_OK;
}

void put_block_header(std::vector<uint8_t> &o, bool last, uint32_t type, uint32_t length)
{
	o.push_back((uint8_t)((last ? 0x80 : 0) | type));
	o.push_back((uint8_t)(length >> 16));
	o.push_back((uint8_t)(length >> 8));
	o.push_back((uint8_t)length);
}

void put_vorbis_comment(std::vector<uint8_t> &o, const std::string &vendor, const std::vector<std::string> &ent)
{
	put_le32(o, (uint32_t)vendor.size());
	o.insert(o.end(), vendor.begin(), vendor.end());
	put_le32(o, (uint32_t)ent.size());
	for(const std::string &s : ent) {
		put_le32(o, (uint32_t)s.size());
		o.insert(o.end(), s.begin(), s.end());
	}
}

void put_block(std::vector<uint8_t> &m, uint32_t type, const std::vector<uint8_t> &body)
{
	put_block_header(m, false, type, (uint32_t)body.size());
	m.insert(m.end(), body.begin(), body.end());
}

std::vector<uint8_t> seek_template(int32_t spacing_s, uint64_t samples, uint32_t sample_rate)
{
	std::vector<uint8_t> st;
	if(spacing_s <= 0 || samples == 0) return st;
	// grabbag__seektable_convert_specification_to_template "<n>s;" (seektable.c) + append_spaced_points_by_samples
	// (metadata_object.c:1126-1162)
	uint32_t spacing = (uint32_t)((double)spacing_s * (double)sample_rate);
	if(spacing < sample_rate / 2) spacing = sample_rate / 2;
	if(spacing > 0) {
		uint64_t num = 1 + samples / spacing;
		if(samples % spacing == 0) num--;
		if(num > 32768) {
			num = 32768;
			spacing = (uint32_t)(samples / num);
		}
		st.assign(18 * num, 0);
		for(uint64_t j = 0; j < num; j++) {
			const uint64_t s = j * spacing;
			for(int b = 0; b < 8; b++) st[18 * j + b] = (uint8_t)(s >> (56 - 8 * b));
		}
	}
	return st;
}

void set_channel_mask_tag(std::vector<std::string> &ent, uint32_t mask)
{
	// flac__utils_set_channel_mask_tag: FLAC__metadata_object_vorbiscomment_replace_comment(all=true) -- the first entry of that
	// name takes the new value, later ones go; none: appended
	static const char kName[] = "WAVEFORMATEXTENSIBLE_CHANNEL_MASK";
	char tag[128];
	snprintf(tag, sizeof tag, "%s=0x%04X", kName, mask);
	bool done = false;
	std::vector<std::string> kept;
	for(auto &s : ent) {
		if(!vorbis_entry_matches(s.data(), s.size(), kName)) kept.push_back(s);
		else if(!done) { kept.push_back(tag); done = true; }
	}
	if(!done) kept.push_back(tag);
	ent.swap(kept);
}

void put_file_metadata(const FileMeta &M, std::vector<uint8_t> &m)
{
	m.insert(m.end(), M.before.begin(), M.before.end());
	std::vector<uint8_t> vc;
	put_vorbis_comment(vc, "", M.ent);  // vendor: the encoder writes its own
	put_block(m, 4, vc);
	m.insert(m.end(), M.after.begin(), M.after.end());
	if(M.padding >= 0) put_block(m, 1, std::vector<uint8_t>((size_t)M.padding, 0));
}

int64_t chain_padding(int64_t initial, int64_t current, int64_t padding)
{
	if(current < initial && padding >= 0) return padding + initial - current;  // shrank: the trailing PADDING takes up the room
	if(current + 4 <= initial) return initial - 4 - current;                    // shrank by a block header or more: a new PADDING
	if(current > initial && padding >= 0) {                                     // grew: use up or trim the PADDING when it covers the growth
		const int64_t delta = current - initial;
		if(padding + 4 == delta) return -1;
		if(padding >= delta) return padding - delta;
	}
	return padding;
}

// ---- ReplayGain tags (grabbag/replaygain.c:353-500)

const char *const kRgName[5] = {"REPLAYGAIN_REFERENCE_LOUDNESS", "REPLAYGAIN_TRACK_GAIN", "REPLAYGAIN_TRACK_PEAK", "REPLAYGAIN_ALBUM_GAIN",
                                "REPLAYGAIN_ALBUM_PEAK"};

namespace {

// FLAC__metadata_object_vorbiscomment_remove_entries_matching
void vorbis_remove_matching(std::vector<std::string> &ent, const char *name)
{
	std::vector<std::string> kept;
	for(auto &s : ent)
		if(!vorbis_entry_matches(s.data(), s.size(), name)) kept.push_back(s);
	ent.swap(kept);
}

// append_tag_: "name=value" printed with fmt in the C locale
std::string rg_tag(const char *fmt, const char *name, float value)
{
	static const locale_t c_locale = newlocale(LC_ALL_MASK, "C", (locale_t)0);
	const locale_t old = uselocale(c_locale);
	char buf[256];
	snprintf(buf, sizeof buf, fmt, name, (double)value);
	uselocale(old);
	return buf;
}

// the bytes --replay-gain's edits can change: the VORBIS_COMMENT block and the PADDING block, headers included (the other blocks
// keep theirs)
int64_t edited_length(const FileMeta &M)
{
	int64_t n = 4 + 8;
	for(auto &s : M.ent) n += 4 + (int64_t)s.size();
	return n + (M.padding >= 0 ? 4 + M.padding : 0);
}

// One of flac --replay-gain's metadata writes: the edit, then the blocks laid out as the chain write lays them out. The only
// PADDING block is the last block here, so FLAC__metadata_chain_sort_padding leaves the list as it is. (A FLAC input's list ends
// in its one PADDING block too, when it has one.)
void rg_write(FileMeta &M, RgField edit, float gain, float peak)
{
	const int64_t initial = edited_length(M);
	rg_edit(M.ent, edit, gain, peak);
	M.padding = chain_padding(initial, edited_length(M), M.padding);
	if(M.padding > (1 << 24) - 1) M.padding = (1 << 24) - 1;
}

}  // namespace

void rg_edit(std::vector<std::string> &ent, RgField edit, float gain, float peak)
{
	static const char *const kFormat[5] = {"%s=%2.1f dB", "%s=%+2.2f dB", "%s=%1.8f", "%s=%+2.2f dB", "%s=%1.8f"};
	const int n = edit == RG_REFERENCE ? 1 : 2;
	const float value[2] = {edit == RG_REFERENCE ? 89.0f : gain, peak};
	for(int i = 0; i < n; i++) vorbis_remove_matching(ent, kRgName[edit + i]);
	for(int i = 0; i < n; i++) ent.push_back(rg_tag(kFormat[edit + i], kRgName[edit + i], value[i]));
}

int rg_rebuild(void *ctx, const fb200_replaygain_info *info, std::vector<uint8_t> *meta, std::vector<uint64_t> *moffs)
{
	const RgRebuild &R = *static_cast<const RgRebuild *>(ctx);
	moffs->assign(1, 0);
	for(size_t f = 0; f < R.files.size(); f++) {
		FileMeta M = R.files[f];
		const fb200_replaygain_info &I = info[f];
		// after each file's encode, the reference and the track tags (main.c:1775-1785); after every file's, the album tags (:575-590)
		rg_write(M, RG_REFERENCE, 0.f, 0.f);
		rg_write(M, RG_TRACK_GAIN, I.track_gain, I.track_peak);
		if(R.album) rg_write(M, RG_ALBUM_GAIN, I.album_gain, I.album_peak);
		put_file_metadata(M, *meta);
		moffs->push_back(meta->size());
	}
	meta->push_back(0);
	return FB200_OK;
}

}  // namespace fb200
