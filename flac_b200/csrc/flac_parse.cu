// flac_parse.cu -- host-side parsing of .flac containers (flac_parse.h). No device code.
#include <stdio.h>
#include <string.h>
#include <strings.h>

#include <string>

#include "flac_parse.h"

namespace fb200 {

void get_streaminfo(const uint8_t *b, FLAC__StreamMetadata_StreamInfo &s)
{
	s.min_blocksize = (b[0] << 8) | b[1]; s.max_blocksize = (b[2] << 8) | b[3];
	s.min_framesize = (b[4] << 16) | (b[5] << 8) | b[6]; s.max_framesize = (b[7] << 16) | (b[8] << 8) | b[9];
	uint64_t packed = 0;
	for(int i = 0; i < 8; i++) packed = (packed << 8) | b[10 + i];
	s.sample_rate = (uint32_t)(packed >> 44); s.channels = (uint32_t)((packed >> 41) & 7) + 1; s.bits_per_sample = (uint32_t)((packed >> 36) & 31) + 1;
	s.total_samples = packed & 0xFFFFFFFFFull;
	memcpy(s.md5sum, b + 18, 16);
}

size_t id3v2_tag_bytes(const uint8_t *h)
{
	return 10 + (((size_t)h[6] & 0x7f) << 21 | ((size_t)h[7] & 0x7f) << 14 | ((size_t)h[8] & 0x7f) << 7 | ((size_t)h[9] & 0x7f));
}

MetaBlockHeader metadata_block_header(const uint8_t *h)
{
	MetaBlockHeader m;
	m.last = (h[0] & 0x80) != 0;
	m.type = h[0] & 0x7f;
	m.length = be(h + 1, 3);
	return m;
}

MetaRegion read_metadata_region(const uint8_t *p, size_t n)
{
	MetaRegion r{MetaRegion::NO_MARKER, 0, 0, {}};
	size_t pos = 0;
	// optional ID3v2 tag, then "fLaC" (stream_decoder.c:1654-1742)
	if(n >= 10 && memcmp(p, "ID3", 3) == 0) pos = id3v2_tag_bytes(p);
	if(pos > n || n - pos < 4 || memcmp(p + pos, "fLaC", 4) != 0) return r;
	r.end = MetaRegion::SHORT;
	r.marker = pos;
	pos += 4;
	for(bool last = false; !last;) {
		if(n - pos < 4) return r;
		const MetaBlockHeader h = metadata_block_header(p + pos);
		if(n - pos - 4 < h.length) return r;
		r.blocks.push_back(MetaBlock{h, pos + 4});
		last = h.last;
		pos += 4 + (size_t)h.length;
	}
	r.end = MetaRegion::OK;
	r.audio = pos;
	return r;
}

bool walk_metadata(const uint8_t *p, size_t n, FLAC__StreamMetadata_StreamInfo &si, bool *has_streaminfo, uint32_t *streaminfo_length,
                   size_t *audio_offset)
{
	*has_streaminfo = false;
	*streaminfo_length = 0;
	const MetaRegion r = read_metadata_region(p, n);
	if(r.end != MetaRegion::OK) return false;
	for(const MetaBlock &b : r.blocks)
		if(b.type == FLAC__METADATA_TYPE_STREAMINFO && b.length >= 34 && !*has_streaminfo) {
			get_streaminfo(p + b.body, si);
			*has_streaminfo = true;
			*streaminfo_length = b.length;
		}
	*audio_offset = r.audio;
	return true;
}

bool vorbis_entry_matches(const char *entry, size_t len, const char *name)
{
	const size_t k = strlen(name);
	const char *eq = static_cast<const char *>(memchr(entry, '=', len));
	return eq && (size_t)(eq - entry) == k && strncasecmp(entry, name, k) == 0;
}

// flac__utils_get_channel_mask_tag (utils.c:474-493) on one VORBIS_COMMENT body as read_metadata_vorbiscomment_
// (stream_decoder.c:2026-2121) delivers it: entries up to the first that does not fit the block
static bool vorbis_channel_mask(const uint8_t *b, uint32_t len, uint32_t *mask)
{
	static const char kName[] = "WAVEFORMATEXTENSIBLE_CHANNEL_MASK";
	const uint32_t name_len = sizeof kName - 1;
	if(len < 8) return false;
	uint32_t left = len - 8;
	const uint32_t vendor = le32(b);
	if(left < vendor) return false;
	left -= vendor;
	const uint8_t *q = b + 4 + vendor;
	const uint32_t num = le32(q);
	q += 4;
	for(uint32_t i = 0; i < num && left >= 4; i++) {
		const uint32_t el = le32(q);
		if(left - 4 < el) return false;
		left -= 4 + el;
		const char *e = reinterpret_cast<const char *>(q + 4);
		q += 4 + el;
		// FLAC__metadata_object_vorbiscomment_find_entry_from: the first entry of that name
		if(!vorbis_entry_matches(e, el, kName)) continue;
		if(el < name_len + 4) return false;
		const std::string s(e, el);  // the entry as the tool holds it, NUL-terminated
		const char *p = strchr(s.c_str(), '=');
		unsigned val;
		if(!p || strncasecmp(p, "=0x", 3) != 0 || sscanf(p + 3, "%x", &val) != 1) return false;
		*mask = val;
		return true;
	}
	return false;
}

void for_each_vorbis_comment(const uint8_t *p, size_t n, const std::function<void(const uint8_t *, uint32_t)> &fn)
{
	for(const MetaBlock &b : read_metadata_region(p, n).blocks)
		if(b.type == FLAC__METADATA_TYPE_VORBIS_COMMENT) fn(p + b.body, b.length);
}

uint32_t channel_mask_tag(const uint8_t *p, size_t n)
{
	uint32_t mask = 0;
	for_each_vorbis_comment(p, n, [&](const uint8_t *b, uint32_t len) { vorbis_channel_mask(b, len, &mask); });
	return mask;
}

bool read_metadata_vorbiscomment(const uint8_t *b, uint32_t len, std::vector<std::string> *ent)
{
	ent->clear();
	if(len < 8) return false;
	uint32_t left = len - 4;
	const uint32_t vendor = le32(b);
	if(left < vendor) return false;
	left -= vendor;
	if(left < 4) return false;
	left -= 4;
	const uint8_t *q = b + 4 + vendor;
	const uint32_t num = le32(q);
	q += 4;
	if(num > 100000) return false;
	for(uint32_t i = 0; i < num; i++) {
		if(left < 4) break;  // the block ends here: the entries read so far stand, unless bytes are left over (below)
		left -= 4;
		const uint32_t el = le32(q);
		if(left < el) return false;
		left -= el;
		ent->emplace_back(reinterpret_cast<const char *>(q + 4), el);
		q += 4 + el;
	}
	return left == 0;
}

bool read_metadata_block_data_vorbis_comment(const uint8_t *p, uint64_t n, std::string *vendor, std::vector<std::string> *ent)
{
	if(n < 4 || n - 4 < le32(p)) return false;
	vendor->assign(reinterpret_cast<const char *>(p + 4), le32(p));
	uint64_t pos = 4 + (uint64_t)le32(p);
	if(n - pos < 4) return true;
	const uint32_t count = le32(p + pos);
	pos += 4;
	if(count > (n - pos) / 4) return false;
	for(uint32_t i = 0; i < count; i++) {
		if(n - pos < 4) return false;
		const uint32_t l = le32(p + pos);
		pos += 4;
		if(n - pos < l) return false;
		ent->emplace_back(reinterpret_cast<const char *>(p + pos), l);
		pos += l;
	}
	return true;
}

const char *vorbis_comment_exact(const uint8_t *b, uint64_t len, std::vector<std::string> *ent)
{
	if(len < 8) return "VORBIS_COMMENT shorter than its fixed fields";
	uint64_t q = 4 + (uint64_t)le32(b);
	if(q + 4 > len) return "VORBIS_COMMENT vendor string runs past the block";
	const uint32_t nc = le32(b + q);
	q += 4;
	for(uint32_t c = 0; c < nc; c++) {
		if(q + 4 > len) return "VORBIS_COMMENT comment runs past the block";
		const uint32_t l = le32(b + q);
		q += 4 + (uint64_t)l;
		if(q > len) return "VORBIS_COMMENT comment runs past the block";
		if(ent) ent->emplace_back(reinterpret_cast<const char *>(b + q - l), l);
	}
	if(q != len) return "VORBIS_COMMENT length differs from its fields";
	return nullptr;
}

bool cuesheet_zero_reserved(uint8_t *b, size_t n)
{
	if(n < 396) return false;
	b[136] &= 0x80;
	memset(b + 137, 0, 258);
	size_t pos = 396;
	for(uint32_t t = 0; t < b[395]; t++) {
		if(n - pos < 36) return false;
		b[pos + 21] &= 0xc0;
		memset(b + pos + 22, 0, 13);
		const uint32_t nidx = b[pos + 35];
		pos += 36;
		if((n - pos) / 12 < nidx) return false;
		for(uint32_t k = 0; k < nidx; k++, pos += 12) memset(b + pos + 9, 0, 3);
	}
	return pos == n;
}

}  // namespace fb200
