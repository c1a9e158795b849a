// flac_parse.h -- host-side parsing of .flac containers and metadata blocks: the one reader of each format rule
// for the FLAC__stream_decoder_* shell (stream_api.cu), the batch decoders and every batch-file path that reads FLAC metadata.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

#include "../../include/flac_b200_stream.h"
#include "flac_frame.cuh"

namespace fb200 {

// The 34-byte STREAMINFO body (format.c:65-73) into its fields.
void get_streaminfo(const uint8_t *body, FLAC__StreamMetadata_StreamInfo &si);

// Bytes to skip for an ID3v2 tag whose 10-byte header starts at h ("ID3" ...): the header plus its syncsafe size.
size_t id3v2_tag_bytes(const uint8_t *h);

// Byte readers: little-endian 32 bits (VORBIS_COMMENT lengths), big-endian n <= 4 bytes, big-endian 64 bits.
inline uint32_t le32(const uint8_t *p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline uint32_t be(const uint8_t *p, int n)
{
	uint32_t v = 0;
	for(int i = 0; i < n; i++) v = v << 8 | p[i];
	return v;
}
inline uint64_t be64(const uint8_t *p) { return (uint64_t)be(p, 4) << 32 | be(p + 4, 4); }

// A metadata block header (4 bytes, stream_decoder.c:1744-1797).
struct MetaBlockHeader {
	bool last;
	uint32_t type, length;
};
MetaBlockHeader metadata_block_header(const uint8_t *h);

// The metadata region of a .flac file held whole in memory: an optional ID3v2 tag, "fLaC" at `marker`, then the blocks up to
// the one marked last. `blocks` holds every block that lies whole in the file, in order, each with the offset of its body.
struct MetaBlock : MetaBlockHeader {
	size_t body;
};
struct MetaRegion {
	enum End { OK, NO_MARKER, SHORT } end;  // SHORT: a block header or body runs past the file
	size_t marker, audio;                   // audio: where the frames begin (end OK)
	std::vector<MetaBlock> blocks;
};
MetaRegion read_metadata_region(const uint8_t *p, size_t n);

// Walks the metadata of a .flac file held whole in memory (optional ID3v2 tag, "fLaC", metadata blocks). Returns false when
// there is no "fLaC" or a block runs past the file; otherwise *has_streaminfo tells whether a STREAMINFO block of at least 34
// bytes was found (then si holds it; the length of the first one is in *streaminfo_length) and *audio_offset is where the
// frames begin.
bool walk_metadata(const uint8_t *p, size_t n, FLAC__StreamMetadata_StreamInfo &si, bool *has_streaminfo, uint32_t *streaminfo_length,
                   size_t *audio_offset);

// The channel mask the flac tool takes from a .flac file's VORBIS_COMMENT blocks (metadata_callback, decode.c:1820): per block,
// the value of its first WAVEFORMATEXTENSIBLE_CHANNEL_MASK entry (name in any case) when that entry is at least 4 bytes longer
// than the name and its value is "0x" (any case) followed by what sscanf("%x") reads; a later block's valid tag overrides an
// earlier one. 0 when no block has one.
uint32_t channel_mask_tag(const uint8_t *p, size_t n);

// Calls fn(body, length) for every VORBIS_COMMENT block of a .flac file held whole in memory, in order (optional ID3v2 tag,
// "fLaC", then the blocks up to the last one or the first that runs past the file).
void for_each_vorbis_comment(const uint8_t *p, size_t n, const std::function<void(const uint8_t *, uint32_t)> &fn);

// FLAC__metadata_object_vorbiscomment_entry_matches: whether the entry's field name (before its first '=') is `name` without
// ASCII case.
bool vorbis_entry_matches(const char *entry, size_t len, const char *name);

// The VORBIS_COMMENT readers, one per libFLAC rule. Each entry is kept as its raw bytes at its full length (embedded NULs included).

// The stream decoder's read_metadata_vorbiscomment_ (stream_decoder.c:2020-2125). Returns false where libFLAC fails the block
// (the metadata callback then never sees it): the vendor string or an entry running past the block, more than 100000 entries,
// or bytes left after the last entry read. When the block ends exactly between entries, the entries read so far are kept.
bool read_metadata_vorbiscomment(const uint8_t *b, uint32_t len, std::vector<std::string> *ent);

// The metadata chain's read_metadata_block_data_vorbis_comment_cb_ (metadata_iterators.c): the vendor and every entry must fit
// the block (else BAD_METADATA); a block that ends after the vendor string has no entries; bytes after the last entry are skipped.
bool read_metadata_block_data_vorbis_comment(const uint8_t *b, uint64_t len, std::string *vendor, std::vector<std::string> *ent);

// The encoder's rule for a client VORBIS_COMMENT: its fields fill the block exactly. nullptr, or the way the block breaks it;
// the entries are appended to *ent when ent is not null.
const char *vorbis_comment_exact(const uint8_t *b, uint64_t len, std::vector<std::string> *ent);

// A CUESHEET body with the reserved fields the encoder writes as zeros cleared (stream_encoder_framing.c:162-191); true when the
// body is exactly its fields.
bool cuesheet_zero_reserved(uint8_t *b, size_t len);

}  // namespace fb200
