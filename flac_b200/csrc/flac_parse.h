// flac_parse.h -- host-side parsing of .flac containers and frame headers, shared by the FLAC__stream_decoder_* shell
// (stream_api.cu) and the whole-file batch decoder (decoder.cu, fb200_decode_files_*).
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

#include "../../include/flac_b200_stream.h"

namespace fb200 {

// The facts of one frame header (stream_decoder.c:2624-2947).
struct FrameHeader {
	uint32_t blocksize;
	uint64_t number;      // frame or sample number from the header
	uint32_t variable;    // blocking strategy bit
	uint32_t sample_rate, channels, bps, ca;
	uint8_t crc8;
};

// Parses the frame header at p (avail bytes readable) incl. its CRC-8; sample rate / bps code 0 take STREAMINFO's values.
// Returns the header length in bytes, or 0 when there is no valid header at p.
uint32_t parse_frame_header(const uint8_t *p, size_t avail, const FLAC__StreamMetadata_StreamInfo &si, FrameHeader &fh);

// The 34-byte STREAMINFO body (format.c:65-73) into its fields.
void get_streaminfo(const uint8_t *body, FLAC__StreamMetadata_StreamInfo &si);

// Bytes to skip for an ID3v2 tag whose 10-byte header starts at h ("ID3" ...): the header plus its syncsafe size.
size_t id3v2_tag_bytes(const uint8_t *h);

// A metadata block header (4 bytes, stream_decoder.c:1744-1797).
struct MetaBlockHeader {
	bool last;
	uint32_t type, length;
};
MetaBlockHeader metadata_block_header(const uint8_t *h);

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

// The entries of one VORBIS_COMMENT body as read_metadata_vorbiscomment_ (stream_decoder.c:2020-2125) keeps them: each its raw
// bytes at its full length (embedded NULs included). Returns false where libFLAC fails the block (the metadata callback then
// never sees it): the vendor string or an entry running past the block, more than 100000 entries, or bytes left after the last
// entry read. When the block ends exactly between entries, the entries read so far are kept.
bool vorbis_entries(const uint8_t *b, uint32_t len, std::vector<std::string> *ent);

}  // namespace fb200
