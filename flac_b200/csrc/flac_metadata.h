// flac_metadata.h -- writing FLAC metadata blocks on the host (flac_metadata.cu): the block and VORBIS_COMMENT writers, the
// metadata lists of the batch encoders, the padding rule of the metadata chain and the ReplayGain tag edits.
#pragma once

#include <stdint.h>

#include <string>
#include <vector>

#include "fb200_internal.h"

namespace fb200 {

inline void put_le32(std::vector<uint8_t> &o, uint32_t v)
{
	for(int i = 0; i < 4; i++) o.push_back((uint8_t)(v >> (8 * i)));
}
// A metadata block header (format.c:154-170): the last flag, the type and the 24-bit body length.
void put_block_header(std::vector<uint8_t> &o, bool last, uint32_t type, uint32_t length);
// A VORBIS_COMMENT body: the vendor string, the entry count and the entries (stream_encoder_framing.c:118-133).
void put_vorbis_comment(std::vector<uint8_t> &o, const std::string &vendor, const std::vector<std::string> &ent);

// Checks every file's blocks metadata[metadata_offsets[f] .. [f + 1]) (both may be null: none) and plans the headers of
// fb200_encode_flac_files_*; FB200_ERR_INVALID with fb200_last_error naming the file, block and rule.
int plan_flac_headers(const uint8_t *metadata, const uint64_t *metadata_offsets, uint32_t nfiles, FlacHeaderPlan *plan);

// ---- the metadata lists of fb200_encode_pcm_files_* and fb200_reencode_flac_files_*
// One file's blocks after STREAMINFO around its VORBIS_COMMENT: whole blocks (4-byte header and body) before and after it, its
// entries (the vendor is the encoder's), and a last PADDING block of `padding` bytes (-1: none)
struct FileMeta {
	std::vector<uint8_t> before, after;
	std::vector<std::string> ent;
	int64_t padding = -1;
};
void put_block(std::vector<uint8_t> &m, uint32_t type, const std::vector<uint8_t> &body);
void put_file_metadata(const FileMeta &M, std::vector<uint8_t> &m);
// the SEEKTABLE template body of "-S <spacing_s>s" for a file of `samples` (empty: no point)
std::vector<uint8_t> seek_template(int32_t spacing_s, uint64_t samples, uint32_t sample_rate);
// flac__utils_set_channel_mask_tag on a VORBIS_COMMENT's entries
void set_channel_mask_tag(std::vector<std::string> &ent, uint32_t mask);

// chain_prepare_for_write_ with use_padding (metadata_iterators.c:1169-1243) once the chain's blocks, headers included, have gone
// from `initial` to `current` bytes: the new length of the trailing PADDING block `padding` (-1 before or after: none).
int64_t chain_padding(int64_t initial, int64_t current, int64_t padding);

// ---- ReplayGain tags (grabbag/replaygain.c)
enum RgField { RG_REFERENCE, RG_TRACK_GAIN, RG_TRACK_PEAK, RG_ALBUM_GAIN, RG_ALBUM_PEAK };
extern const char *const kRgName[5];  // "REPLAYGAIN_REFERENCE_LOUDNESS", ... in RgField order
// One of the three edits grabbag__replaygain_store_to_vorbiscomment_{reference,title,album} make: edit RG_REFERENCE (89.0 dB),
// RG_TRACK_GAIN or RG_ALBUM_GAIN (gain and peak) removes every entry of the edit's names and appends them with the new values.
void rg_edit(std::vector<std::string> &ent, RgField edit, float gain, float peak);
// --replay-gain's three tag writes on every file's list (a ReplayGainJob's rebuild, ctx an RgRebuild); without album, the album
// tags are not written (the tool writes them only when every file of the invocation succeeded)
struct RgRebuild {
	std::vector<FileMeta> files;
	bool album = true;
};
int rg_rebuild(void *ctx, const fb200_replaygain_info *info, std::vector<uint8_t> *meta, std::vector<uint64_t> *moffs);

}  // namespace fb200
