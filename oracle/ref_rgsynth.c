/* oracle/ref_rgsynth.c -- TEST INFRASTRUCTURE ONLY: the reference arm of ReplayGain synthesis. The unmodified
 * FLAC__replaygain_synthesis__apply_gain applied to constructed int32 channels in given block lengths, as the flac tool's write
 * callback calls it (source bps, target = the container's width, little-endian signed bytes), with the values read back as val32.
 * The process-global dither generator can first be advanced by `burn` draws (even) on a scratch buffer. ref_tanh_array calls the
 * host libm's tanh() in a loop. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "share/replaygain_synthesis.h"

/* in: channels x samples, interleaved; blocks: nblocks lengths summing to samples; out: val32, interleaved.
 * Returns 0, or -1 when memory runs out. The generator state is the process's: callers reload the library for a fresh start. */
int ref_rgsynth(const int32_t *in, uint32_t channels, uint64_t samples, const uint32_t *blocks, uint32_t nblocks, uint32_t bps, double scale,
                int hard_limit, int shaping, uint64_t burn, int32_t *out)
{
	const uint32_t target = 8 * ((bps + 7) / 8), B = target / 8;
	DitherContext dc;
	if(burn) {
		const uint32_t chunk = 1u << 20;
		int32_t *z = calloc(chunk, sizeof(int32_t));
		FLAC__byte *o = malloc((size_t)chunk * 4);
		if(!z || !o) { free(z); free(o); return -1; }
		const FLAC__int32 *const zi[1] = {z};
		FLAC__replaygain_synthesis__init_dither_context(&dc, 16, 1);
		for(uint64_t left = burn / 2; left;) {
			const uint32_t m = left < chunk ? (uint32_t)left : chunk;
			FLAC__replaygain_synthesis__apply_gain(o, 1, 0, zi, m, 1, 16, 16, 1.0, 0, 1, &dc);
			left -= m;
		}
		free(z); free(o);
	}
	FLAC__replaygain_synthesis__init_dither_context(&dc, (int)bps, shaping);
	int32_t *ch[8];
	FLAC__byte *buf = malloc((size_t)65536 * channels * 4 + 16);
	for(uint32_t c = 0; c < channels; c++) ch[c] = malloc((size_t)65536 * sizeof(int32_t));
	uint64_t s = 0;
	for(uint32_t j = 0; j < nblocks; j++) {
		const uint32_t n = blocks[j];
		for(uint32_t c = 0; c < channels; c++)
			for(uint32_t t = 0; t < n; t++) ch[c][t] = in[(s + t) * channels + c];
		FLAC__replaygain_synthesis__apply_gain(buf, 1, 0, (const FLAC__int32 *const *)ch, n, channels, bps, target, scale, hard_limit, shaping != 0, &dc);
		for(uint64_t v = 0; v < (uint64_t)n * channels; v++) {
			uint32_t u = 0;
			for(uint32_t b = 0; b < B; b++) u |= (uint32_t)buf[v * B + b] << (8 * b);
			out[s * channels + v] = (int32_t)(u << (32 - target)) >> (32 - target);
		}
		s += n;
	}
	for(uint32_t c = 0; c < channels; c++) free(ch[c]);
	free(buf);
	return 0;
}

void ref_tanh_array(const double *x, double *y, uint64_t n)
{
	for(uint64_t i = 0; i < n; i++) y[i] = tanh(x[i]);
}
