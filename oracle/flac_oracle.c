/*
 * flac_oracle.c -- TEST INFRASTRUCTURE ONLY (see flac_oracle.h).
 *
 * CPU restatement of the reference libFLAC 1.5.0 per-frame encode pipeline and frame
 * decoder. Written from scratch; each function cites the reference file:line whose
 * arithmetic it reproduces (paths relative to /root/reference/). Floating point is
 * evaluated in source order (compile with -ffp-contract=off, no fast-math).
 *
 * Scope: bits_per_sample 4..24 (subframe bps <= 25, i.e. no 33-bit side channel),
 * every apodization function of the specification string, no escape
 * coding / rice parameter search (both compiled out of the reference:
 * stream_encoder.c:77-82, 2107-2114).
 */
#include "flac_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif
#ifndef M_LN2
#define M_LN2 0.69314718055994530942
#endif

/* format.c:117-154 bit lengths */
#define SUBFRAME_HEADER_BITS 8u            /* zero pad 1 + type 6 + wasted flag 1 */
#define LPC_QLP_PRECISION_LEN 4u
#define LPC_QLP_SHIFT_LEN 5u
#define ENTROPY_TYPE_LEN 2u
#define RICE_ORDER_LEN 4u
#define RICE_PARAM_LEN 4u
#define RICE2_PARAM_LEN 5u
#define RICE_ESCAPE 15u
#define RICE2_ESCAPE 31u
#define MAX_RICE_PARTITION_ORDER 15u
#define MIN_QLP_PRECISION 5u
#define MAX_QLP_PRECISION 15u
#define MAX_FIXED_ORDER 4u
#define MAX_EXTRA_RESIDUAL_BPS 4u /* private/stream_encoder.h:44 */

#define MINU(a, b) ((a) < (b) ? (a) : (b))
#define MAXU(a, b) ((a) > (b) ? (a) : (b))

struct fo_encoder {
	fo_config cfg;
	uint32_t win_blocksize;                 /* blocksize the tables below were computed for */
	float *window[FO_MAX_APODIZATIONS];
	/* scratch */
	int32_t *sig[4];                        /* L,R,M,S (or ch0..) working copies */
	int32_t *chan[FO_MAX_CHANNELS];
	int32_t *residual;
	float *windowed;
	uint64_t *psums;
	fo_lpc_cand lpc_cands[FO_MAX_LPC_CANDIDATES];  /* one apodization's candidates */
};

/* ------------------------------------------------------------------ bit math */

/* bitmath.h FLAC__bitmath_ilog2 / _wide: floor(log2(v)), v > 0 */
static uint32_t ilog2_64(uint64_t v)
{
	uint32_t l = 0;
	while(v >>= 1) l++;
	return l;
}

/* bitmath.c:63-73 FLAC__bitmath_silog2 */
static uint32_t silog2(int64_t v)
{
	if(v == 0) return 0;
	if(v == -1) return 2;
	v = (v < 0) ? (-(v + 1)) : v;
	return ilog2_64((uint64_t)v) + 2;
}

uint32_t fo_silog2(int64_t v) { return silog2(v); }

static fo_lpc_counters counters;

void fo_lpc_counters_get(fo_lpc_counters *out, int reset)
{
	if(out) *out = counters;
	if(reset) memset(&counters, 0, sizeof counters);
}

/* ------------------------------------------------------------------ CRC (crc.c:39-396) */

static uint8_t crc8_table[256];
static uint16_t crc16_table[256];
static int crc_ready = 0;

static void crc_init(void)
{
	uint32_t i, j;
	if(crc_ready) return;
	for(i = 0; i < 256; i++) {
		uint32_t c8 = i, c16 = i << 8;
		for(j = 0; j < 8; j++) {
			c8 = (c8 & 0x80) ? ((c8 << 1) ^ 0x07) : (c8 << 1);          /* poly x^8+x^2+x+1 */
			c16 = (c16 & 0x8000) ? ((c16 << 1) ^ 0x8005) : (c16 << 1);  /* poly x^16+x^15+x^2+1 */
		}
		crc8_table[i] = (uint8_t)c8;
		crc16_table[i] = (uint16_t)c16;
	}
	crc_ready = 1;
}

uint8_t fo_crc8(const uint8_t *data, size_t len)
{
	uint8_t crc = 0;
	crc_init();
	while(len--) crc = crc8_table[crc ^ *data++];
	return crc;
}

uint16_t fo_crc16(const uint8_t *data, size_t len)
{
	uint16_t crc = 0;
	crc_init();
	while(len--) crc = (uint16_t)((crc << 8) ^ crc16_table[(crc >> 8) ^ *data++]);
	return crc;
}

/* ------------------------------------------------------------------ bit writer
 * MSB-first, big-endian (bitwriter.c:55-106, 316-394). */

typedef struct {
	uint8_t *buf;
	size_t cap;      /* bytes */
	uint64_t bits;   /* bits written */
	int overflow;
} bitw;

static void bw_init(bitw *bw, uint8_t *buf, size_t cap)
{
	bw->buf = buf; bw->cap = cap; bw->bits = 0; bw->overflow = 0;
	memset(buf, 0, cap);
}

static void bw_write(bitw *bw, uint64_t val, uint32_t nbits)
{
	/* writes the low nbits of val, most significant first (bitwriter.c:316-394) */
	while(nbits) {
		const size_t byte = (size_t)(bw->bits >> 3);
		const uint32_t room = 8 - (uint32_t)(bw->bits & 7);
		const uint32_t take = nbits < room ? nbits : room;
		uint64_t chunk;
		if(byte >= bw->cap) { bw->overflow = 1; return; }
		chunk = (val >> (nbits - take)) & ((1u << take) - 1u);
		bw->buf[byte] |= (uint8_t)(chunk << (room - take));
		bw->bits += take;
		nbits -= take;
	}
}

static void bw_write_signed(bitw *bw, int64_t val, uint32_t nbits)
{
	bw_write(bw, (uint64_t)val, nbits); /* two's complement truncated to nbits (bitwriter.c:357-394) */
}

/* bitwriter.c:429 FLAC__bitwriter_write_unary_unsigned: val zero bits then a one */
static void bw_write_unary(bitw *bw, uint32_t val)
{
	bw->bits += val; /* buffer is pre-zeroed */
	bw_write(bw, 1, 1);
}

/* bitwriter.c:575-706 FLAC__bitwriter_write_rice_signed_block, one value */
static void bw_write_rice(bitw *bw, int32_t val, uint32_t k)
{
	const uint32_t u = ((uint32_t)val << 1) ^ (uint32_t)(val >> 31); /* zig-zag fold */
	bw_write_unary(bw, u >> k);
	if(k) bw_write(bw, u & ((1u << k) - 1u), k);
}

/* bitwriter.c:832-933 FLAC__bitwriter_write_utf8_uint32 (frame number, up to 31 bits) */
static void bw_write_utf8(bitw *bw, uint32_t val)
{
	if(val < 0x80) bw_write(bw, val, 8);
	else if(val < 0x800) { bw_write(bw, 0xC0 | (val >> 6), 8); bw_write(bw, 0x80 | (val & 0x3F), 8); }
	else if(val < 0x10000) { bw_write(bw, 0xE0 | (val >> 12), 8); bw_write(bw, 0x80 | ((val >> 6) & 0x3F), 8); bw_write(bw, 0x80 | (val & 0x3F), 8); }
	else if(val < 0x200000) { bw_write(bw, 0xF0 | (val >> 18), 8); bw_write(bw, 0x80 | ((val >> 12) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 6) & 0x3F), 8); bw_write(bw, 0x80 | (val & 0x3F), 8); }
	else if(val < 0x4000000) { bw_write(bw, 0xF8 | (val >> 24), 8); bw_write(bw, 0x80 | ((val >> 18) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 12) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 6) & 0x3F), 8); bw_write(bw, 0x80 | (val & 0x3F), 8); }
	else { bw_write(bw, 0xFC | (val >> 30), 8); bw_write(bw, 0x80 | ((val >> 24) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 18) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 12) & 0x3F), 8); bw_write(bw, 0x80 | ((val >> 6) & 0x3F), 8); bw_write(bw, 0x80 | (val & 0x3F), 8); }
}

/* ------------------------------------------------------------------ windows (window.c:46-55, 195-220) */

void fo_window_tukey(float *window, int32_t L, float p)
{
	int32_t n;
	if(p <= 0.0) {
		for(n = 0; n < L; n++) window[n] = 1.0f;
	}
	else if(p >= 1.0) {
		/* window.c:136-143 FLAC__window_hann */
		const int32_t N = L - 1;
		for(n = 0; n < L; n++)
			window[n] = (float)(0.5f - 0.5f * cosf(2.0f * M_PI * n / N));
	}
	else if(!(p > 0.0f && p < 1.0f)) {
		fo_window_tukey(window, L, 0.5f);
	}
	else {
		const int32_t Np = (int32_t)(p / 2.0f * L) - 1;
		for(n = 0; n < L; n++) window[n] = 1.0f;
		if(Np > 0) {
			for(n = 0; n <= Np; n++) {
				window[n] = (float)(0.5f - 0.5f * cosf(M_PI * n / Np));
				window[L - Np - 1 + n] = (float)(0.5f - 0.5f * cosf(M_PI * (n + Np) / Np));
			}
		}
	}
}

/* window.c:50-197, 224-302: the other generators. Sub-expression types as C promotes them
 * in the reference (float * double M_PI -> double, narrowed to float by cosf's prototype). */
static float half_cos(int32_t i, int32_t Np) { return (float)(0.5f - 0.5f * cosf(M_PI * i / Np)); }

int fo_window(const fo_apodization *a, float *w, int32_t L)
{
	const int32_t N = L - 1;
	const double N2 = (double)N / 2.;
	int32_t n, i;
	switch(a->type) {
		case FO_APOD_TUKEY:
		case FO_APOD_SUBDIVIDE_TUKEY: /* stream_encoder.c:2962-2964 */
			fo_window_tukey(w, L, a->p);
			return 1;
		case FO_APOD_BARTLETT: /* :50-67 */
			if(L & 1) {
				for(n = 0; n <= N / 2; n++) w[n] = 2.0f * n / (float)N;
				for(; n <= N; n++) w[n] = 2.0f - 2.0f * n / (float)N;
			}
			else {
				for(n = 0; n <= L / 2 - 1; n++) w[n] = 2.0f * n / (float)N;
				for(; n <= N; n++) w[n] = 2.0f - 2.0f * n / (float)N;
			}
			return 1;
		case FO_APOD_BARTLETT_HANN: /* :69-76 */
			for(n = 0; n < L; n++)
				w[n] = (float)(0.62f - 0.48f * fabsf((float)n / (float)N - 0.5f) - 0.38f * cosf(2.0f * M_PI * ((float)n / (float)N)));
			return 1;
		case FO_APOD_BLACKMAN: /* :78-85 */
			for(n = 0; n < L; n++) w[n] = (float)(0.42f - 0.5f * cosf(2.0f * M_PI * n / N) + 0.08f * cosf(4.0f * M_PI * n / N));
			return 1;
		case FO_APOD_BLACKMAN_HARRIS: /* :88-95 */
			for(n = 0; n <= N; n++)
				w[n] = (float)(0.35875f - 0.48829f * cosf(2.0f * M_PI * n / N) + 0.14128f * cosf(4.0f * M_PI * n / N) - 0.01168f * cosf(6.0f * M_PI * n / N));
			return 1;
		case FO_APOD_CONNES: /* :97-108 */
			for(n = 0; n <= N; n++) {
				double k = ((double)n - N2) / N2;
				k = 1.0f - k * k;
				w[n] = (float)(k * k);
			}
			return 1;
		case FO_APOD_FLATTOP: /* :110-117 */
			for(n = 0; n < L; n++)
				w[n] = (float)(0.21557895f - 0.41663158f * cosf(2.0f * M_PI * n / N) + 0.277263158f * cosf(4.0f * M_PI * n / N) - 0.083578947f * cosf(6.0f * M_PI * n / N) + 0.006947368f * cosf(8.0f * M_PI * n / N));
			return 1;
		case FO_APOD_GAUSS: { /* :119-135 */
			const float stddev = (a->p > 0.0f && a->p <= 0.5f) ? a->p : 0.25f;
			for(n = 0; n <= N; n++) {
				const double k = ((double)n - N2) / (stddev * N2);
				w[n] = (float)exp(-0.5f * k * k);
			}
			return 1;
		}
		case FO_APOD_HAMMING: /* :137-144 */
			for(n = 0; n < L; n++) w[n] = (float)(0.54f - 0.46f * cosf(2.0f * M_PI * n / N));
			return 1;
		case FO_APOD_HANN: /* :146-153 */
			for(n = 0; n < L; n++) w[n] = (float)(0.5f - 0.5f * cosf(2.0f * M_PI * n / N));
			return 1;
		case FO_APOD_KAISER_BESSEL: /* :155-162 */
			for(n = 0; n < L; n++)
				w[n] = (float)(0.402f - 0.498f * cosf(2.0f * M_PI * n / N) + 0.098f * cosf(4.0f * M_PI * n / N) - 0.001f * cosf(6.0f * M_PI * n / N));
			return 1;
		case FO_APOD_NUTTALL: /* :164-171 */
			for(n = 0; n < L; n++)
				w[n] = (float)(0.3635819f - 0.4891775f * cosf(2.0f * M_PI * n / N) + 0.1365995f * cosf(4.0f * M_PI * n / N) - 0.0106411f * cosf(6.0f * M_PI * n / N));
			return 1;
		case FO_APOD_RECTANGLE: /* :173-179 */
			for(n = 0; n < L; n++) w[n] = 1.0f;
			return 1;
		case FO_APOD_TRIANGLE: /* :181-197 */
			for(n = 1; n <= ((L & 1) ? (L + 1) / 2 : L / 2); n++) w[n - 1] = 2.0f * n / ((float)L + 1.0f);
			for(; n <= L; n++) w[n - 1] = (float)(2 * (L - n + 1)) / ((float)L + 1.0f);
			return 1;
		case FO_APOD_WELCH: /* :292-302 */
			for(n = 0; n <= N; n++) {
				const double k = ((double)n - N2) / N2;
				w[n] = (float)(1.0f - k * k);
			}
			return 1;
		case FO_APOD_PARTIAL_TUKEY:
		case FO_APOD_PUNCHOUT_TUKEY: {
			/* :231-238 / :262-269 parameter clamps */
			float p = a->p;
			const int32_t start_n = (int32_t)(a->start * L), end_n = (int32_t)(a->end * L);
			if(p <= 0.0f) p = 0.05f;
			else if(p >= 1.0f) p = 0.95f;
			else if(!(p > 0.0f && p < 1.0f)) p = 0.5f;
			if(a->type == FO_APOD_PARTIAL_TUKEY) { /* :224-254 */
				const int32_t Np = (int32_t)(p / 2.0f * (end_n - start_n));
				for(n = 0; n < start_n && n < L; n++) w[n] = 0.0f;
				for(i = 1; n < (start_n + Np) && n < L; n++, i++) w[n] = half_cos(i, Np);
				for(; n < (end_n - Np) && n < L; n++) w[n] = 1.0f;
				for(i = Np; n < end_n && n < L; n++, i--) w[n] = half_cos(i, Np);
				for(; n < L; n++) w[n] = 0.0f;
			}
			else { /* :256-290 */
				const int32_t Ns = (int32_t)(p / 2.0f * start_n), Ne = (int32_t)(p / 2.0f * (L - end_n));
				for(n = 0, i = 1; n < Ns && n < L; n++, i++) w[n] = half_cos(i, Ns);
				for(; n < start_n - Ns && n < L; n++) w[n] = 1.0f;
				for(i = Ns; n < start_n && n < L; n++, i--) w[n] = half_cos(i, Ns);
				for(; n < end_n && n < L; n++) w[n] = 0.0f;
				for(i = 1; n < end_n + Ne && n < L; n++, i++) w[n] = half_cos(i, Ne);
				for(; n < L - Ne && n < L; n++) w[n] = 1.0f;
				for(i = Ne; n < L; n++, i--) w[n] = half_cos(i, Ne);
			}
			return 1;
		}
	}
	return 0;
}

/* stream_encoder.c:1940-2065 FLAC__stream_encoder_set_apodization */
void fo_config_set_apodization(fo_config *cfg, const char *spec)
{
	static const struct { const char *name; int32_t type; } names[] = {
		{"bartlett", FO_APOD_BARTLETT}, {"bartlett_hann", FO_APOD_BARTLETT_HANN}, {"blackman", FO_APOD_BLACKMAN},
		{"blackman_harris_4term_92db", FO_APOD_BLACKMAN_HARRIS}, {"connes", FO_APOD_CONNES}, {"flattop", FO_APOD_FLATTOP},
		{"hamming", FO_APOD_HAMMING}, {"hann", FO_APOD_HANN}, {"kaiser_bessel", FO_APOD_KAISER_BESSEL}, {"nuttall", FO_APOD_NUTTALL},
		{"rectangle", FO_APOD_RECTANGLE}, {"triangle", FO_APOD_TRIANGLE}, {"welch", FO_APOD_WELCH}};
	fo_apodization *A = cfg->apodizations;
	uint32_t num = 0;
	memset(A, 0, sizeof cfg->apodizations);
	while(1) {
		const char *s = strchr(spec, ';');
		const size_t n = s ? (size_t)(s - spec) : strlen(spec);
		size_t t;
		int hit = 0;
		for(t = 0; t < sizeof names / sizeof names[0]; t++)
			if(n == strlen(names[t].name) && 0 == strncmp(names[t].name, spec, n)) { A[num++].type = names[t].type; hit = 1; break; }
		if(hit) {}
		else if(n > 7 && 0 == strncmp("gauss(", spec, 6)) {
			float stddev = (float)strtod(spec + 6, 0);
			if(stddev > 0.0 && stddev <= 0.5) { A[num].p = stddev; A[num++].type = FO_APOD_GAUSS; }
		}
		else if(n > 7 && 0 == strncmp("tukey(", spec, 6)) {
			float p = (float)strtod(spec + 6, 0);
			if(p >= 0.0 && p <= 1.0) { A[num].p = p; A[num++].type = FO_APOD_TUKEY; }
		}
		else if((n > 15 && 0 == strncmp("partial_tukey(", spec, 14)) || (n > 16 && 0 == strncmp("punchout_tukey(", spec, 15))) {
			const int partial = (spec[1] == 'a');
			int32_t parts = (int32_t)strtod(spec + (partial ? 14 : 15), 0), m;
			const char *si_1 = strchr(spec, '/');
			float overlap = si_1 ? (float)strtod(si_1 + 1, 0) : (partial ? 0.1f : 0.2f);
			float overlap_units, tukey_p;
			const char *si_2;
			if(si_1 && !(overlap < 0.99f)) overlap = 0.99f;
			overlap_units = 1.0f / (1.0f - overlap) - 1.0f;
			si_2 = strchr((si_1 ? (si_1 + 1) : spec), '/');
			tukey_p = si_2 ? (float)strtod(si_2 + 1, 0) : 0.2f;
			if(parts <= 1) { A[num].p = tukey_p; A[num++].type = FO_APOD_TUKEY; }
			else if(num + parts < 32)
				for(m = 0; m < parts; m++) {
					A[num].p = tukey_p;
					A[num].start = m / (parts + overlap_units);
					A[num].end = (m + 1 + overlap_units) / (parts + overlap_units);
					A[num++].type = partial ? FO_APOD_PARTIAL_TUKEY : FO_APOD_PUNCHOUT_TUKEY;
				}
		}
		else if(n > 17 && 0 == strncmp("subdivide_tukey(", spec, 16)) {
			int32_t parts = (int32_t)strtod(spec + 16, 0);
			if(parts > 1) {
				const char *si_1 = strchr(spec, '/');
				float p = si_1 ? (float)strtod(si_1 + 1, 0) : 5e-1;
				if(p > 1) p = 1;
				else if(p < 0) p = 0;
				A[num].parts = parts;
				A[num].p = p / parts;
				A[num++].type = FO_APOD_SUBDIVIDE_TUKEY;
			}
		}
		if(num == 32) break;
		if(s) spec = s + 1;
		else break;
	}
	if(num == 0) { num = 1; A[0].type = FO_APOD_TUKEY; A[0].p = 0.5f; }
	cfg->num_apodizations = num;
}

/* ------------------------------------------------------------------ LPC analysis */

/* lpc.c:68-74 FLAC__lpc_window_data */
void fo_window_data(const int32_t *in, const float *window, float *out, uint32_t data_len)
{
	uint32_t i;
	for(i = 0; i < data_len; i++)
		out[i] = in[i] * window[i];
}

/* lpc.c:82-94 FLAC__lpc_window_data_partial */
void fo_window_data_partial(const int32_t *in, const float *window, float *out, uint32_t data_len, uint32_t part_size, uint32_t data_shift)
{
	uint32_t i, j;
	if((part_size + data_shift) < data_len) {
		for(i = 0; i < part_size; i++)
			out[i] = in[data_shift + i] * window[i];
		i = MINU(i, data_len - part_size - data_shift);
		for(j = data_len - part_size; j < data_len; i++, j++)
			out[i] = in[data_shift + i] * window[j];
		if(i < data_len)
			out[i] = 0.0f;
	}
}

/* lpc.c:110-174 + deduplication/lpc_compute_autocorrelation_intrin.c:5-14.
 * For every lag l the terms data[i]*data[i-l] (exact in double) are added in ascending i
 * into one accumulator. Both branches of the reference produce this sequence; the
 * intrin branch computes MAX_LAG (8/12/16) lags, of which only `lag` are used. */
void fo_autocorrelation(const float *data, uint32_t data_len, uint32_t lag, double *autoc)
{
	uint32_t l, i;
	for(l = 0; l < lag; l++) {
		double d = 0.0;
		for(i = l; i < data_len; i++)
			d += (double)data[i] * (double)data[i - l];
		autoc[l] = d;
	}
}

/* lpc.c:176-218 FLAC__lpc_compute_lp_coefficients (Levinson-Durbin) */
void fo_lp_coefficients(const double *autoc, uint32_t *max_order, float lp_coeff[][FO_MAX_LPC_ORDER], double *error)
{
	uint32_t i, j;
	double r, err, lpc[FO_MAX_LPC_ORDER];

	err = autoc[0];
	for(i = 0; i < *max_order; i++) {
		r = -autoc[i + 1];
		for(j = 0; j < i; j++)
			r -= lpc[j] * autoc[i - j];
		r /= err;

		lpc[i] = r;
		for(j = 0; j < (i >> 1); j++) {
			double tmp = lpc[j];
			lpc[j] += r * lpc[i - 1 - j];
			lpc[i - 1 - j] += r * tmp;
		}
		if(i & 1)
			lpc[j] += lpc[j] * r;

		err *= (1.0 - r * r);

		for(j = 0; j <= i; j++)
			lp_coeff[i][j] = (float)(-lpc[j]);
		error[i] = err;

		if(err == 0.0) {
			if(i + 1 < *max_order) counters.levinson_early++;
			*max_order = i + 1;
			return;
		}
	}
}

/* lpc.c:1580-1606 FLAC__lpc_compute_expected_bits_per_residual_sample_with_error_scale */
static double expected_bits_with_scale(double lpc_error, double error_scale)
{
	if(lpc_error > 0.0) {
		double bps = (double)0.5 * log(error_scale * lpc_error) / M_LN2;
		return bps >= 0.0 ? bps : 0.0;
	}
	else if(lpc_error < 0.0)
		return 1e32;
	else
		return 0.0;
}

/* lpc.c:1580-1590 */
static double expected_bits(double lpc_error, uint32_t total_samples)
{
	double error_scale = 0.5 / (double)total_samples;
	return expected_bits_with_scale(lpc_error, error_scale);
}

/* lpc.c:1608-1630 FLAC__lpc_compute_best_order */
uint32_t fo_best_order(const double *lpc_error, uint32_t max_order, uint32_t total_samples, uint32_t overhead_bits_per_order)
{
	uint32_t order, indx, best_index = 0;
	double bits, best_bits, error_scale;

	error_scale = 0.5 / (double)total_samples;
	best_bits = (uint32_t)(-1);
	for(indx = 0, order = 1; indx < max_order; indx++, order++) {
		bits = expected_bits_with_scale(lpc_error[indx], error_scale) * (double)(total_samples - order) + (double)(order * overhead_bits_per_order);
		if(bits < best_bits) {
			best_index = indx;
			best_bits = bits;
		}
	}
	return best_index + 1;
}

/* lpc.c:220-314 FLAC__lpc_quantize_coefficients */
int fo_quantize_coefficients(const float *lp_coeff, uint32_t order, uint32_t precision, int32_t *qlp_coeff, int *shift)
{
	uint32_t i;
	double cmax;
	int32_t qmax, qmin;

	precision--;
	qmax = 1 << precision;
	qmin = -qmax;
	qmax--;

	cmax = 0.0;
	for(i = 0; i < order; i++) {
		const double d = fabs(lp_coeff[i]);
		if(d > cmax) cmax = d;
	}
	if(cmax <= 0.0) {
		counters.cmax_zero++;
		return 2;
	}
	else {
		const int max_shiftlimit = (1 << (LPC_QLP_SHIFT_LEN - 1)) - 1;
		const int min_shiftlimit = -max_shiftlimit - 1;
		int log2cmax;
		(void)frexp(cmax, &log2cmax);
		log2cmax--;
		*shift = (int)precision - log2cmax - 1;
		if(*shift > max_shiftlimit) {
			*shift = max_shiftlimit;
			counters.shift_clamped++;
		}
		else if(*shift < min_shiftlimit) {
			counters.shift_too_small++;
			return 1;
		}
	}

	if(*shift >= 0) {
		double error = 0.0;
		int32_t q;
		for(i = 0; i < order; i++) {
			error += lp_coeff[i] * (1 << *shift);   /* float * int -> float product, then double add */
			if(fabs(error - trunc(error)) == 0.5) counters.round_half++;
			q = (int32_t)lround(error);
			if(q > qmax || q < qmin) counters.coef_clipped++;
			if(q > qmax) q = qmax;
			else if(q < qmin) q = qmin;
			error -= q;
			qlp_coeff[i] = q;
		}
	}
	else {
		const int nshift = -(*shift);
		double error = 0.0;
		counters.negative_shift++;
		int32_t q;
		for(i = 0; i < order; i++) {
			error += lp_coeff[i] / (1 << nshift);
			if(fabs(error - trunc(error)) == 0.5) counters.round_half++;
			q = (int32_t)lround(error);
			if(q > qmax || q < qmin) counters.coef_clipped++;
			if(q > qmax) q = qmax;
			else if(q < qmin) q = qmin;
			error -= q;
			qlp_coeff[i] = q;
		}
		*shift = 0;
	}
	return 0;
}

/* lpc.c:942-968 */
uint64_t fo_max_prediction_value_before_shift(uint32_t subframe_bps, const int32_t *qlp, uint32_t order)
{
	uint64_t max_abs_sample_value = (uint64_t)1 << (subframe_bps - 1);
	uint32_t abs_sum = 0, i;
	for(i = 0; i < order; i++)
		abs_sum += (uint32_t)abs(qlp[i]);
	return max_abs_sample_value * abs_sum;
}

uint32_t fo_max_residual_bps(uint32_t subframe_bps, const int32_t *qlp, uint32_t order, int lp_quantization)
{
	uint64_t max_abs_sample_value = (uint64_t)1 << (subframe_bps - 1);
	uint64_t max_pred_after = (uint64_t)(-1 * ((-1 * (int64_t)fo_max_prediction_value_before_shift(subframe_bps, qlp, order)) >> lp_quantization));
	uint64_t max_residual_value = max_abs_sample_value + max_pred_after;
	return silog2((int64_t)max_residual_value);
}

/* lpc.c:321-938: every variant (32-bit, 16-bit, wide, limit_residual) computes
 * residual[i] = data[i] - ((sum_j qlp[j]*data[i-1-j]) >> shift); the 32-bit variants are
 * only selected when the sum provably fits (stream_encoder.c:4601-4617), so int64
 * arithmetic reproduces all of them. limit != 0: fail when a residual leaves
 * (INT32_MIN, INT32_MAX] (lpc.c:868-884). */
static int lpc_residual(const int32_t *data, uint32_t data_len, const int32_t *qlp, uint32_t order, int shift, int32_t *residual, int limit)
{
	uint32_t i, j;
	for(i = 0; i < data_len; i++) {
		int64_t sum = 0, r;
		for(j = 0; j < order; j++)
			sum += (int64_t)qlp[j] * (int64_t)data[(int64_t)i - 1 - (int64_t)j];
		r = (int64_t)data[i] - (sum >> shift);
		if(limit && (r <= INT32_MIN || r > INT32_MAX))
			return 0;
		residual[i] = (int32_t)r;
	}
	return 1;
}

/* ------------------------------------------------------------------ fixed predictors */

/* fixed.c:222-290 (+ _wide :302-370): abs sums of the 0..4th differences over data[0..len)
 * (data points 4 samples into the block), lower order preferred on ties, and the float
 * bits-per-sample estimates. 64-bit sums are exact for subframe bps < 28. */
static uint32_t fixed_best_predictor(const int32_t *data, uint32_t data_len, int avx2_wide, float rbps[MAX_FIXED_ORDER + 1])
{
	uint64_t te[5] = {0, 0, 0, 0, 0};
	uint32_t order, k;
	int64_t i;
	if(!avx2_wide) {
		for(i = 0; i < (int64_t)data_len; i++) {
			const int64_t d0 = data[i], d1 = data[i - 1], d2 = data[i - 2], d3 = data[i - 3], d4 = data[i - 4];
			const int64_t e0 = d0, e1 = d0 - d1, e2 = d0 - 2 * d1 + d2, e3 = d0 - 3 * d1 + 3 * d2 - d3, e4 = d0 - 4 * d1 + 6 * d2 - 4 * d3 + d4;
			te[0] += (uint64_t)(e0 < 0 ? -e0 : e0);
			te[1] += (uint64_t)(e1 < 0 ? -e1 : e1);
			te[2] += (uint64_t)(e2 < 0 ? -e2 : e2);
			te[3] += (uint64_t)(e3 < 0 ? -e3 : e3);
			te[4] += (uint64_t)(e4 < 0 ? -e4 : e4);
		}
	}
	else {
		/* fixed_intrin_avx2.c:57-138 FLAC__fixed_compute_best_predictor_wide_intrin_avx2, as written: four lanes walk
		 * data_len / 4 samples each; lane j READS from offset (j * data_len) / 4 (:88-91) but its difference history is
		 * seeded from offset j * (data_len / 4) (:77-82) -- the two agree only when data_len is a multiple of 4 -- and
		 * the data_len % 4 samples past the last lane are never summed (:138). The estimates still divide by data_len. */
		const int64_t q = (int64_t)(data_len / 4);
		int j;
		for(j = 0; j < 4; j++) {
			const int64_t op = j * q, od = ((int64_t)j * (int64_t)data_len) / 4;
			int64_t p0 = data[-1 + op];
			int64_t p1 = (int64_t)data[-1 + op] - data[-2 + op];
			int64_t p2 = p1 - ((int64_t)data[-2 + op] - data[-3 + op]);
			int64_t p3 = p2 - ((int64_t)data[-2 + op] - 2 * (int64_t)data[-3 + op] + data[-4 + op]);
			for(i = 0; i < q; i++) {
				const int64_t e0 = data[i + od];
				const int64_t e1 = e0 - p0, e2 = e1 - p1, e3 = e2 - p2, e4 = e3 - p3;
				p0 = e0; p1 = e1; p2 = e2; p3 = e3;
				te[0] += (uint64_t)(e0 < 0 ? -e0 : e0);
				te[1] += (uint64_t)(e1 < 0 ? -e1 : e1);
				te[2] += (uint64_t)(e2 < 0 ? -e2 : e2);
				te[3] += (uint64_t)(e3 < 0 ? -e3 : e3);
				te[4] += (uint64_t)(e4 < 0 ? -e4 : e4);
			}
		}
	}
	if(te[0] <= MINU(MINU(MINU(te[1], te[2]), te[3]), te[4])) order = 0;
	else if(te[1] <= MINU(MINU(te[2], te[3]), te[4])) order = 1;
	else if(te[2] <= MINU(te[3], te[4])) order = 2;
	else if(te[3] <= te[4]) order = 3;
	else order = 4;
	for(k = 0; k < 5; k++)
		rbps[k] = (float)((te[k] > 0) ? log(M_LN2 * (double)te[k] / (double)data_len) / M_LN2 : 0.0);
	return order;
}

/* fixed.c:470-530 FLAC__fixed_compute_residual(_wide): data points `order` samples into the block */
static void fixed_residual(const int32_t *data, uint32_t data_len, uint32_t order, int32_t *residual)
{
	int64_t i;
	for(i = 0; i < (int64_t)data_len; i++) {
		int64_t r;
		switch(order) {
			case 0: r = data[i]; break;
			case 1: r = (int64_t)data[i] - data[i - 1]; break;
			case 2: r = (int64_t)data[i] - 2 * (int64_t)data[i - 1] + data[i - 2]; break;
			case 3: r = (int64_t)data[i] - 3 * (int64_t)data[i - 1] + 3 * (int64_t)data[i - 2] - data[i - 3]; break;
			default: r = (int64_t)data[i] - 4 * (int64_t)data[i - 1] + 6 * (int64_t)data[i - 2] - 4 * (int64_t)data[i - 3] + data[i - 4]; break;
		}
		residual[i] = (int32_t)r;
	}
}

/* ------------------------------------------------------------------ Rice partition search */

/* format.c:540-562 */
static uint32_t max_rice_partition_order_from_blocksize(uint32_t blocksize)
{
	uint32_t o = 0;
	while(!(blocksize & 1)) { o++; blocksize >>= 1; }
	return MINU(MAX_RICE_PARTITION_ORDER, o);
}

static uint32_t max_rice_partition_order_limited(uint32_t limit, uint32_t blocksize, uint32_t predictor_order)
{
	uint32_t o = limit;
	while(o > 0 && (blocksize >> o) <= predictor_order) o--;
	return o;
}

/* stream_encoder.c:4929-4951 count_rice_bits_in_partition_ (estimate, not exact) */
static uint32_t count_rice_bits(uint32_t k, uint32_t partition_samples, uint64_t abs_sum)
{
	uint64_t v = (uint64_t)RICE_PARAM_LEN + (uint64_t)(1 + k) * partition_samples
	             + (k ? (abs_sum >> (k - 1)) : (abs_sum << 1)) - (partition_samples >> 1);
	return (uint32_t)(v < UINT32_MAX ? v : UINT32_MAX);
}

/* stream_encoder.c:4954-5075 set_partitioned_rice_ (no escapes, no parameter search) */
static int set_partitioned_rice(const uint64_t *sums, uint32_t residual_samples, uint32_t predictor_order, uint32_t rice_parameter_limit, uint32_t partition_order, int32_t *parameters, uint32_t *bits)
{
	uint32_t bits_ = ENTROPY_TYPE_LEN + RICE_ORDER_LEN;
	const uint32_t partitions = 1u << partition_order;
	const uint32_t partition_samples_base = (residual_samples + predictor_order) >> partition_order;
	const uint32_t divisor_base = 0x40000 / partition_samples_base;
	uint32_t partition;
	for(partition = 0; partition < partitions; partition++) {
		uint32_t partition_samples = partition_samples_base, divisor, rice_parameter, pbits;
		uint64_t mean;
		if(partition > 0)
			divisor = divisor_base;
		else {
			if(partition_samples <= predictor_order)
				return 0;
			partition_samples -= predictor_order;
			divisor = 0x40000 / partition_samples;
		}
		mean = sums[partition];
		if(mean < 2 || (((mean - 1) * divisor) >> 18) == 0)
			rice_parameter = 0;
		else
			rice_parameter = ilog2_64(((mean - 1) * divisor) >> 18) + 1;
		if(rice_parameter >= rice_parameter_limit)
			rice_parameter = rice_parameter_limit - 1;
		pbits = count_rice_bits(rice_parameter, partition_samples, sums[partition]);
		parameters[partition] = (int32_t)rice_parameter;
		if(pbits < UINT32_MAX - bits_) bits_ += pbits;
		else bits_ = UINT32_MAX;
	}
	*bits = bits_;
	return 1;
}

/* stream_encoder.c:4701-4795 find_best_partition_order_ + :4797-4852 precompute_partition_info_sums_ */
static uint32_t find_best_partition_order(fo_encoder *e, const int32_t *residual, uint32_t residual_samples, uint32_t predictor_order,
                                          uint32_t rice_parameter_limit, uint32_t min_po, uint32_t max_po, uint32_t bps, fo_subframe_plan *plan)
{
	const uint32_t blocksize = residual_samples + predictor_order;
	uint64_t *sums = e->psums;
	uint32_t best_bits = 0, best_po = 0;
	int32_t params[2][FO_MAX_PARTITIONS];
	int best_idx = 0;

	max_po = max_rice_partition_order_limited(max_po, blocksize, predictor_order);
	min_po = MINU(min_po, max_po);

	{   /* sums at max_po: 32-bit wrapping accumulator when bps+4 < 32-ilog2(partition samples) (:4814-4834) */
		const uint32_t default_partition_samples = blocksize >> max_po;
		const uint32_t threshold = 32 - ilog2_64(default_partition_samples);
		const int narrow = (bps + MAX_EXTRA_RESIDUAL_BPS < threshold);
		uint32_t partitions = 1u << max_po, partition, rs = 0, end = (uint32_t)(-(int32_t)predictor_order);
		uint32_t from = 0, to;
		int po;
		for(partition = 0; partition < partitions; partition++) {
			uint64_t s = 0;
			end += default_partition_samples;
			for(; rs < end; rs++) {
				const int32_t r = residual[rs];
				s += (uint32_t)(r < 0 ? -(uint32_t)r : (uint32_t)r);
			}
			if(narrow && s > UINT32_MAX) counters.narrow_wrapped++;
			sums[partition] = narrow ? (uint64_t)(uint32_t)s : s;
		}
		to = partitions;
		for(po = (int)max_po - 1; po >= (int)min_po; po--) {
			uint32_t i;
			partitions >>= 1;
			for(i = 0; i < partitions; i++) {
				sums[to++] = sums[from] + sums[from + 1];
				from += 2;
			}
		}
	}
	{
		int po;
		uint32_t sum = 0, bits;
		for(po = (int)max_po; po >= (int)min_po; po--) {
			if(!set_partitioned_rice(sums + sum, residual_samples, predictor_order, rice_parameter_limit, (uint32_t)po, params[!best_idx], &bits))
				break;
			sum += 1u << po;
			if(best_bits == 0 || bits < best_bits) {
				best_bits = bits;
				best_idx = !best_idx;
				best_po = (uint32_t)po;
			}
		}
	}
	plan->partition_order = (int32_t)best_po;
	plan->rice_method = 0;
	{
		uint32_t p;
		memset(plan->rice_params, 0, sizeof plan->rice_params);
		for(p = 0; p < (1u << best_po); p++) {
			plan->rice_params[p] = params[best_idx][p];
			if((uint32_t)params[best_idx][p] >= RICE_ESCAPE)
				plan->rice_method = 1;
		}
	}
	return best_bits;
}

/* ------------------------------------------------------------------ subframe candidate search */

static void plan_reset(fo_subframe_plan *p, uint32_t wasted, uint32_t bps)
{
	memset(p, 0, sizeof *p);
	p->wasted_bits = (int32_t)wasted;
	p->subframe_bps = (int32_t)bps;
}

/* stream_encoder.c:4489-4561 evaluate_fixed_subframe_ */
static uint32_t evaluate_fixed(fo_encoder *e, const int32_t *signal, uint32_t blocksize, uint32_t subframe_bps, uint32_t wasted, uint32_t order,
                               uint32_t rice_limit, uint32_t min_po, uint32_t max_po, fo_subframe_plan *plan)
{
	const uint32_t residual_samples = blocksize - order;
	uint32_t residual_bits, estimate;
	fixed_residual(signal + order, residual_samples, order, e->residual);
	plan_reset(plan, wasted, subframe_bps);
	plan->type = 2;
	plan->order = (int32_t)order;
	residual_bits = find_best_partition_order(e, e->residual, residual_samples, order, rice_limit, min_po, max_po, subframe_bps, plan);
	estimate = SUBFRAME_HEADER_BITS + wasted + order * subframe_bps;
	if(residual_bits < UINT32_MAX - estimate) estimate += residual_bits;
	else estimate = UINT32_MAX;
	plan->estimate_bits = estimate;
	return estimate;
}

/* stream_encoder.c:4564-4666 evaluate_lpc_subframe_, from :4600 on (the candidate was quantised by fo_lpc_candidates) */
static uint32_t evaluate_lpc(fo_encoder *e, const int32_t *signal, const fo_lpc_cand *c, uint32_t blocksize, uint32_t subframe_bps, uint32_t wasted,
                             uint32_t rice_limit, uint32_t min_po, uint32_t max_po, fo_subframe_plan *plan)
{
	const uint32_t order = (uint32_t)c->order, qlp_coeff_precision = (uint32_t)c->precision;
	const int32_t *qlp = c->qlp;
	const int quantization = c->shift;
	const uint32_t residual_samples = blocksize - order;
	uint32_t residual_bits, estimate;
	int limit;

	limit = fo_max_residual_bps(subframe_bps, qlp, order, quantization) > 32;
	if(limit) counters.limit++;
	if(limit || silog2((int64_t)fo_max_prediction_value_before_shift(subframe_bps, qlp, order)) > 32) counters.wide++;
	if(!lpc_residual(signal + order, residual_samples, qlp, order, quantization, e->residual, limit)) {
		counters.limit_rejected++;
		return 0;
	}

	plan_reset(plan, wasted, subframe_bps);
	plan->type = 3;
	plan->order = (int32_t)order;
	plan->qlp_precision = (int32_t)qlp_coeff_precision;
	plan->qlp_shift = quantization;
	plan->qlp_negative_shift = c->negative_shift;
	memcpy(plan->qlp_coeff, qlp, sizeof plan->qlp_coeff);
	residual_bits = find_best_partition_order(e, e->residual, residual_samples, order, rice_limit, min_po, max_po, subframe_bps, plan);

	estimate = SUBFRAME_HEADER_BITS + wasted + LPC_QLP_PRECISION_LEN + LPC_QLP_SHIFT_LEN + order * (qlp_coeff_precision + subframe_bps);
	if(residual_bits < UINT32_MAX - estimate) estimate += residual_bits;
	else estimate = UINT32_MAX;
	plan->estimate_bits = estimate;
	return estimate;
}

uint32_t fo_lpc_estimate(fo_encoder *e, const int32_t *signal, uint32_t blocksize, uint32_t subframe_bps, uint32_t wasted,
                         const fo_lpc_cand *c, uint32_t min_po, uint32_t max_po)
{
	fo_subframe_plan plan;
	if(blocksize > e->cfg.blocksize || c->order < 1 || (uint32_t)c->order >= blocksize) return 0;
	return evaluate_lpc(e, signal, c, blocksize, subframe_bps, wasted, e->cfg.bits_per_sample > 16 ? RICE2_ESCAPE : RICE_ESCAPE, min_po,
	                    max_po, &plan);
}

/* stream_encoder.c:4293-4316 set_next_subdivide_tukey */
static void next_subdivide_tukey(int32_t parts, uint32_t *a, uint32_t *depth, uint32_t *part)
{
	if(*depth == 2) {
		if(*part == 0) *part = 2;
		else { *part = 0; (*depth)++; }
	}
	else if(*part < (2 * (*depth) - 1)) (*part)++;
	else { *part = 0; (*depth)++; }
	if(*depth > (uint32_t)parts) { (*a)++; *depth = 1; *part = 0; }
}

typedef struct {
	uint32_t a, b, c;
	double autoc_root[FO_MAX_LPC_ORDER + 1];
	double autoc[FO_MAX_LPC_ORDER + 1];
} apod_state;

/* stream_encoder.c:4318-4392 apply_apodization_. Note the reference quirks kept here:
 * autoc_root copies only max_order entries (:4340) and the punch-out subtraction covers
 * only max_order entries (:4370-4371), so autoc[max_order] keeps the preceding partial
 * window's value. Each new autocorrelation has `lags` values (the reference's max_order + 1; fo_stage_a asks for as many
 * as the CUDA kernel computes). Returns 2 when it computed a new autocorrelation, 1 for a punch-out, 0 for a skipped part. */
static int apply_apodization(fo_encoder *e, apod_state *st, uint32_t blocksize, uint32_t max_order, uint32_t lags, const int32_t *signal)
{
	const fo_apodization *cur = &e->cfg.apodizations[st->a];
	const float *win = e->window[st->a];

	if(st->b == 1) {
		fo_window_data(signal, win, e->windowed, blocksize);
		fo_autocorrelation(e->windowed, blocksize, lags, st->autoc);
		if(cur->type == FO_APOD_SUBDIVIDE_TUKEY) {
			memcpy(st->autoc_root, st->autoc, max_order * sizeof(st->autoc[0]));
			st->b++;
		}
		else
			st->a++;
		return 2;
	}
	else {
		int made = 1;
		if(blocksize / st->b <= FO_MAX_LPC_ORDER) {
			next_subdivide_tukey(cur->parts, &st->a, &st->b, &st->c);
			return 0;
		}
		if(!(st->c % 2)) {
			fo_window_data_partial(signal, win, e->windowed, blocksize, blocksize / st->b / 2, (st->c / 2 * blocksize) / st->b);
			fo_autocorrelation(e->windowed, blocksize / st->b, lags, st->autoc);
			made = 2;
		}
		else {
			uint32_t i;
			for(i = 0; i < max_order; i++)
				st->autoc[i] = st->autoc_root[i] - st->autoc[i];
		}
		next_subdivide_tukey(cur->parts, &st->a, &st->b, &st->c);
		return made;
	}
}

/* stream_encoder.c:4376-4391 (the tail of apply_apodization_) and :4220-4260 + 4591-4599 (process_subframe_'s order and
 * precision loops, and the start of evaluate_lpc_subframe_ up to the quantisation) */
size_t fo_lpc_candidates(const double *autoc, uint32_t max_order, uint32_t subframe_bps, uint32_t blocksize, const fo_config *cfg,
                         fo_lpc_cand *out)
{
	float lp_coeff[FO_MAX_LPC_ORDER][FO_MAX_LPC_ORDER];
	double lpc_error[FO_MAX_LPC_ORDER];
	uint32_t min_lpc, lo, guess;
	size_t n = 0;

	if(autoc[0] == 0.0)
		return 0;
	fo_lp_coefficients(autoc, &max_order, lp_coeff, lpc_error);
	guess = fo_best_order(lpc_error, max_order, blocksize,
	                      subframe_bps + (cfg->do_qlp_coeff_prec_search ? MIN_QLP_PRECISION : cfg->qlp_coeff_precision));
	if(cfg->do_exhaustive_model_search) min_lpc = 1;
	else min_lpc = max_order = guess;
	for(lo = min_lpc; lo <= max_order; lo++) {
		uint32_t minp, maxp, prec;
		double lbps = expected_bits(lpc_error[lo - 1], blocksize - lo);
		if(lbps >= (double)subframe_bps) {
			counters.order_skipped++;
			memset(&out[n], 0, sizeof out[n]);
			out[n].status = FO_LPC_DONT_EVEN_TRY;
			out[n++].order = (int32_t)lo;
			continue;
		}
		if(cfg->do_qlp_coeff_prec_search) {
			minp = MIN_QLP_PRECISION;
			if(subframe_bps <= 17) {
				maxp = MINU(32 - subframe_bps - ilog2_64(lo), MAX_QLP_PRECISION);
				maxp = MAXU(maxp, minp);
			}
			else maxp = MAX_QLP_PRECISION;
		}
		else minp = maxp = cfg->qlp_coeff_precision;
		for(prec = minp; prec <= maxp; prec++) {
			fo_lpc_cand *c = &out[n++];
			uint32_t precision = prec;
			memset(c, 0, sizeof *c);
			if(subframe_bps <= 17 && 32 - subframe_bps - ilog2_64(lo) < precision) {
				precision = 32 - subframe_bps - ilog2_64(lo);
				counters.precision_capped++;
			}
			c->order = (int32_t)lo;
			c->precision_tried = (int32_t)prec;
			c->precision = (int32_t)precision;
			{
				const uint64_t neg = counters.negative_shift;
				c->status = fo_quantize_coefficients(lp_coeff[lo - 1], lo, precision, c->qlp, &c->shift);
				c->negative_shift = counters.negative_shift != neg;
			}
			if(c->status != FO_LPC_QUANTIZED) c->shift = 0;
		}
	}
	return n;
}

/* stream_encoder.c:4045-4290 process_subframe_: best-of-two search in evaluation order
 * verbatim -> constant | fixed -> LPC candidates, strict '<' keeps the earlier candidate. */
static uint32_t process_subframe(fo_encoder *e, const int32_t *signal, uint32_t blocksize, uint32_t subframe_bps, uint32_t wasted,
                                 uint32_t min_po, uint32_t max_po, int disable_constant, fo_subframe_plan *best)
{
	const fo_config *cfg = &e->cfg;
	const uint32_t rice_limit = cfg->bits_per_sample > 16 ? RICE2_ESCAPE : RICE_ESCAPE;
	float rbps[MAX_FIXED_ORDER + 1];
	uint32_t best_bits, cand_bits;
	fo_subframe_plan cand;

	/* verbatim baseline (:4669-4699) */
	plan_reset(best, wasted, subframe_bps);
	best->type = 1;
	if(cfg->disable_verbatim_subframes && blocksize >= MAX_FIXED_ORDER)
		best_bits = UINT32_MAX;
	else
		best_bits = SUBFRAME_HEADER_BITS + wasted + blocksize * subframe_bps;
	best->estimate_bits = best_bits;

	if(blocksize > MAX_FIXED_ORDER) {
		int signal_is_constant = 0;
		/* stream_encoder.c:4098-4103: the _wide routine is the one with an AVX2 version */
		const uint32_t dl = blocksize - MAX_FIXED_ORDER;
		const int wide_routine = subframe_bps < 28 && !(subframe_bps + ilog2_64((uint64_t)dl * 17) < 32);
		uint32_t guess_fixed_order = fixed_best_predictor(signal + MAX_FIXED_ORDER, dl, e->cfg.x86_avx2_fixed_guess && wide_routine, rbps);

		if(!disable_constant && rbps[1] == 0.0) {
			uint32_t i;
			signal_is_constant = 1;
			for(i = 1; i < blocksize; i++)
				if(signal[0] != signal[i]) { signal_is_constant = 0; break; }
		}
		if(signal_is_constant) {
			cand_bits = SUBFRAME_HEADER_BITS + wasted + subframe_bps; /* :4466-4487 */
			if(cand_bits < best_bits) {
				plan_reset(best, wasted, subframe_bps);
				best->type = 0;
				best->estimate_bits = cand_bits;
				best_bits = cand_bits;
			}
		}
		else {
			if(!cfg->disable_fixed_subframes || (cfg->max_lpc_order == 0 && best_bits == UINT32_MAX)) {
				uint32_t min_fixed, max_fixed, fo;
				if(cfg->do_exhaustive_model_search) { min_fixed = 0; max_fixed = MAX_FIXED_ORDER; }
				else min_fixed = max_fixed = guess_fixed_order;
				if(max_fixed >= blocksize) max_fixed = blocksize - 1;
				for(fo = min_fixed; fo <= max_fixed; fo++) {
					if(rbps[fo] >= (float)subframe_bps)
						continue;
					cand_bits = evaluate_fixed(e, signal, blocksize, subframe_bps, wasted, fo, rice_limit, min_po, max_po, &cand);
					if(cand_bits < best_bits) { *best = cand; best_bits = cand_bits; }
				}
			}
			if(cfg->max_lpc_order > 0) {
				uint32_t max_lpc_order = cfg->max_lpc_order >= blocksize ? blocksize - 1 : cfg->max_lpc_order;
				if(max_lpc_order > 0) {
					apod_state st;
					memset(&st, 0, sizeof st);
					st.a = 0; st.b = 1; st.c = 0;
					while(st.a < cfg->num_apodizations) {
						size_t n, i;
						if(!apply_apodization(e, &st, blocksize, max_lpc_order, max_lpc_order + 1, signal))
							continue;
						n = fo_lpc_candidates(st.autoc, max_lpc_order, subframe_bps, blocksize, cfg, e->lpc_cands);
						for(i = 0; i < n; i++) {
							if(e->lpc_cands[i].status != FO_LPC_QUANTIZED)
								continue;
							cand_bits = evaluate_lpc(e, signal, &e->lpc_cands[i], blocksize, subframe_bps, wasted, rice_limit, min_po, max_po, &cand);
							if(cand_bits > 0 && cand_bits < best_bits) { *best = cand; best_bits = cand_bits; }
						}
					}
				}
			}
		}
	}
	if(best_bits == UINT32_MAX) {
		plan_reset(best, wasted, subframe_bps);
		best->type = 1;
		best_bits = SUBFRAME_HEADER_BITS + wasted + blocksize * subframe_bps;
		best->estimate_bits = best_bits;
	}
	return best_bits;
}

/* stream_encoder.c:5077-5099 get_wasted_bits_ (shifts in place) */
static uint32_t get_wasted_bits(int32_t *signal, uint32_t samples)
{
	uint32_t i, shift;
	int32_t x = 0;
	for(i = 0; i < samples && !(x & 1); i++)
		x |= signal[i];
	if(x == 0) shift = 0;
	else for(shift = 0; !(x & 1); shift++) x >>= 1;
	if(shift > 0)
		for(i = 0; i < samples; i++)
			signal[i] >>= shift;
	return shift;
}

/* ------------------------------------------------------------------ frame emission */

/* stream_encoder_framing.c:245-391 FLAC__frame_add_header */
static void write_frame_header(bitw *bw, const fo_config *cfg, uint32_t blocksize, uint32_t channel_assignment, uint32_t frame_number)
{
	uint32_t u, blocksize_hint = 0, sample_rate_hint = 0;
	const size_t start_byte = (size_t)(bw->bits >> 3);
	bw_write(bw, 0x3ffe, 14);
	bw_write(bw, 0, 1);
	bw_write(bw, 0, 1); /* fixed blocksize stream: frame number */
	switch(blocksize) {
		case 192: u = 1; break; case 576: u = 2; break; case 1152: u = 3; break; case 2304: u = 4; break;
		case 4608: u = 5; break; case 256: u = 8; break; case 512: u = 9; break; case 1024: u = 10; break;
		case 2048: u = 11; break; case 4096: u = 12; break; case 8192: u = 13; break; case 16384: u = 14; break;
		case 32768: u = 15; break;
		default: blocksize_hint = u = (blocksize <= 0x100) ? 6 : 7; break;
	}
	bw_write(bw, u, 4);
	switch(cfg->sample_rate) {
		case 88200: u = 1; break; case 176400: u = 2; break; case 192000: u = 3; break; case 8000: u = 4; break;
		case 16000: u = 5; break; case 22050: u = 6; break; case 24000: u = 7; break; case 32000: u = 8; break;
		case 44100: u = 9; break; case 48000: u = 10; break; case 96000: u = 11; break;
		default:
			if(cfg->sample_rate <= 255000 && cfg->sample_rate % 1000 == 0) sample_rate_hint = u = 12;
			else if(cfg->sample_rate <= 655350 && cfg->sample_rate % 10 == 0) sample_rate_hint = u = 14;
			else if(cfg->sample_rate <= 0xffff) sample_rate_hint = u = 13;
			else u = 0;
			break;
	}
	bw_write(bw, u, 4);
	switch(channel_assignment) {
		case 0: u = cfg->channels - 1; break;
		case 1: u = 8; break;
		case 2: u = 9; break;
		default: u = 10; break;
	}
	bw_write(bw, u, 4);
	switch(cfg->bits_per_sample) {
		case 8: u = 1; break; case 12: u = 2; break; case 16: u = 4; break; case 20: u = 5; break;
		case 24: u = 6; break; case 32: u = 7; break; default: u = 0; break;
	}
	bw_write(bw, u, 3);
	bw_write(bw, 0, 1);
	bw_write_utf8(bw, frame_number);
	if(blocksize_hint)
		bw_write(bw, blocksize - 1, (blocksize_hint == 6) ? 8 : 16);
	switch(sample_rate_hint) {
		case 12: bw_write(bw, cfg->sample_rate / 1000, 8); break;
		case 13: bw_write(bw, cfg->sample_rate, 16); break;
		case 14: bw_write(bw, cfg->sample_rate / 10, 16); break;
	}
	bw_write(bw, fo_crc8(bw->buf + start_byte, (size_t)(bw->bits >> 3) - start_byte), 8);
}

/* stream_encoder_framing.c:538-594 add_residual_partitioned_rice_ (raw_bits == 0 everywhere) */
static void write_residual(bitw *bw, const int32_t *residual, uint32_t residual_samples, uint32_t predictor_order, const fo_subframe_plan *p)
{
	const uint32_t plen = p->rice_method ? RICE2_PARAM_LEN : RICE_PARAM_LEN;
	const uint32_t po = (uint32_t)p->partition_order;
	const uint32_t default_partition_samples = (residual_samples + predictor_order) >> po;
	uint32_t i, j, k = 0, k_last = 0;
	bw_write(bw, (uint32_t)p->rice_method, ENTROPY_TYPE_LEN);
	bw_write(bw, po, RICE_ORDER_LEN);
	for(i = 0; i < (1u << po); i++) {
		uint32_t partition_samples = default_partition_samples;
		if(i == 0) partition_samples -= predictor_order;
		k += partition_samples;
		bw_write(bw, (uint32_t)p->rice_params[i], plen);
		for(j = k_last; j < k; j++)
			bw_write_rice(bw, residual[j], (uint32_t)p->rice_params[i]);
		k_last = k;
	}
}

/* stream_encoder_framing.c:393-520 FLAC__subframe_add_{constant,verbatim,fixed,lpc} */
static void write_subframe(fo_encoder *e, bitw *bw, const int32_t *signal, uint32_t blocksize, const fo_subframe_plan *p)
{
	const uint32_t bps = (uint32_t)p->subframe_bps, w = (uint32_t)p->wasted_bits, order = (uint32_t)p->order;
	uint32_t i;
	switch(p->type) {
		case 0: bw_write(bw, 0x00 | (w ? 1 : 0), 8); break;
		case 1: bw_write(bw, 0x02 | (w ? 1 : 0), 8); break;
		case 2: bw_write(bw, 0x10 | (order << 1) | (w ? 1 : 0), 8); break;
		default: bw_write(bw, 0x40 | ((order - 1) << 1) | (w ? 1 : 0), 8); break;
	}
	if(w) bw_write_unary(bw, w - 1);
	switch(p->type) {
		case 0:
			bw_write_signed(bw, signal[0], bps);
			break;
		case 1:
			for(i = 0; i < blocksize; i++) bw_write_signed(bw, signal[i], bps);
			break;
		case 2:
			for(i = 0; i < order; i++) bw_write_signed(bw, signal[i], bps);
			fixed_residual(signal + order, blocksize - order, order, e->residual);
			write_residual(bw, e->residual, blocksize - order, order, p);
			break;
		default:
			for(i = 0; i < order; i++) bw_write_signed(bw, signal[i], bps);
			bw_write(bw, (uint32_t)p->qlp_precision - 1, LPC_QLP_PRECISION_LEN);
			bw_write_signed(bw, p->qlp_shift, LPC_QLP_SHIFT_LEN);
			for(i = 0; i < order; i++) bw_write_signed(bw, p->qlp_coeff[i], (uint32_t)p->qlp_precision);
			lpc_residual(signal + order, blocksize - order, p->qlp_coeff, order, p->qlp_shift, e->residual, 0);
			write_residual(bw, e->residual, blocksize - order, order, p);
			break;
	}
}

/* ------------------------------------------------------------------ encoder object */

void fo_config_preset(fo_config *cfg, uint32_t channels, uint32_t bps, uint32_t sample_rate, uint32_t level, uint32_t blocksize)
{
	/* stream_encoder.c:117-140 compression_levels_ */
	static const struct { int ms, loose; uint32_t lpc, maxpo; int parts; } L[9] = {
		{0, 0, 0, 3, 0}, {1, 1, 0, 3, 0}, {1, 0, 0, 3, 0}, {0, 0, 6, 4, 0}, {1, 1, 8, 4, 0},
		{1, 0, 8, 5, 0}, {1, 0, 8, 6, 2}, {1, 0, 12, 6, 2}, {1, 0, 12, 6, 3}};
	if(level > 8) level = 8;
	memset(cfg, 0, sizeof *cfg);
	cfg->channels = channels; cfg->bits_per_sample = bps; cfg->sample_rate = sample_rate; cfg->blocksize = blocksize;
	cfg->do_mid_side = L[level].ms; cfg->loose_mid_side = L[level].loose;
	cfg->max_lpc_order = L[level].lpc;
	cfg->max_residual_partition_order = L[level].maxpo;
	cfg->num_apodizations = 1;
	if(L[level].parts) {
		/* stream_encoder.c:2040-2053: p = 5e-1 (as float) / parts */
		float p = 5e-1;
		cfg->apodizations[0].type = FO_APOD_SUBDIVIDE_TUKEY;
		cfg->apodizations[0].parts = L[level].parts;
		cfg->apodizations[0].p = p / L[level].parts;
	}
	else {
		cfg->apodizations[0].type = FO_APOD_TUKEY;
		cfg->apodizations[0].p = 0.5f;
	}
}

fo_encoder *fo_encoder_new(const fo_config *cfg_in)
{
	fo_encoder *e;
	fo_config *cfg;
	uint32_t i;
	crc_init();
	e = (fo_encoder *)calloc(1, sizeof *e);
	if(!e) return NULL;
	e->cfg = *cfg_in;
	cfg = &e->cfg;
	/* stream_encoder.c:725-830 init_stream_internal_ validation and defaults */
	if(cfg->channels == 0 || cfg->channels > FO_MAX_CHANNELS) goto fail;
	if(cfg->channels != 2) { cfg->do_mid_side = 0; cfg->loose_mid_side = 0; }
	else if(!cfg->do_mid_side) cfg->loose_mid_side = 0;
	if(cfg->bits_per_sample < 4 || cfg->bits_per_sample > 24) goto fail; /* oracle scope: <= 24 */
	if(cfg->blocksize == 0) cfg->blocksize = cfg->max_lpc_order == 0 ? 1152 : 4096;
	if(cfg->blocksize < 16 || cfg->blocksize > 65535) goto fail;
	if(cfg->max_lpc_order > FO_MAX_LPC_ORDER) goto fail;
	if(cfg->blocksize < cfg->max_lpc_order) goto fail;
	if(cfg->qlp_coeff_precision == 0) {
		if(cfg->bits_per_sample < 16)
			cfg->qlp_coeff_precision = MAXU(MIN_QLP_PRECISION, 2 + cfg->bits_per_sample / 2);
		else if(cfg->bits_per_sample == 16) {
			if(cfg->blocksize <= 192) cfg->qlp_coeff_precision = 7;
			else if(cfg->blocksize <= 384) cfg->qlp_coeff_precision = 8;
			else if(cfg->blocksize <= 576) cfg->qlp_coeff_precision = 9;
			else if(cfg->blocksize <= 1152) cfg->qlp_coeff_precision = 10;
			else if(cfg->blocksize <= 2304) cfg->qlp_coeff_precision = 11;
			else if(cfg->blocksize <= 4608) cfg->qlp_coeff_precision = 12;
			else cfg->qlp_coeff_precision = 13;
		}
		else {
			if(cfg->blocksize <= 384) cfg->qlp_coeff_precision = MAX_QLP_PRECISION - 2;
			else if(cfg->blocksize <= 1152) cfg->qlp_coeff_precision = MAX_QLP_PRECISION - 1;
			else cfg->qlp_coeff_precision = MAX_QLP_PRECISION;
		}
	}
	else if(cfg->qlp_coeff_precision < MIN_QLP_PRECISION || cfg->qlp_coeff_precision > MAX_QLP_PRECISION) goto fail;
	if(cfg->max_residual_partition_order >= (1u << RICE_ORDER_LEN)) cfg->max_residual_partition_order = (1u << RICE_ORDER_LEN) - 1;
	if(cfg->max_residual_partition_order > 8) goto fail; /* oracle scope: FO_MAX_PARTITIONS */
	if(cfg->min_residual_partition_order >= cfg->max_residual_partition_order) cfg->min_residual_partition_order = cfg->max_residual_partition_order;
	if(cfg->num_apodizations == 0 || cfg->num_apodizations > FO_MAX_APODIZATIONS) goto fail;

	for(i = 0; i < 4; i++) {
		e->sig[i] = (int32_t *)malloc(sizeof(int32_t) * (cfg->blocksize + 8));
		if(!e->sig[i]) goto fail;
	}
	for(i = 0; i < cfg->channels; i++) {
		e->chan[i] = (int32_t *)malloc(sizeof(int32_t) * (cfg->blocksize + 8));
		if(!e->chan[i]) goto fail;
	}
	for(i = 0; i < cfg->num_apodizations; i++) {
		e->window[i] = (float *)malloc(sizeof(float) * cfg->blocksize);
		if(!e->window[i]) goto fail;
	}
	e->residual = (int32_t *)malloc(sizeof(int32_t) * (cfg->blocksize + 8));
	e->windowed = (float *)malloc(sizeof(float) * (cfg->blocksize + 8));
	e->psums = (uint64_t *)malloc(sizeof(uint64_t) * 2 * FO_MAX_PARTITIONS);
	if(!e->residual || !e->windowed || !e->psums) goto fail;
	e->win_blocksize = 0;
	return e;
fail:
	fo_encoder_delete(e);
	return NULL;
}

void fo_encoder_delete(fo_encoder *e)
{
	uint32_t i;
	if(!e) return;
	for(i = 0; i < 4; i++) free(e->sig[i]);
	for(i = 0; i < FO_MAX_CHANNELS; i++) free(e->chan[i]);
	for(i = 0; i < FO_MAX_APODIZATIONS; i++) free(e->window[i]);
	free(e->residual); free(e->windowed); free(e->psums);
	free(e);
}

const fo_config *fo_encoder_config(const fo_encoder *e) { return &e->cfg; }

/* stream_encoder.c:2915-2975 (resize_buffers_): window tables follow the blocksize,
 * both TUKEY and SUBDIVIDE_TUKEY use FLAC__window_tukey(window, blocksize, p). */
static void ensure_windows(fo_encoder *e, uint32_t blocksize)
{
	uint32_t i;
	if(e->win_blocksize == blocksize) return;
	if(e->cfg.max_lpc_order > 0 && blocksize > 1)
		for(i = 0; i < e->cfg.num_apodizations; i++)
			fo_window(&e->cfg.apodizations[i], e->window[i], (int32_t)blocksize);
	e->win_blocksize = blocksize;
}

/* stream_encoder.c:3777-3867: the channels (e->chan), mid and side (e->sig[2], e->sig[3]) when the block codes them, the
 * loose mid-side decision, and each coded signal's wasted bits shifted out in place with its subframe bps */
static void form_signals(fo_encoder *e, const int32_t *interleaved, uint32_t blocksize, int *do_independent_out, int *do_mid_side_out,
                         uint32_t *channel_assignment, uint32_t wasted[], uint32_t sbps[], uint32_t ms_wasted[2], uint32_t ms_bps[2])
{
	const fo_config *cfg = &e->cfg;
	const uint32_t ch = cfg->channels, bps = cfg->bits_per_sample;
	int do_independent, do_mid_side;
	uint32_t c, i;

	*channel_assignment = 0;
	for(c = 0; c < ch; c++)
		for(i = 0; i < blocksize; i++)
			e->chan[c][i] = interleaved[(size_t)i * ch + c];

	if(cfg->do_mid_side) {
		if(cfg->loose_mid_side) {
			uint64_t sumAbsLR = 0, sumAbsMS = 0;
			for(i = 1; i < blocksize; i++) {
				int32_t pl = e->chan[0][i] - e->chan[0][i - 1];
				int32_t pr = e->chan[1][i] - e->chan[1][i - 1];
				sumAbsLR += (uint64_t)(abs(pl) + abs(pr));
				sumAbsMS += (uint64_t)(abs((pl + pr) >> 1) + abs(pl - pr));
			}
			if(sumAbsLR < sumAbsMS) { do_independent = 1; do_mid_side = 0; *channel_assignment = 0; }
			else { do_independent = 0; do_mid_side = 1; *channel_assignment = 3; }
		}
		else { do_independent = 1; do_mid_side = 1; }
	}
	else { do_independent = 1; do_mid_side = 0; }

	if(do_mid_side) {
		for(i = 0; i < blocksize; i++) {
			e->sig[3][i] = e->chan[0][i] - e->chan[1][i];
			e->sig[2][i] = (e->chan[0][i] + e->chan[1][i]) >> 1;
		}
	}
	if(do_independent) {
		for(c = 0; c < ch; c++) {
			uint32_t w = get_wasted_bits(e->chan[c], blocksize);
			if(w > bps) w = bps;
			wasted[c] = w;
			sbps[c] = bps - w;
		}
	}
	if(do_mid_side) {
		for(c = 0; c < 2; c++) {
			uint32_t w = get_wasted_bits(e->sig[2 + c], blocksize);
			if(w > bps) w = bps;
			ms_wasted[c] = w;
			ms_bps[c] = bps - w + (c == 0 ? 0 : 1);
		}
	}
	*do_independent_out = do_independent;
	*do_mid_side_out = do_mid_side;
}

int fo_stage_a(fo_encoder *e, const int32_t *interleaved, uint32_t nblocks, uint32_t lags, uint32_t lag_stride, int unshifted,
               double *rows, size_t rows_cap, int32_t *meta, uint32_t *sigor)
{
	const fo_config *cfg = &e->cfg;
	const uint32_t bs = cfg->blocksize, ch = cfg->channels, nsig = ch + (cfg->do_mid_side ? 2u : 0u);
	const size_t nitems = (size_t)nblocks * nsig;
	uint32_t max_order, nsec = 0, a, b, blk, s, i;
	int32_t *x;

	if(cfg->max_lpc_order == 0 || bs < 2 || lags < 1 || lags > FO_MAX_LPC_ORDER + 1 || lag_stride < lags) return -1;
	for(a = 0; a < cfg->num_apodizations; a++) {
		nsec++;
		if(cfg->apodizations[a].type == FO_APOD_SUBDIVIDE_TUKEY)
			for(b = 2; b <= (uint32_t)cfg->apodizations[a].parts; b++)
				if(bs / b > FO_MAX_LPC_ORDER) nsec += b == 2 ? 2 : b;
	}
	if((size_t)nsec * nitems * lag_stride > rows_cap) return -1;
	max_order = cfg->max_lpc_order >= bs ? bs - 1 : cfg->max_lpc_order;
	x = (int32_t *)malloc(sizeof(int32_t) * bs);
	if(!x) return -1;
	memset(rows, 0, sizeof(double) * (size_t)nsec * nitems * lag_stride);
	ensure_windows(e, bs);
	for(blk = 0; blk < nblocks; blk++) {
		int do_independent, do_mid_side;
		uint32_t ca, wasted[FO_MAX_CHANNELS], sbps[FO_MAX_CHANNELS], ms_wasted[2], ms_bps[2];
		form_signals(e, interleaved + (size_t)blk * bs * ch, bs, &do_independent, &do_mid_side, &ca, wasted, sbps, ms_wasted, ms_bps);
		for(s = 0; s < nsig; s++) {
			const size_t item = (size_t)blk * nsig + s;
			const int ms = s >= ch;
			const int32_t *sig = ms ? e->sig[2 + s - ch] : e->chan[s];
			const uint32_t w = ms ? ms_wasted[s - ch] : wasted[s];
			uint32_t o = 0, sec = 0;
			apod_state st;
			meta[2 * item] = 0;
			meta[2 * item + 1] = 0;
			sigor[item] = 0;
			if(!(ms ? do_mid_side : do_independent)) continue;
			meta[2 * item] = (int32_t)w;
			meta[2 * item + 1] = (int32_t)(ms ? ms_bps[s - ch] : sbps[s]);
			for(i = 0; i < bs; i++) {
				x[i] = (int32_t)((uint32_t)sig[i] << w);  /* the signal before get_wasted_bits shifted its w zero bits out */
				o |= (uint32_t)x[i];
			}
			sigor[item] = o;
			memset(&st, 0, sizeof st);
			st.b = 1;
			while(st.a < cfg->num_apodizations)
				if(apply_apodization(e, &st, bs, max_order, lags, unshifted ? x : sig) == 2) {
					if(sec == nsec) { free(x); return -1; }
					memcpy(rows + ((size_t)sec * nitems + item) * lag_stride, st.autoc, lags * sizeof(double));
					sec++;
				}
		}
	}
	free(x);
	return (int)nsec;
}

/* stream_encoder.c:3747-4043 process_subframes_ + :3435-3480 process_frame_ (pad, CRC-16) */
size_t fo_encode_frame(fo_encoder *e, const int32_t *interleaved, uint32_t blocksize, uint32_t frame_number,
                       uint8_t *out, size_t out_cap, fo_frame_plan *plan_out)
{
	const fo_config *cfg = &e->cfg;
	const uint32_t ch = cfg->channels;
	uint32_t min_po = cfg->min_residual_partition_order, max_po;
	int do_independent, do_mid_side, all_constant = 1, disable_constant = cfg->disable_constant_subframes;
	uint32_t channel_assignment = 0, c;
	fo_subframe_plan plans[FO_MAX_CHANNELS], ms_plans[2];
	uint32_t bits[FO_MAX_CHANNELS], ms_bits[2] = {0, 0};
	uint32_t wasted[FO_MAX_CHANNELS], sbps[FO_MAX_CHANNELS], ms_wasted[2], ms_bps[2];
	bitw bw;

	if(blocksize == 0 || blocksize > cfg->blocksize) return 0;
	ensure_windows(e, blocksize);

	max_po = max_rice_partition_order_from_blocksize(blocksize);
	max_po = MINU(max_po, cfg->max_residual_partition_order);
	min_po = MINU(min_po, max_po);

	form_signals(e, interleaved, blocksize, &do_independent, &do_mid_side, &channel_assignment, wasted, sbps, ms_wasted, ms_bps);
	if(plan_out) memset(plan_out, 0, sizeof *plan_out);

	if(do_independent) {
		for(c = 0; c < ch; c++) {
			if(cfg->limit_min_bitrate && all_constant && (c + 1) == ch)
				disable_constant = 1;
			bits[c] = process_subframe(e, e->chan[c], blocksize, sbps[c], wasted[c], min_po, max_po, disable_constant, &plans[c]);
			if(plans[c].type != 0) all_constant = 0;
			if(plan_out && ch == 2) { plan_out->cand[c] = plans[c]; plan_out->cand_valid[c] = 1; }
		}
	}
	if(do_mid_side) {
		for(c = 0; c < 2; c++) {
			ms_bits[c] = process_subframe(e, e->sig[2 + c], blocksize, ms_bps[c], ms_wasted[c], min_po, max_po, disable_constant, &ms_plans[c]);
			if(plan_out) { plan_out->cand[2 + c] = ms_plans[c]; plan_out->cand_valid[2 + c] = 1; }
		}
	}

	bw_init(&bw, out, out_cap);
	if((do_independent && do_mid_side) || cfg->loose_mid_side) {
		const int32_t *lsig, *rsig;
		const fo_subframe_plan *lp, *rp;
		if(!cfg->loose_mid_side) {
			uint32_t b[4], min_bits, ca;
			b[0] = bits[0] + bits[1];
			b[1] = bits[0] + ms_bits[1];
			b[2] = bits[1] + ms_bits[1];
			b[3] = ms_bits[0] + ms_bits[1];
			channel_assignment = 0; min_bits = b[0];
			for(ca = 1; ca <= 3; ca++)
				if(b[ca] < min_bits) { min_bits = b[ca]; channel_assignment = ca; }
		}
		write_frame_header(&bw, cfg, blocksize, channel_assignment, frame_number);
		switch(channel_assignment) {
			case 0: lsig = e->chan[0]; lp = &plans[0]; rsig = e->chan[1]; rp = &plans[1]; break;
			case 1: lsig = e->chan[0]; lp = &plans[0]; rsig = e->sig[3]; rp = &ms_plans[1]; break;
			case 2: lsig = e->sig[3]; lp = &ms_plans[1]; rsig = e->chan[1]; rp = &plans[1]; break;
			default: lsig = e->sig[2]; lp = &ms_plans[0]; rsig = e->sig[3]; rp = &ms_plans[1]; break;
		}
		write_subframe(e, &bw, lsig, blocksize, lp);
		write_subframe(e, &bw, rsig, blocksize, rp);
		if(plan_out) { plan_out->sub[0] = *lp; plan_out->sub[1] = *rp; }
	}
	else {
		write_frame_header(&bw, cfg, blocksize, 0, frame_number);
		for(c = 0; c < ch; c++) {
			write_subframe(e, &bw, e->chan[c], blocksize, &plans[c]);
			if(plan_out) plan_out->sub[c] = plans[c];
		}
	}
	if(plan_out) plan_out->channel_assignment = (int32_t)channel_assignment;

	/* zero-pad to byte boundary, CRC-16 of everything (stream_encoder.c:3465-3480) */
	bw.bits = (bw.bits + 7) & ~(uint64_t)7;
	if(bw.overflow || (bw.bits >> 3) + 2 > out_cap) return 0;
	{
		const size_t n = (size_t)(bw.bits >> 3);
		const uint16_t crc = fo_crc16(out, n);
		out[n] = (uint8_t)(crc >> 8);
		out[n + 1] = (uint8_t)(crc & 0xff);
		return n + 2;
	}
}

int fo_encode_stream(fo_encoder *e, const int32_t *interleaved, uint64_t samples_per_channel,
                     uint8_t *out, size_t out_cap, size_t *out_len,
                     uint32_t *frame_sizes, size_t max_frames, size_t *nframes)
{
	const uint32_t bs = e->cfg.blocksize, ch = e->cfg.channels;
	uint64_t done = 0;
	size_t pos = 0, nf = 0;
	while(done < samples_per_channel) {
		const uint32_t n = (uint32_t)MINU((uint64_t)bs, samples_per_channel - done);
		const size_t len = fo_encode_frame(e, interleaved + done * ch, n, (uint32_t)nf, out + pos, out_cap - pos, NULL);
		if(len == 0) return -1;
		if(nf < max_frames && frame_sizes) frame_sizes[nf] = (uint32_t)len;
		nf++;
		pos += len;
		done += n;
	}
	if(out_len) *out_len = pos;
	if(nframes) *nframes = nf;
	return 0;
}

/* ================================================================== decode */

typedef struct {
	const uint8_t *buf;
	size_t len;      /* bytes */
	uint64_t pos;    /* bits */
	int err;
} bitr;

static uint64_t br_read(bitr *br, uint32_t nbits)
{
	uint64_t v = 0;
	while(nbits) {
		const size_t byte = (size_t)(br->pos >> 3);
		const uint32_t avail = 8 - (uint32_t)(br->pos & 7);
		const uint32_t take = nbits < avail ? nbits : avail;
		if(byte >= br->len) { br->err = 1; return 0; }
		v = (v << take) | ((br->buf[byte] >> (avail - take)) & ((1u << take) - 1u));
		br->pos += take;
		nbits -= take;
	}
	return v;
}

static int64_t br_read_signed(bitr *br, uint32_t nbits)
{
	uint64_t v = br_read(br, nbits);
	if(nbits < 64 && (v >> (nbits - 1)) & 1)
		v |= ~(uint64_t)0 << nbits;
	return (int64_t)v;
}

/* bitreader.c:725 FLAC__bitreader_read_unary_unsigned */
static uint32_t br_read_unary(bitr *br)
{
	uint32_t n = 0;
	while(!br->err && br_read(br, 1) == 0) n++;
	return n;
}

/* stream_decoder.c:3299-3357 read_residual_partitioned_rice_ + bitreader_read_rice_signed_block.c */
static int read_residual(bitr *br, uint32_t blocksize, uint32_t predictor_order, int32_t *residual)
{
	const uint32_t method = (uint32_t)br_read(br, 2);
	uint32_t po, partitions, p, sample = 0, plen, esc;
	if(method > 1) return 0;
	plen = method ? 5 : 4; esc = method ? 31 : 15;
	po = (uint32_t)br_read(br, 4);
	partitions = 1u << po;
	if((blocksize >> po) < predictor_order || (po > 0 && (blocksize % partitions) != 0)) return 0;
	for(p = 0; p < partitions; p++) {
		uint32_t n = (po == 0) ? blocksize - predictor_order : ((p == 0) ? (blocksize >> po) - predictor_order : (blocksize >> po));
		const uint32_t k = (uint32_t)br_read(br, plen);
		uint32_t i;
		if(k < esc) {
			for(i = 0; i < n; i++) {
				const uint32_t q = br_read_unary(br);
				/* a quotient that does not fit 32 bits with its k low bits fails the frame (bitreader_read_rice_signed_block.c:17,69) */
				if(k && q > (UINT32_MAX >> k)) return 0;
				const uint32_t u = (q << k) | (k ? (uint32_t)br_read(br, k) : 0);
				residual[sample++] = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
				if(br->err) return 0;
			}
		}
		else {
			const uint32_t raw = (uint32_t)br_read(br, 5);
			for(i = 0; i < n; i++)
				residual[sample++] = raw ? (int32_t)br_read_signed(br, raw) : 0;
		}
		if(br->err) return 0;
	}
	return 1;
}

/* stream_decoder.c:2949-3297 read_subframe_* ; lpc.c:978-1491 / fixed.c:571-629 restore */
static int read_subframe(bitr *br, uint32_t blocksize, uint32_t bps, int64_t *out, int32_t *residual)
{
	uint32_t x = (uint32_t)br_read(br, 8), wasted = 0, i;
	if(x & 0x80) return 0;
	if(x & 1) {
		wasted = br_read_unary(br) + 1;
		if(wasted >= bps) return 0;
		bps -= wasted;
	}
	x &= 0xfe;
	if(x == 0) {
		const int64_t v = br_read_signed(br, bps);
		for(i = 0; i < blocksize; i++) out[i] = v;
	}
	else if(x == 2) {
		for(i = 0; i < blocksize; i++) out[i] = br_read_signed(br, bps);
	}
	else if(x >= 16 && x <= 24) {
		const uint32_t order = (x >> 1) & 7;
		if(order > 4 || blocksize <= order) return 0;
		for(i = 0; i < order; i++) out[i] = br_read_signed(br, bps);
		if(!read_residual(br, blocksize, order, residual)) return 0;
		for(i = order; i < blocksize; i++) {
			const int64_t r = residual[i - order];
			switch(order) {
				case 0: out[i] = r; break;
				case 1: out[i] = r + out[i - 1]; break;
				case 2: out[i] = r + 2 * out[i - 1] - out[i - 2]; break;
				case 3: out[i] = r + 3 * out[i - 1] - 3 * out[i - 2] + out[i - 3]; break;
				default: out[i] = r + 4 * out[i - 1] - 6 * out[i - 2] + 4 * out[i - 3] - out[i - 4]; break;
			}
		}
	}
	else if(x >= 64) {
		const uint32_t order = ((x >> 1) & 31) + 1;
		int32_t qlp[32];
		uint32_t prec;
		int shift;
		if(blocksize <= order) return 0;
		for(i = 0; i < order; i++) out[i] = br_read_signed(br, bps);
		prec = (uint32_t)br_read(br, 4);
		if(prec == 15) return 0;
		prec++;
		shift = (int)br_read_signed(br, 5);
		if(shift < 0) return 0;
		for(i = 0; i < order; i++) qlp[i] = (int32_t)br_read_signed(br, prec);
		if(!read_residual(br, blocksize, order, residual)) return 0;
		for(i = order; i < blocksize; i++) {
			int64_t sum = 0;
			uint32_t j;
			for(j = 0; j < order; j++) sum += (int64_t)qlp[j] * out[i - 1 - j];
			out[i] = residual[i - order] + (sum >> shift);
		}
	}
	else
		return 0;
	if(wasted)
		for(i = 0; i < blocksize; i++) out[i] = (int64_t)((uint64_t)out[i] << wasted);
	return br->err ? 0 : 1;
}

/* stream_decoder.c:2373-2622 read_frame_, :2624-2947 read_frame_header_, :3476-3527 undo_channel_coding */
size_t fo_decode_frame(const uint8_t *data, size_t len, const fo_streaminfo *si,
                       int32_t *out_interleaved, size_t out_cap, uint32_t *blocksize_out, uint32_t *channels_out, uint32_t *bps_out, uint64_t *number_out)
{
	bitr br;
	uint32_t bs_code, sr_code, ca_code, bps_code, blocksize, channels, bps, variable, c, i;
	uint64_t number = 0;
	int64_t *chan[FO_MAX_CHANNELS] = {0};
	int32_t *residual = NULL;
	size_t consumed = 0;
	crc_init();
	br.buf = data; br.len = len; br.pos = 0; br.err = 0;

	if(br_read(&br, 14) != 0x3ffe) return 0;
	if(br_read(&br, 1) != 0) return 0;
	variable = (uint32_t)br_read(&br, 1);
	bs_code = (uint32_t)br_read(&br, 4);
	sr_code = (uint32_t)br_read(&br, 4);
	ca_code = (uint32_t)br_read(&br, 4);
	bps_code = (uint32_t)br_read(&br, 3);
	if(br_read(&br, 1) != 0) return 0;
	{   /* UTF-8 coded frame/sample number (bitreader.c:935-1039) */
		uint32_t first = (uint32_t)br_read(&br, 8), n;
		if(!(first & 0x80)) { number = first; n = 0; }
		else if((first & 0xE0) == 0xC0) { number = first & 0x1F; n = 1; }
		else if((first & 0xF0) == 0xE0) { number = first & 0x0F; n = 2; }
		else if((first & 0xF8) == 0xF0) { number = first & 0x07; n = 3; }
		else if((first & 0xFC) == 0xF8) { number = first & 0x03; n = 4; }
		else if((first & 0xFE) == 0xFC) { number = first & 0x01; n = 5; }
		else if(first == 0xFE && variable) { number = 0; n = 6; }
		else return 0;
		while(n--) {
			uint32_t b = (uint32_t)br_read(&br, 8);
			if((b & 0xC0) != 0x80) return 0;
			number = (number << 6) | (b & 0x3F);
		}
	}
	switch(bs_code) {
		case 0: return 0;
		case 1: blocksize = 192; break;
		case 2: case 3: case 4: case 5: blocksize = 576u << (bs_code - 2); break;
		case 6: blocksize = (uint32_t)br_read(&br, 8) + 1; break;
		case 7: blocksize = (uint32_t)br_read(&br, 16) + 1; break;
		default: blocksize = 256u << (bs_code - 8); break;
	}
	if(sr_code == 12) (void)br_read(&br, 8);
	else if(sr_code == 13 || sr_code == 14) (void)br_read(&br, 16);
	else if(sr_code == 15) return 0;
	{
		const size_t hdr_bytes = (size_t)(br.pos >> 3);
		const uint8_t crc = (uint8_t)br_read(&br, 8);
		if(br.err || fo_crc8(data, hdr_bytes) != crc) return 0;
	}
	if(ca_code < 8) channels = ca_code + 1;
	else if(ca_code <= 10) channels = 2;
	else return 0;
	switch(bps_code) {
		case 0: bps = si ? si->bits_per_sample : 0; break;
		case 1: bps = 8; break; case 2: bps = 12; break; case 4: bps = 16; break;
		case 5: bps = 20; break; case 6: bps = 24; break; case 7: bps = 32; break;
		default: return 0;
	}
	/* 25- to 32-bit samples are outside this restatement's scope, as they are the engine's (DEC_UNSUPPORTED) */
	if(bps == 0 || bps > 24 || blocksize > out_cap) return 0;

	residual = (int32_t *)malloc(sizeof(int32_t) * (blocksize + 1));
	for(c = 0; c < channels; c++) chan[c] = (int64_t *)malloc(sizeof(int64_t) * (blocksize + 1));
	for(c = 0; c < channels; c++) {
		uint32_t sub_bps = bps;
		if((ca_code == 8 && c == 1) || (ca_code == 9 && c == 0) || (ca_code == 10 && c == 1)) sub_bps++;
		if(!read_subframe(&br, blocksize, sub_bps, chan[c], residual)) goto done;
	}
	/* the padding to the byte boundary must be zero bits (stream_decoder.c:3359-3373 read_zero_padding_) */
	if(br.pos & 7) {
		if(br_read(&br, 8 - (uint32_t)(br.pos & 7)) != 0) goto done;
	}
	{
		const size_t n = (size_t)(br.pos >> 3);
		const uint16_t crc = (uint16_t)br_read(&br, 16);
		if(br.err || fo_crc16(data, n) != crc) goto done;
		consumed = n + 2;
	}
	for(i = 0; i < blocksize; i++) {
		int64_t l, r;
		switch(ca_code) {
			case 8: l = chan[0][i]; r = l - chan[1][i]; break;
			case 9: r = chan[1][i]; l = chan[0][i] + r; break;
			case 10: {
				int64_t mid = chan[0][i], side = chan[1][i];
				mid = (int64_t)((uint64_t)mid << 1) | (side & 1);
				l = (mid + side) >> 1; r = (mid - side) >> 1;
				break;
			}
			default: l = r = 0; break;
		}
		/* every decoded sample must fit the stream's sample width (stream_decoder.c:2458-2472) */
		for(c = 0; c < channels; c++) {
			const int64_t v = ca_code >= 8 ? (c ? r : l) : chan[c][i];
			if(v < -((int64_t)1 << (bps - 1)) || v >= ((int64_t)1 << (bps - 1))) { consumed = 0; goto done; }
		}
		if(ca_code >= 8) {
			out_interleaved[(size_t)i * 2] = (int32_t)l;
			out_interleaved[(size_t)i * 2 + 1] = (int32_t)r;
		}
		else
			for(c = 0; c < channels; c++)
				out_interleaved[(size_t)i * channels + c] = (int32_t)chan[c][i];
	}
	if(blocksize_out) *blocksize_out = blocksize;
	if(channels_out) *channels_out = channels;
	if(bps_out) *bps_out = bps;
	if(number_out) *number_out = number;
done:
	free(residual);
	for(c = 0; c < channels; c++) free(chan[c]);
	return consumed;
}
