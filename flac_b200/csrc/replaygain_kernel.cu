// replaygain_kernel.cu -- ReplayGain 1.0 analysis (flac --replay-gain): k_replaygain runs every channel of every file through
// the equal-loudness filters and sums the squared output over 50 ms windows; the host turns the windows into gains as
// replaygain_analysis.c does (analyzeResult) and fb200_replaygain_device / fb200_debug_replaygain_windows expose it on
// device PCM. The filter is one strictly sequential recurrence per channel, so a lane runs one channel's whole chain.
#include <math.h>
#include <string.h>

#include <map>

#include "fb200_internal.h"

namespace fb200 {

// The ReplayGain 1.0 equal-loudness filter design (David Robinson, replaygain.org; the coefficients every ReplayGain analyser
// shares, as replaygain_analysis.c lists them): per filter rate, the Yule-Walker numerator and denominator (10th order), then the
// Butterworth high-pass numerator and denominator (2nd order). The analysis filters in float with coefficients initialised from
// these decimals, so they are kept as doubles and rounded to float on the device (decimal -> double -> float, as a C
// initialiser of a float array from double literals rounds).
struct RgFilter { double by[11], ay[11], bb[3], ab[3]; };
constexpr int kRgFilters = 13;
static const uint32_t kRgRates[kRgFilters] = {48000, 44100, 37800, 36000, 32000, 28000, 24000, 22050, 18900, 16000, 12000, 11025, 8000};
__constant__ RgFilter c_rg_filters[kRgFilters] = {  // in kRgRates' order
	{{0.03857599435200, -0.02160367184185, -0.00123395316851, -0.00009291677959, -0.01655260341619, 0.02161526843274, -0.02074045215285, 0.00594298065125, 0.00306428023191, 0.00012025322027, 0.00288463683916},  // 48000
	 {1.00000000000000, -3.84664617118067, 7.81501653005538, -11.34170355132042, 13.05504219327545, -12.28759895145294, 9.48293806319790, -5.87257861775999, 2.75465861874613, -0.86984376593551, 0.13919314567432},
	 {0.98621192462708, -1.97242384925416, 0.98621192462708},
	 {1.00000000000000, -1.97223372919527, 0.97261396931306}},
	{{0.05418656406430, -0.02911007808948, -0.00848709379851, -0.00851165645469, -0.00834990904936, 0.02245293253339, -0.02596338512915, 0.01624864962975, -0.00240879051584, 0.00674613682247, -0.00187763777362},  // 44100
	 {1.00000000000000, -3.47845948550071, 6.36317777566148, -8.54751527471874, 9.47693607801280, -8.81498681370155, 6.85401540936998, -4.39470996079559, 2.19611684890774, -0.75104302451432, 0.13149317958808},
	 {0.98500175787242, -1.97000351574484, 0.98500175787242},
	 {1.00000000000000, -1.96977855582618, 0.97022847566350}},
	{{0.10296717174470, -0.04877975583256, -0.02878009075237, -0.03519509188311, 0.02888717172493, -0.00609872684844, 0.00209851217112, 0.00911704668543, 0.01154404718589, -0.00630293688700, 0.00107527155228},  // 37800
	 {1.00000000000000, -2.64848054923531, 3.58406058405771, -3.83794914179161, 3.90142345804575, -3.50179818637243, 2.67085284083076, -1.82581142372418, 1.09530368139801, -0.47689017820395, 0.11171431535905},
	 {0.98252400815195, -1.96504801630391, 0.98252400815195},
	 {1.00000000000000, -1.96474258269041, 0.96535344991740}},
	{{0.11572297028613, -0.04120916051252, -0.04977731768022, -0.01047308680426, 0.00750863219157, 0.00055507694408, 0.00140344192886, 0.01286095246036, 0.00998223033885, -0.00725013810661, 0.00326503346879},  // 36000
	 {1.00000000000000, -2.43606802820871, 3.01907406973844, -2.90372016038192, 2.67947188094303, -2.17606479220391, 1.44912956803015, -0.87785765549050, 0.53592202672557, -0.26469344817509, 0.07495878059717},
	 {0.98165826840326, -1.96331653680652, 0.98165826840326},
	 {1.00000000000000, -1.96298008938934, 0.96365298422371}},
	{{0.15457299681924, -0.09331049056315, -0.06247880153653, 0.02163541888798, -0.05588393329856, 0.04781476674921, 0.00222312597743, 0.03174092540049, -0.01390589421898, 0.00651420667831, -0.00881362733839},  // 32000
	 {1.00000000000000, -2.37898834973084, 2.84868151156327, -2.64577170229825, 2.23697657451713, -1.67148153367602, 1.00595954808547, -0.45953458054983, 0.16378164858596, -0.05032077717131, 0.02347897407020},
	 {0.97938932735214, -1.95877865470428, 0.97938932735214},
	 {1.00000000000000, -1.95835380975398, 0.95920349965459}},
	{{0.23882392323383, -0.22007791534089, -0.06014581950332, 0.05004458058021, -0.03293111254977, 0.02348678189717, 0.04290549799671, -0.00938141862174, 0.00015095146303, -0.00712601540885, -0.00626520210162},  // 28000
	 {1.00000000000000, -2.06894080899139, 1.76944699577212, -0.81404732584187, 0.25418286850232, -0.30340791669762, 0.35616884070937, -0.14967310591258, -0.07024154183279, 0.11078404345174, -0.03551838002425},
	 {0.97647981663949, -1.95295963327897, 0.97647981663949},
	 {1.00000000000000, -1.95240635772520, 0.95351290883275}},
	{{0.30296907319327, -0.22613988682123, -0.08587323730772, 0.03282930172664, -0.00915702933434, -0.02364141202522, -0.00584456039913, 0.06276101321749, -0.00000828086748, 0.00205861885564, -0.02950134983287},  // 24000
	 {1.00000000000000, -1.61273165137247, 1.07977492259970, -0.25656257754070, -0.16276719120440, -0.22638893773906, 0.39120800788284, -0.22138138954925, 0.04500235387352, 0.02005851806501, 0.00302439095741},
	 {0.97531843204928, -1.95063686409857, 0.97531843204928},
	 {1.00000000000000, -1.95002759149878, 0.95124613669835}},
	{{0.33642304856132, -0.25572241425570, -0.11828570177555, 0.11921148675203, -0.07834489609479, -0.00469977914380, -0.00589500224440, 0.05724228140351, 0.00832043980773, -0.01635381384540, -0.01760176568150},  // 22050
	 {1.00000000000000, -1.49858979367799, 0.87350271418188, 0.12205022308084, -0.80774944671438, 0.47854794562326, -0.12453458140019, -0.04067510197014, 0.08333755284107, -0.04237348025746, 0.02977207319925},
	 {0.97316523498161, -1.94633046996323, 0.97316523498161},
	 {1.00000000000000, -1.94561023566527, 0.94705070426118}},
	{{0.38412657295385, -0.44533729608120, 0.20426638066221, -0.28031676047946, 0.31484202614802, -0.26078311203207, 0.12925201224848, -0.01141164696062, 0.03036522115769, -0.03776339305406, 0.00692036603586},  // 18900
	 {1.00000000000000, -1.74403915585708, 1.96686095832499, -2.10081452941881, 1.90753918182846, -1.83814263754422, 1.36971352214969, -0.77883609116398, 0.39266422457649, -0.12529383592986, 0.05424760697665},
	 {0.96535326815829, -1.93070653631658, 0.96535326815829},
	 {1.00000000000000, -1.92950577983524, 0.93190729279793}},
	{{0.44915256608450, -0.14351757464547, -0.22784394429749, -0.01419140100551, 0.04078262797139, -0.12398163381748, 0.04097565135648, 0.10478503600251, -0.01863887810927, -0.03193428438915, 0.00541907748707},  // 16000
	 {1.00000000000000, -0.62820619233671, 0.29661783706366, -0.37256372942400, 0.00213767857124, -0.42029820170918, 0.22199650564824, 0.00613424350682, 0.06747620744683, 0.05784820375801, 0.03222754072173},
	 {0.96454515552826, -1.92909031105652, 0.96454515552826},
	 {1.00000000000000, -1.92783286977036, 0.93034775234268}},
	{{0.56619470757641, -0.75464456939302, 0.16242137742230, 0.16744243493672, -0.18901604199609, 0.30931782841830, -0.27562961986224, 0.00647310677246, 0.08647503780351, -0.03788984554840, -0.00588215443421},  // 12000
	 {1.00000000000000, -1.04800335126349, 0.29156311971249, -0.26806001042947, 0.00819999645858, 0.45054734505008, -0.33032403314006, 0.06739368333110, -0.04784254229033, 0.01639907836189, 0.01807364323573},
	 {0.96009142950541, -1.92018285901082, 0.96009142950541},
	 {1.00000000000000, -1.91858953033784, 0.92177618768381}},
	{{0.58100494960553, -0.53174909058578, -0.14289799034253, 0.17520704835522, 0.02377945217615, 0.15558449135573, -0.25344790059353, 0.01628462406333, 0.06920467763959, -0.03721611395801, -0.00749618797172},  // 11025
	 {1.00000000000000, -0.51035327095184, -0.31863563325245, -0.20256413484477, 0.14728154134330, 0.38952639978999, -0.23313271880868, -0.05246019024463, -0.02505961724053, 0.02442357316099, 0.01818801111503},
	 {0.95856916599601, -1.91713833199203, 0.95856916599601},
	 {1.00000000000000, -1.91542108074780, 0.91885558323625}},
	{{0.53648789255105, -0.42163034350696, -0.00275953611929, 0.04267842219415, -0.10214864179676, 0.14590772289388, -0.02459864859345, -0.11202315195388, -0.04060034127000, 0.04788665548180, -0.02217936801134},  // 8000
	 {1.00000000000000, -0.25049871956020, -0.43193942311114, -0.03424681017675, -0.04678328784242, 0.26408300200955, 0.15113130533216, -0.17556493366449, -0.18823009262115, 0.05477720428674, 0.04704409688120},
	 {0.94597685600279, -1.89195371200558, 0.94597685600279},
	 {1.00000000000000, -1.88903307939452, 0.89487434461664}},
};

constexpr int kRgBatch = 16;  // decimated samples loaded one batch ahead of the filter chain

// One filter rate's coefficients in float, as the analysis holds them.
struct RgCoefs { float by[11], ay[11], bb[3], ab[3]; };

__device__ __forceinline__ void rg_coefs(uint32_t filt, RgCoefs &K)
{
	const RgFilter &R = c_rg_filters[filt];
#pragma unroll
	for(int k = 0; k < 11; k++) { K.by[k] = __double2float_rn(R.by[k]); K.ay[k] = __double2float_rn(R.ay[k]); }
#pragma unroll
	for(int k = 0; k < 3; k++) { K.bb[k] = __double2float_rn(R.bb[k]); K.ab[k] = __double2float_rn(R.ab[k]); }
}

// One channel's filter state: input and Yule-Walker output histories, Butterworth input and output histories ([0] = the latest),
// the window's sum of squares, its sample count and the next window's index.
struct RgChain {
	float xh[10], yh[10], sh[2], oh[2];
	double sum;
	uint32_t cnt;
	unsigned long long w;
};

__device__ __forceinline__ void rg_chain_init(RgChain &C, unsigned long long win)
{
#pragma unroll
	for(int k = 0; k < 10; k++) C.xh[k] = C.yh[k] = 0.f;
	C.sh[0] = C.sh[1] = C.oh[0] = C.oh[1] = 0.f;
	C.sum = 0.0;
	C.cnt = 0;
	C.w = win;
}

// One sample through the chain, as filter() in replaygain_analysis.c: each term x * b[k] - y * a[k] in float (two products, one
// difference), added in k order to a double, the sum rounded to float; the Yule-Walker output feeds the Butterworth filter, whose
// squared output (a float product) is added to the channel's double sum. At a window's end (W samples) the pair's sums meet
// with one shuffle (`pair`: the two lanes of the file) and lane c == 0 writes v[w] (kCapped: only when w < w_end).
template <bool kCapped>
__device__ __forceinline__ void rg_step(RgChain &C, const RgCoefs &K, float x, uint32_t W, unsigned pair, int c, double *__restrict__ v,
                                        unsigned long long w_end)
{
	double y = (double)__fmul_rn(x, K.by[0]);
#pragma unroll
	for(int k = 1; k <= 10; k++) y = __dadd_rn(y, (double)__fsub_rn(__fmul_rn(C.xh[k - 1], K.by[k]), __fmul_rn(C.yh[k - 1], K.ay[k])));
	const float st = __double2float_rn(y);
#pragma unroll
	for(int k = 9; k > 0; k--) { C.xh[k] = C.xh[k - 1]; C.yh[k] = C.yh[k - 1]; }
	C.xh[0] = x;
	C.yh[0] = st;
	double z = (double)__fmul_rn(st, K.bb[0]);
	z = __dadd_rn(z, (double)__fsub_rn(__fmul_rn(C.sh[0], K.bb[1]), __fmul_rn(C.oh[0], K.ab[1])));
	z = __dadd_rn(z, (double)__fsub_rn(__fmul_rn(C.sh[1], K.bb[2]), __fmul_rn(C.oh[1], K.ab[2])));
	const float o = __double2float_rn(z);
	C.sh[1] = C.sh[0]; C.sh[0] = st;
	C.oh[1] = C.oh[0]; C.oh[0] = o;
	C.sum = __dadd_rn(C.sum, (double)__fmul_rn(o, o));
	if(++C.cnt == W) {
		const double other = __shfl_xor_sync(pair, C.sum, 1);
		if(c == 0 && (!kCapped || C.w < w_end)) v[C.w] = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(C.sum, other), (double)W), 0.5), 1e-37);
		C.w++;
		C.cnt = 0;
		C.sum = 0.0;
	}
}

// One lane per (file, channel): lanes 2f and 2f + 1 are file f's left and right channel (a mono file runs its one channel on
// both, which makes the pair's sum left + left as the analysis has it). The decimated samples go through rg_step; histories
// start at zero for every file.
__global__ void __launch_bounds__(32) k_replaygain(const int32_t *__restrict__ pcm, const RgFileDev *__restrict__ files, int nfiles,
                                                  double *__restrict__ v, uint32_t *__restrict__ peak)
{
	const int lane = blockIdx.x * 32 + threadIdx.x;
	const int f = lane >> 1, c = lane & 1;
	if(f >= nfiles) return;
	const unsigned pair = 3u << (threadIdx.x & 30);
	const RgFileDev F = files[f];
	RgCoefs K;
	rg_coefs(F.filt, K);
	// the tool's input conversion, (float)(2^(16 - bps) * s): exact here, since |s| < 2^23
	const float scale = ldexpf(1.0f, 16 - (int)F.bps);
	const unsigned ch = F.channels, cc = ch == 2 ? (unsigned)c : 0u;
	const int32_t *pa = pcm + F.a + cc, *pb = pcm + F.b + cc;
	const unsigned long long na = F.na, n = F.n, ds = F.ds, nd = n / ds;
	auto at = [&](unsigned long long i) -> int32_t { return __ldg(i < na ? pa + i * ch : pb + (i - na) * ch); };

	RgChain C;
	rg_chain_init(C, F.win);
	uint32_t pk = 0;
	int32_t cur[kRgBatch];
#pragma unroll
	for(int j = 0; j < kRgBatch; j++) cur[j] = (unsigned long long)j < nd ? at(j * ds) : 0;
	for(unsigned long long base = 0; base < nd; base += kRgBatch) {
		int32_t nxt[kRgBatch];
#pragma unroll
		for(int j = 0; j < kRgBatch; j++) nxt[j] = base + kRgBatch + j < nd ? at((base + kRgBatch + j) * ds) : 0;
#pragma unroll
		for(int j = 0; j < kRgBatch; j++) {
			if(base + j >= nd) break;
			const int32_t s = cur[j];
			pk = max(pk, (uint32_t)abs(s));
			rg_step<false>(C, K, __fmul_rn(__int2float_rn(s), scale), F.W, pair, c, v, 0);
		}
#pragma unroll
		for(int j = 0; j < kRgBatch; j++) cur[j] = nxt[j];
	}
	// the peak is over every sample: with decimation, the ones the filters skipped (and the last n % ds) too
	for(unsigned long long i = ds == 1 ? n : 0; i < n; i++) pk = max(pk, (uint32_t)abs(at(i)));
	pk = max(pk, __shfl_xor_sync(pair, pk, 1));
	if(c == 0) peak[f] = pk;
}

constexpr uint32_t kRgCall = 2048;  // samples per AnalyzeSamples call at most (grabbag__replaygain_analyze's buffer)

// metaflac's feed (grabbag__replaygain_analyze from the decoder's write callback): lanes as k_replaygain, each walking its file's
// accepted frames (candidates with place n > 0) in order. Each frame is split into calls of at most kRgCall samples; a call of
// len samples runs m = len / ds decimated samples from its own start (the remainder is dropped), and after a call with
// 0 < m < 10 the input history is the old one shifted by m followed by the call's first m undecimated samples (AnalyzeSamples'
// memcpy into linprebuf; the Yule-Walker and Butterworth histories run on). The peak is over every sample of every frame. The
// lane also checks what makes a file analysable: no decode error in its state, every accepted frame whole (n = blocksize x
// channels) at STREAMINFO's rate, and the frames tiling [audio, end).
__global__ void __launch_bounds__(32) k_replaygain_frames(const int32_t *__restrict__ pcm, const RgFramesFileDev *__restrict__ files, int nfiles,
                                                         const FilePlace *__restrict__ place, const unsigned long long *__restrict__ begins,
                                                         const uint32_t *__restrict__ bytes, const FileDecCand *__restrict__ cands,
                                                         const FileDecState *__restrict__ states, double *__restrict__ v, RgFramesOut *__restrict__ out)
{
	const int lane = blockIdx.x * 32 + threadIdx.x;
	const int f = lane >> 1, c = lane & 1;
	if(f >= nfiles) return;
	const unsigned pair = 3u << (threadIdx.x & 30);
	const RgFramesFileDev F = files[f];
	RgCoefs K;
	rg_coefs(F.filt, K);
	const float scale = ldexpf(1.0f, 16 - (int)F.bps);
	const unsigned ch = F.channels, cc = ch == 2 ? (unsigned)c : 0u;
	const uint32_t ds = F.ds;
	const unsigned long long w_end = F.win + F.nwin_cap;
	RgChain C;
	rg_chain_init(C, F.win);
	uint32_t pk = 0;
	bool ok = states[F.state].errors == 0;
	unsigned long long next = F.audio;  // where the next accepted frame must begin
	unsigned long long next_sample = ~0ull;  // where the next frame's samples must begin (none before the first frame)
	for(unsigned long long i = F.cand0; ok && i < F.cand0 + F.ncand; i++) {
		const FilePlace p = place[i];
		if(p.n == 0) continue;
		const FileDecCand cd = cands[i];
		const uint32_t bs = cd.blocksize;
		// a gap in the sample numbers is a missing frame: libFLAC reports MISSING_FRAME (stream_decoder.c:2487-2494) and
		// metaflac fails the file, even when the frames around it tile the bytes
		if(begins[i] != next || cd.rate_differs || p.n != bs * ch || (next_sample != ~0ull && cd.first_sample > next_sample)) { ok = false; break; }
		next = begins[i] + bytes[i];
		next_sample = cd.first_sample + bs;
		const int32_t *fr = pcm + p.dst + cc;
		for(uint32_t s0 = 0; s0 < bs; s0 += kRgCall) {
			const uint32_t len = min(kRgCall, bs - s0), m = len / ds;
			const int32_t *q = fr + (size_t)s0 * ch;
			if(ds > 1)
				for(uint32_t t = 0; t < len; t++) pk = max(pk, (uint32_t)abs(__ldg(q + (size_t)t * ch)));
			for(uint32_t b = 0; b < m; b += kRgBatch) {
				int32_t cur[kRgBatch];
#pragma unroll
				for(int j = 0; j < kRgBatch; j++) cur[j] = b + j < m ? __ldg(q + (size_t)(b + j) * ds * ch) : 0;
#pragma unroll
				for(int j = 0; j < kRgBatch; j++) {
					if(b + j >= m) break;
					if(ds == 1) pk = max(pk, (uint32_t)abs(cur[j]));
					rg_step<true>(C, K, __fmul_rn(__int2float_rn(cur[j]), scale), F.W, pair, c, v, w_end);
				}
			}
			if(ds > 1 && m > 0 && m < 10) {
#pragma unroll
				for(int k = 0; k < 9; k++)
					if((uint32_t)k < m) C.xh[k] = __fmul_rn(__int2float_rn(__ldg(q + (size_t)(m - 1 - k) * ch)), scale);
			}
		}
	}
	ok = ok && next == F.end;
	pk = max(pk, __shfl_xor_sync(pair, pk, 1));
	if(c == 0) out[f] = RgFramesOut{C.w - F.win, pk, ok ? 1u : 0u};
}

void launch_replaygain(const int32_t *pcm, const RgFileDev *files, int nfiles, double *v, uint32_t *peak, cudaStream_t st)
{
	if(nfiles) k_replaygain<<<(unsigned)((2 * (long long)nfiles + 31) / 32), 32, 0, st>>>(pcm, files, nfiles, v, peak);
}

void launch_replaygain_frames(const int32_t *pcm, const RgFramesFileDev *files, int nfiles, const FilePlace *place, const unsigned long long *begins,
                              const uint32_t *bytes, const FileDecCand *cands, const FileDecState *states, double *v, RgFramesOut *out, cudaStream_t st)
{
	if(nfiles)
		k_replaygain_frames<<<(unsigned)((2 * (long long)nfiles + 31) / 32), 32, 0, st>>>(pcm, files, nfiles, place, begins, bytes, cands, states, v, out);
}

// ---- host

// CreateGainFilter (replaygain_analysis.c): a filter rate itself, or halved (integer division) until it is at most 48000, which
// must then be a filter rate
bool replaygain_rate(uint32_t sample_rate, uint32_t *ds, uint32_t *W, uint32_t *filt)
{
	uint32_t d = 1, r = sample_rate;
	while(r > kRgRates[0]) { r /= 2; d *= 2; }
	for(int i = 0; i < kRgFilters; i++)
		if(kRgRates[i] == r) {
			*ds = d;
			*W = (r * 50 + 999) / 1000;  // RMS_WINDOW_TIME
			*filt = (uint32_t)i;
			return true;
		}
	return false;
}

namespace {

constexpr int kRgSteps = 120 * 100;  // histogram entries: 0.01 dB steps up to 120 dB

// analyzeResult: the 95th percentile of the windows' loudness, in float as the analysis returns it
float rg_gain(const std::vector<uint32_t> &h)
{
	uint32_t elems = 0;
	for(uint32_t x : h) elems += x;
	if(elems == 0) return -24601.f;  // GAIN_NOT_ENOUGH_SAMPLES
	int32_t upper = (int32_t)(elems / 20 + (elems % 20 ? 1 : 0));
	size_t i = h.size();
	while(i-- > 0)
		if((upper -= (int32_t)h[i]) <= 0) break;
	return (float)((float)64.82 - (float)i / (float)100.);
}

}  // namespace

void replaygain_results(const std::vector<RgFileDev> &files, const uint32_t *album, const double *v, const uint32_t *peak, fb200_replaygain_info *info,
                        const uint64_t *nwin_of)
{
	struct Album { std::vector<uint32_t> h; double peak = 0.0; };
	std::map<uint32_t, Album> albums;
	std::vector<uint32_t> h(kRgSteps);
	for(size_t f = 0; f < files.size(); f++) {
		const RgFileDev &F = files[f];
		const uint64_t nwin = nwin_of ? nwin_of[f] : F.n / F.ds / F.W;
		std::fill(h.begin(), h.end(), 0u);
		for(uint64_t j = 0; j < nwin; j++) {
			// the loudness step, with the process's own log10 (the function the tool calls)
			int ival = (int)(1000. * log10(v[F.win + j]));
			if(ival < 0) ival = 0;
			if(ival >= kRgSteps) ival = kRgSteps - 1;
			h[ival]++;
		}
		const double pk = (double)peak[f] / (double)(1u << (F.bps - 1));
		Album &A = albums[album[f]];
		if(A.h.empty()) A.h.assign(kRgSteps, 0u);
		for(int i = 0; i < kRgSteps; i++) A.h[i] += h[i];
		if(pk > A.peak) A.peak = pk;
		info[f].track_gain = rg_gain(h);
		info[f].track_peak = (float)pk;
		info[f].windows = nwin;
	}
	for(size_t f = 0; f < files.size(); f++) {
		const Album &A = albums[album[f]];
		info[f].album_gain = rg_gain(A.h);
		info[f].album_peak = (float)A.peak;
	}
}

namespace {

// the checks and launch plan of fb200_replaygain_device / fb200_debug_replaygain_windows
int rg_plan(const int32_t *d_pcm, uint64_t pcm_values, const fb200_replaygain_file *files, uint32_t nfiles, std::vector<RgFileDev> *dev,
            std::vector<uint32_t> *album, uint64_t *nwin)
{
	if(!d_pcm || !files) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	if(nfiles >= (1u << 30)) { set_error("too many files in one call"); return FB200_ERR_INVALID; }
	std::map<uint32_t, uint32_t> album_rate;
	uint64_t win = 0;
	for(uint32_t f = 0; f < nfiles; f++) {
		const fb200_replaygain_file &I = files[f];
		RgFileDev D{};
		if(I.channels < 1 || I.channels > 2) { set_error("file %u: %u channels (ReplayGain takes 1 or 2)", f, I.channels); return FB200_ERR_INVALID; }
		if(I.bits_per_sample < 4 || I.bits_per_sample > 24) { set_error("file %u: %u bits per sample (4-24)", f, I.bits_per_sample); return FB200_ERR_INVALID; }
		if(!replaygain_rate(I.sample_rate, &D.ds, &D.W, &D.filt)) { set_error("file %u: invalid sample rate %u for ReplayGain", f, I.sample_rate); return FB200_ERR_INVALID; }
		auto it = album_rate.emplace(I.album, I.sample_rate).first;
		if(it->second != I.sample_rate) {
			set_error("file %u: %u Hz in album %u, whose files are %u Hz", f, I.sample_rate, I.album, it->second);
			return FB200_ERR_INVALID;
		}
		if(I.first_value > pcm_values || I.samples > (pcm_values - I.first_value) / I.channels) {
			set_error("file %u runs past the %llu values of d_pcm", f, (unsigned long long)pcm_values);
			return FB200_ERR_INVALID;
		}
		D.a = I.first_value;
		D.na = D.n = I.samples;
		D.b = I.first_value;
		D.win = win;
		D.channels = I.channels;
		D.bps = I.bits_per_sample;
		win += D.n / D.ds / D.W;
		dev->push_back(D);
		album->push_back(I.album);
	}
	*nwin = win;
	return FB200_OK;
}

// one launch over the planned files; v[nwin] and peak[nfiles] back on the host
int rg_run(int device, const int32_t *d_pcm, const std::vector<RgFileDev> &dev, uint64_t nwin, std::vector<double> *v, std::vector<uint32_t> *peak,
           void *cuda_stream)
{
	const size_t nf = dev.size();
	v->resize(nwin);
	peak->resize(nf);
	if(nf == 0) return FB200_OK;
	FB_CUDA(cudaSetDevice(device));
	cudaStream_t st = static_cast<cudaStream_t>(cuda_stream);
	const size_t o_peak = (nf * sizeof(RgFileDev) + 15) & ~(size_t)15, o_v = (o_peak + nf * sizeof(uint32_t) + 15) & ~(size_t)15;
	uint8_t *d = nullptr;
	FB_CUDA(cudaMalloc(&d, o_v + nwin * sizeof(double) + 8));
	struct Free { uint8_t *p; ~Free() { cudaFree(p); } } hold{d};
	FB_CUDA(cudaMemcpyAsync(d, dev.data(), nf * sizeof(RgFileDev), cudaMemcpyHostToDevice, st));
	launch_replaygain(d_pcm, reinterpret_cast<const RgFileDev *>(d), (int)nf, reinterpret_cast<double *>(d + o_v), reinterpret_cast<uint32_t *>(d + o_peak), st);
	FB_CUDA(cudaGetLastError());
	FB_CUDA(cudaMemcpyAsync(peak->data(), d + o_peak, nf * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
	if(nwin) FB_CUDA(cudaMemcpyAsync(v->data(), d + o_v, nwin * sizeof(double), cudaMemcpyDeviceToHost, st));
	FB_CUDA(cudaStreamSynchronize(st));
	return FB200_OK;
}

}  // namespace

}  // namespace fb200

using namespace fb200;

int fb200_replaygain_device(int device, const int32_t *d_pcm, uint64_t pcm_values, const fb200_replaygain_file *files, uint32_t nfiles,
                            fb200_replaygain_info *info, void *cuda_stream)
{
	if(!info) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	std::vector<RgFileDev> dev;
	std::vector<uint32_t> album, peak;
	std::vector<double> v;
	uint64_t nwin = 0;
	int rc = rg_plan(d_pcm, pcm_values, files, nfiles, &dev, &album, &nwin);
	if(rc == FB200_OK) rc = rg_run(device, d_pcm, dev, nwin, &v, &peak, cuda_stream);
	if(rc != FB200_OK) return rc;
	replaygain_results(dev, album.data(), v.data(), peak.data(), info);
	return FB200_OK;
}

int fb200_debug_replaygain_windows(int device, const int32_t *d_pcm, uint64_t pcm_values, const fb200_replaygain_file *files, uint32_t nfiles,
                                   double *windows, uint64_t capacity, uint64_t *nwindows, void *cuda_stream)
{
	if(!nwindows || (!windows && capacity)) { set_error("a required pointer is NULL"); return FB200_ERR_INVALID; }
	std::vector<RgFileDev> dev;
	std::vector<uint32_t> album, peak;
	std::vector<double> v;
	uint64_t nwin = 0;
	int rc = rg_plan(d_pcm, pcm_values, files, nfiles, &dev, &album, &nwin);
	if(rc != FB200_OK) return rc;
	*nwindows = nwin;
	if(nwin > capacity) { set_error("%llu windows, room for %llu", (unsigned long long)nwin, (unsigned long long)capacity); return FB200_ERR_OUTPUT_TOO_SMALL; }
	if((rc = rg_run(device, d_pcm, dev, nwin, &v, &peak, cuda_stream)) != FB200_OK) return rc;
	if(nwin) memcpy(windows, v.data(), nwin * sizeof(double));
	return FB200_OK;
}
