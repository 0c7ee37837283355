/* hacktv_b200 - host-side table generation.
 *
 * Everything the device needs that the reference derives once in vid_init()
 * (ref video.c:3812-4704) is computed here, on the host, with the same libm
 * double formulas, so the integer tables are bit-identical to the reference's:
 * levels, sync pulse shapes, burst window, Gaussian / Kaiser FIR taps, colour
 * subcarrier LUT, NICAM pulse + carrier, SECAM bell / FM tables. What is NOT
 * taken over is the reference's recurrence NCOs: for each FM LUT entry we store
 * its exact effective angle (atan2 of the rounded Q31 phasor) as a 64-bit
 * fraction of a turn, so phase becomes an integer prefix sum (DESIGN.md §NCO).
 *
 * Pure C + libm, no CUDA: usable (and tested) without a GPU.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include "htv_internal.h"
#include "htv_fm_taps.h"

#define IRT1090 2.0738786  /* 10-90% -> 0-100% for integrated raised-cosine edges (ref common.h:29) */

/* ---- small maths ------------------------------------------------------- */

static int64_t gcd64(int64_t a, int64_t b)
{
	while(b) { int64_t c = a % b; a = b; b = c; }
	return(a < 0 ? -a : a);
}

/* Integrated raised-cosine window, 1 inside [left, left + width] (ref common.c:231-257) */
static double edge_window(double t, double left, double width, double rise)
{
	double d = fabs(t - (left + width / 2)) - (width - rise) / 2;
	if(d <= 0) return(1.0);
	if(d >= rise) return(0.0);
	d = 1.0 - d / rise * 2;
	return(0.5 * (1.0 + d + sin(M_PI * d) / M_PI));
}

/* Root raised cosine (ref common.c:259-283) */
static double root_rc(double x, double b, double t)
{
	if(x == 0) return((1.0 / t) * (1.0 + b * (4.0 / M_PI - 1)));
	if(fabs(x) == t / (4.0 * b))
	{
		return(b / (t * sqrt(2.0)) * ((1.0 + 2.0 / M_PI) * sin(M_PI / (4.0 * b)) + (1.0 - 2.0 / M_PI) * cos(M_PI / (4.0 * b))));
	}
	{
		double t1 = (4.0 * b * (x / t));
		double t2 = (sin(M_PI * (x / t) * (1.0 - b)) + 4.0 * b * (x / t) * cos(M_PI * (x / t) * (1.0 + b)));
		double t3 = (M_PI * (x / t) * (1.0 - t1 * t1));
		return((1.0 / t) * (t2 / t3));
	}
}

/* Modified Bessel I0 by series, Kaiser window beta = 7 (ref fir.c:31-69) */
static double bessel_i0(double x)
{
	double sum = 1, u = 1, halfx = x / 2.0;
	int n = 1;
	do
	{
		double temp = halfx / (double) n;
		n += 1;
		temp *= temp;
		u *= temp;
		sum += u;
	}
	while(u >= 1e-21 * sum);
	return(sum);
}

static void kaiser7(double *w, int n)
{
	double ib = 1.0 / bessel_i0(7.0), inm1 = 1.0 / ((double) (n - 1));
	int i;
	w[0] = ib;
	for(i = 1; i < n - 1; i++)
	{
		double temp = 2 * i * inm1 - 1;
		w[i] = bessel_i0(7.0 * sqrt(1.0 - temp * temp)) * ib;
	}
	w[n - 1] = ib;
}

/* Windowed-sinc low-pass, unity DC gain (ref fir.c:89-137), n odd */
static void lowpass(double *taps, int n, double rate, double cutoff, double gain)
{
	int k, M = (n - 1) / 2;
	double fmax, w0 = 2.0 * M_PI * cutoff / rate;
	kaiser7(taps, n);
	for(k = -M; k <= M; k++)
	{
		if(k == 0) taps[k + M] *= w0 / M_PI;
		else taps[k + M] *= sin(k * w0) / (k * M_PI);
	}
	fmax = taps[M];
	for(k = 1; k <= M; k++) fmax += 2 * taps[k + M];
	gain /= fmax;
	for(k = 0; k < n; k++) taps[k] *= gain;
}

/* Band-reject (ref fir.c:179-228), n odd */
static void bandreject(double *taps, int n, double rate, double lo, double hi, double gain)
{
	int k, M = (n - 1) / 2;
	double fmax, w0 = 2.0 * M_PI * lo / rate, w1 = 2.0 * M_PI * hi / rate;
	kaiser7(taps, n);
	for(k = -M; k <= M; k++)
	{
		if(k == 0) taps[k + M] *= 1.0 + (w0 - w1) / M_PI;
		else taps[k + M] *= (sin(k * w0) - sin(k * w1)) / (k * M_PI);
	}
	fmax = taps[M];
	for(k = 1; k <= M; k++) fmax += 2 * taps[k + M];
	gain /= fmax;
	for(k = 0; k < n; k++) taps[k] *= gain;
}

/* Gaussian low-pass for chroma (ref fir.c:139-177) */
static void gaussian(double *taps, int n, double rate, double cutoff, double gain)
{
	double f = 13.5e6 / rate, s = 354372.0 / cutoff, sum = 0;
	int x, h = n / 2;
	for(x = 0; x <= h; x++)
	{
		double t = (double) x / 5 * f;
		double r = 1.0 / s * pow(2.0 * M_PI, 0.5) * pow(M_E, -pow(t, 2.0) / (2.0 * pow(s, 2)));
		sum += r * (x > 0 ? 2 : 1);
		taps[h + x] = taps[h - x] = r;
	}
	gain /= sum;
	for(x = 0; x < n; x++) taps[x] *= gain;
}

/* int16 quantisation in application order (ref fir.c:263-295 with interpolation 1) */
static void quantise(int32_t *out, const double *taps, int n, int stride)
{
	int i;
	for(i = 0; i < n; i++) out[i] = lround(taps[(n - 1 - i) * stride] * 32767.0);
}

/* ---- reference data tables (filter coefficients, ref video.c:2118-2155) - */

static const double audio_flat[HTV_AFIR_N] = {
	 0.000000,-0.000793, 0.000318,-0.001297, 0.000756,-0.002084, 0.001341,-0.003091, 0.001926,-0.004059, 0.002173,
	-0.004543, 0.001586,-0.003982,-0.000386,-0.001819,-0.004219, 0.002351,-0.010158, 0.008641,-0.018108, 0.016785,
	-0.027575, 0.026122,-0.037697, 0.035663,-0.047356, 0.044249,-0.055360, 0.050742,-0.060650, 0.054238, 0.937500,
	 0.054238,-0.060650, 0.050742,-0.055360, 0.044249,-0.047356, 0.035663,-0.037697, 0.026122,-0.027575, 0.016785,
	-0.018108, 0.008641,-0.010158, 0.002351,-0.004219,-0.001819,-0.000386,-0.003982, 0.001586,-0.004543, 0.002173,
	-0.004059, 0.001926,-0.003091, 0.001341,-0.002084, 0.000756,-0.001297, 0.000318,-0.000793,-0.000000
};
static const double audio_50us[HTV_AFIR_N] = {
	 0.001234,-0.002637, 0.002903,-0.004810, 0.005412,-0.008091, 0.008855,-0.012171, 0.012482,-0.015806, 0.014595,
	-0.016860, 0.012742,-0.012646, 0.004202,-0.000532,-0.013336, 0.021334,-0.041037, 0.053332,-0.078322, 0.093873,
	-0.122521, 0.139174,-0.168825, 0.183024,-0.210266, 0.214647,-0.236618, 0.196560,-0.226183,-0.606600, 2.497308,
	-0.606600,-0.226183, 0.196560,-0.236618, 0.214647,-0.210266, 0.183024,-0.168825, 0.139174,-0.122521, 0.093873,
	-0.078322, 0.053332,-0.041037, 0.021334,-0.013336,-0.000532, 0.004202,-0.012646, 0.012742,-0.016860, 0.014595,
	-0.015806, 0.012482,-0.012171, 0.008855,-0.008091, 0.005412,-0.004810, 0.002903,-0.002637, 0.001234
};
static const double audio_75us[HTV_AFIR_N] = {
	 0.001981,-0.003755, 0.004472,-0.006942, 0.008239,-0.011739, 0.013420,-0.017690, 0.018901,-0.022955, 0.022160,
	-0.024370, 0.019556,-0.017960, 0.007049, 0.000170,-0.018791, 0.032752,-0.059706, 0.080325,-0.114856, 0.140480,
	-0.180353, 0.207455,-0.249292, 0.271550,-0.312119, 0.315065,-0.356561, 0.275266,-0.363286,-0.992136, 3.546394,
	-0.992136,-0.363286, 0.275266,-0.356561, 0.315065,-0.312119, 0.271550,-0.249292, 0.207455,-0.180353, 0.140480,
	-0.114856, 0.080325,-0.059706, 0.032752,-0.018791, 0.000170, 0.007049,-0.017960, 0.019556,-0.024370, 0.022160,
	-0.022955, 0.018901,-0.017690, 0.013420,-0.011739, 0.008239,-0.006942, 0.004472,-0.003755, 0.001981
};
static const double audio_j17[HTV_AFIR_N] = {
	-0.000119,-0.000175,-0.000162,-0.000232,-0.000223,-0.000310,-0.000309,-0.000420,-0.000430,-0.000576,-0.000605,
	-0.000801,-0.000864,-0.001135,-0.001253,-0.001644,-0.001860,-0.002446,-0.002844,-0.003776,-0.004531,-0.006130,
	-0.007663,-0.010705,-0.014141,-0.020784,-0.029556,-0.046668,-0.072530,-0.124846,-0.211267,-0.400931, 2.279077,
	-0.400931,-0.211267,-0.124846,-0.072530,-0.046668,-0.029556,-0.020784,-0.014141,-0.010705,-0.007663,-0.006130,
	-0.004531,-0.003776,-0.002844,-0.002446,-0.001860,-0.001644,-0.001253,-0.001135,-0.000864,-0.000801,-0.000605,
	-0.000576,-0.000430,-0.000420,-0.000309,-0.000310,-0.000223,-0.000232,-0.000162,-0.000175,-0.000119
};

#define SECAM_FM_DEV  1000e3   /* ref video.c:45-48 */
#define SECAM_FM_FREQ 4328125
#define SECAM_CB_FREQ 4250000
#define SECAM_CR_FREQ 4406250

/* ---- line code table --------------------------------------------------- */

/* The reference's per-line sync / burst / content codes (ref video.c:2481-2540,
 * 2541-2598) as data: {first, last, sync mask, burst, left active, right active}.
 * sync mask bits: 0 hsync, 1 short vsync, 2 long vsync (line start); 3 short,
 * 4 long (mid-line). burst: 0 never, 1 always, 2 even frames only, 3 odd frames only. */
typedef struct { short first, last; unsigned char sync, burst, left, right; } code_run_t;

static const code_run_t codes_625[] = {
	{   1,   2, 0x14, 0, 0, 0 }, {   3,   3, 0x0C, 0, 0, 0 }, {   4,   5, 0x0A, 0, 0, 0 },
	{   6,   6, 0x01, 2, 0, 0 }, {   7,  22, 0x01, 1, 0, 0 }, {  23,  23, 0x01, 1, 0, 1 },
	{  24, 309, 0x01, 1, 1, 1 }, { 310, 310, 0x01, 2, 1, 1 }, { 311, 312, 0x0A, 0, 0, 0 },
	{ 313, 313, 0x12, 0, 0, 0 }, { 314, 315, 0x14, 0, 0, 0 }, { 316, 317, 0x0A, 0, 0, 0 },
	{ 318, 318, 0x02, 0, 0, 0 }, { 319, 319, 0x01, 3, 0, 0 }, { 320, 335, 0x01, 1, 0, 0 },
	{ 336, 621, 0x01, 1, 1, 1 }, { 622, 622, 0x01, 2, 1, 1 }, { 623, 623, 0x09, 0, 1, 0 },
	{ 624, 625, 0x0A, 0, 0, 0 }, { 0, 0, 0, 0, 0, 0 }
};

static const code_run_t codes_525[] = {
	{   1,   3, 0x0A, 0, 0, 0 }, {   4,   6, 0x14, 0, 0, 0 }, {   7,   9, 0x0A, 0, 0, 0 },
	{  10,  20, 0x01, 1, 0, 0 }, {  21, 262, 0x01, 1, 1, 1 }, { 263, 263, 0x09, 1, 1, 0 },
	{ 264, 265, 0x0A, 0, 0, 0 }, { 266, 266, 0x12, 0, 0, 0 }, { 267, 268, 0x14, 0, 0, 0 },
	{ 269, 269, 0x0C, 0, 0, 0 }, { 270, 271, 0x0A, 0, 0, 0 }, { 272, 272, 0x02, 0, 0, 0 },
	{ 273, 282, 0x01, 1, 0, 0 }, { 283, 283, 0x01, 1, 0, 1 }, { 284, 525, 0x01, 1, 1, 1 },
	{ 0, 0, 0, 0, 0, 0 }
};

static void build_codes(struct htv_tables_t *t)
{
	const code_run_t *r = t->conf.type == HTV_RASTER_625 ? codes_625 : codes_525;
	int l;
	t->ncodes = t->conf.lines + 1;
	t->codes = calloc(t->ncodes, sizeof(uint16_t));
	/* line 0 only exists as a pipeline-fill line: an active line with hsync + burst */
	t->codes[0] = 0x01 | (1 << HTV_LC_BURST_SHIFT) | HTV_LC_LEFT_ACTIVE | HTV_LC_RIGHT_ACTIVE;
	for(; r->first; r++)
	{
		for(l = r->first; l <= r->last && l < t->ncodes; l++)
		{
			t->codes[l] = r->sync | (r->burst << HTV_LC_BURST_SHIFT) |
				(r->left ? HTV_LC_LEFT_ACTIVE : 0) | (r->right ? HTV_LC_RIGHT_ACTIVE : 0);
		}
	}
}

/* ---- sync pulses (ref vbidata.c:36-81, video.c:3766-3810, 3883-3891) ---- */

static int build_pulse(int16_t *dst, int32_t *off, double offset, double width, double rise, int level)
{
	int x1 = floor(offset - rise / 2), x2 = ceil(offset + width + rise / 2), len = 0;
	*off = 0;
	for(; x1 <= x2; x1++)
	{
		int v = round(edge_window(x1, offset, width, rise) * level);
		if(v == 0) continue;           /* leading zeros skipped, interior gaps zero-filled, no trailing zeros */
		if(len == 0) *off = x1;
		while(len < x1 - *off) dst[len++] = 0;
		dst[len++] = v;
	}
	return(len);
}

/* ---- line templates (fused line kernel) ---------------------------------- *
 * Everything of a raster line that does not depend on the picture: the blanking level plus every
 * sync-pulse piece that lands on the line - its own pulses, the previous line's overrun and the next
 * line's leading edge (ref vbidata.c:186-239, video.c:2447-2810 + 2920-2960: the raster adds the pulses
 * of line n into line n's buffer and, where they run past either end, into the neighbours').
 *   tmpl_out[row][x]   what the line holds where no picture is drawn
 *   tmpl_keep[row][x]  the part that is also added INSIDE the picture (the picture overwrites the line's
 *                      own and the previous line's pieces; only the next line's edge comes later)
 * row = line - 1 for lines 1 .. lines; row `lines` = line 1 of the very first frame (nothing before it);
 * row lines + 1 = before the stream (zeros). int16 wrap-around sums, as the reference's line buffer.
 * Every raster kernel takes its blanking and sync from here. -1: out of memory. */
static int build_templates(struct htv_tables_t *t)
{
	const htv_dparams_t *dp = &t->dp;
	const int W = dp->W, nl = dp->lines, rows = nl + 2;
	int r, s, b, d;
	t->tmpl_rows = rows;
	t->tmpl_out = calloc((size_t) rows * W, sizeof(int16_t));
	t->tmpl_keep = calloc((size_t) rows * W, sizeof(int16_t));
	t->tmpl_keep_any = calloc(rows, 1);
	if(!t->pulse_values || !t->tmpl_out || !t->tmpl_keep || !t->tmpl_keep_any) return(-1);
	for(r = 0; r <= nl; r++)
	{
		const int line0 = r == nl ? 0 : r;                 /* 0-based line within the frame */
		int16_t *o = t->tmpl_out + (size_t) r * W, *k = t->tmpl_keep + (size_t) r * W;
		int x;
		for(x = 0; x < W; x++) o[x] = (int16_t) dp->blank;
		for(s = -1; s <= 1; s++)
		{
			int mask;
			if(r == nl && s < 0) continue;                   /* the stream starts here */
			mask = t->codes[((line0 + s + nl) % nl) + 1] & HTV_LC_SYNC_MASK;
			for(b = 0; b < 5; b++)
			{
				const int base = dp->pulse_off[b] + s * W;
				if(!(mask & (1 << b))) continue;
				for(d = 0; d < dp->pulse_len[b]; d++)
				{
					x = base + d;
					if(x < 0 || x >= W) continue;
					o[x] = (int16_t) (o[x] + t->pulse_values[dp->pulse_pos[b] + d]);
					if(s == 1)
					{
						k[x] = (int16_t) (k[x] + t->pulse_values[dp->pulse_pos[b] + d]);
						/* only where a picture can be drawn: the hsync edge of the next line sits in the front porch */
						if(k[x] && x >= dp->active_left && x < dp->active_left + dp->active_width) t->tmpl_keep_any[r] = 1;
					}
				}
			}
		}
	}
	return(0);
}

/* ---- the build --------------------------------------------------------- */

static double dclamp(double v, double lo, double hi) { return(v < lo ? lo : (v > hi ? hi : v)); }

static uint64_t turns_u64(long double rad)
{
	/* radians -> fraction of a turn in 0.64 fixed point (wraps) */
	long double t = rad / (2.0L * 3.14159265358979323846264338327950288L);
	t -= floorl(t);
	t *= 18446744073709551616.0L;
	if(t >= 18446744073709551616.0L) return(0);
	return((uint64_t) t);
}

static void build_fm_angles(uint64_t *ang, int rate, double frequency, double deviation)
{
	/* The reference's FM NCO multiplies its Q31 phasor by a LUT entry rounded with
	 * lround() (ref video.c:2234-2240); the rotation actually applied per sample is
	 * the argument of that rounded entry, not 2*pi*f/fs. Keep that exact angle. */
	int r;
	for(r = -32768; r <= 32767; r++)
	{
		double d = 2.0 * M_PI / rate * (frequency + (double) r / INT16_MAX * deviation);
		long qi = lround(cos(d) * INT32_MAX), qq = lround(sin(d) * INT32_MAX);
		ang[r + 32768] = turns_u64(atan2l((long double) qq, (long double) qi));
	}
}

static uint64_t carrier_angle(int rate, double frequency)
{
	/* AM / offset carriers: one constant Q31 delta (ref video.c:2352-2354, 4599-4601) */
	double d = 2.0 * M_PI / rate * frequency;
	long qi = lround(cos(d) * INT32_MAX), qq = lround(sin(d) * INT32_MAX);
	return(turns_u64(atan2l((long double) qq, (long double) qi)));
}

htv_tables_t *htv_tables_create(const htv_config_t *conf, unsigned int sample_rate)
{
	struct htv_tables_t *t;
	htv_config_t *c;
	htv_dparams_t *dp;
	double line_s, d, slevel;
	int i, n;

	if(!conf || sample_rate == 0) return(NULL);
	if(conf->type != HTV_RASTER_625 && conf->type != HTV_RASTER_525)
	{
		fprintf(stderr, "hacktv_b200: raster type %d is not on the accelerated path\n", conf->type);
		return(NULL);
	}
	if(conf->modulation == HTV_FM && conf->fm_energy_dispersal != 0)
	{
		fprintf(stderr, "hacktv_b200: FM energy dispersal is not on the accelerated path\n");
		return(NULL);
	}

	t = calloc(1, sizeof(*t));
	if(!t) return(NULL);
	t->conf = *conf;
	t->rate = sample_rate;
	c = &t->conf;
	dp = &t->dp;

	/* defaults, ref video.c:3832-3837 */
	if(c->hline <= 0 && c->interlaced != 0) c->hline = (c->lines + 1) / 2;
	if(c->gamma <= 0) c->gamma = 1.0;
	if(c->rw_co <= 0) c->rw_co = 0.299;
	if(c->gw_co <= 0) c->gw_co = 0.587;
	if(c->bw_co <= 0) c->bw_co = 0.114;

	/* geometry, ref video.c:3844-3853 */
	line_s = (double) c->frame_rate_den / c->frame_rate_num / c->lines;
	dp->rate = sample_rate;
	dp->W = round((double) sample_rate * line_s);
	dp->half_width = round((double) sample_rate * line_s / 2);
	dp->active_left = round(sample_rate * c->active_left);
	dp->active_width = ceil(sample_rate * c->active_width);
	if(dp->active_width > dp->W) dp->active_width = dp->W;
	dp->lines = c->lines;
	dp->hline = c->hline;
	dp->active_lines = c->active_lines;
	dp->raster = c->type;
	dp->colour_mode = c->colour_mode;
	dp->complex_out = c->output_type == HTV_INT16_COMPLEX;
	dp->sample_type = HTV_TYPE_INT16;
	dp->interlaced = c->interlaced;
	dp->volume = c->volume;
	dp->swap_iq = c->swap_iq;

	/* levels, ref video.c:3855-3881 */
	/* slevel: sub-carrier level; 1.0 when FM modulating, else the overall level (ref video.c:3856-3860) */
	slevel = c->modulation == HTV_FM ? 1.0 : c->level;
	dp->vlevel = c->video_level * slevel;
	if(c->invert_video)
	{
		double w = c->white_level;
		c->white_level = c->sync_level;
		c->sync_level = w;
		c->blanking_level = c->sync_level - (c->blanking_level - c->white_level);
		c->black_level = c->sync_level - (c->black_level - c->white_level);
	}
	dp->blank = (int16_t) round(c->blanking_level * dp->vlevel * INT16_MAX);

	/* sync pulses */
	{
		const double where[5] = { 0, 0, 0, line_s / 2, line_s / 2 };
		const double wide[5] = { c->hsync_width, c->vsync_short_width, c->vsync_long_width,
		                         c->vsync_short_width, c->vsync_long_width };
		int16_t *buf = calloc(5 * (dp->W + 8), sizeof(int16_t));
		int level = (int) ((c->sync_level - c->blanking_level) * dp->vlevel * INT16_MAX);
		n = 0;
		for(i = 0; i < 5; i++)
		{
			dp->pulse_pos[i] = n;
			dp->pulse_len[i] = build_pulse(buf + n, &dp->pulse_off[i], where[i] * sample_rate,
				wide[i] * sample_rate, c->sync_rise * IRT1090 * sample_rate, level);
			n += dp->pulse_len[i];
		}
		t->pulse_values = buf;
		t->npulse_values = n;
	}

	/* RGB -> YUV constants; the 16M-entry LUT of the reference is replaced by
	 * evaluating its formula per pixel in fp64 (same operation order) */
	for(i = 0; i < 256; i++) t->glut[i] = pow((double) i / 255, 1 / c->gamma);
	dp->rw = c->rw_co; dp->gw = c->gw_co; dp->bw = c->bw_co;
	dp->eu = c->eu_co; dp->ev = c->ev_co;
	dp->black_level = c->black_level;
	dp->white_minus_black = c->white_level - c->black_level;
	dp->uv_scale = (c->white_level - c->black_level) * dp->vlevel;
	{
		/* black pixel levels (ref video.c:2965,2981: yuv_level_lookup[0x000000]) */
		double y = (c->black_level + (0.0 * (c->white_level - c->black_level))) * dp->vlevel, u = 0, v = 0;
		if(c->colour_mode == HTV_SECAM)
		{
			u = (0.0 + SECAM_CB_FREQ - SECAM_FM_FREQ) / SECAM_FM_DEV;
			v = (0.0 + SECAM_CR_FREQ - SECAM_FM_FREQ) / SECAM_FM_DEV;
		}
		dp->black_y = (int16_t) round(dclamp(y, -1, 1) * INT16_MAX);
		dp->black_u = (int16_t) round(dclamp(u, -1, 1) * INT16_MAX);
		dp->black_v = (int16_t) round(dclamp(v, -1, 1) * INT16_MAX);
	}

	build_codes(t);
	if(build_templates(t) != 0)
	{
		fprintf(stderr, "hacktv_b200: out of memory for the line templates\n");
		htv_tables_free(t);
		return(NULL);
	}

	if(c->colour_mode == HTV_PAL || c->colour_mode == HTV_NTSC)
	{
		/* subcarrier LUT, ref video.c:3961-3987 */
		int64_t num = (int64_t) sample_rate * c->colour_carrier_den, den = c->colour_carrier_num;
		int64_t g = gcd64(num, den);
		size_t k;
		num /= g; den /= g;
		dp->clut_width = (uint32_t) num;
		t->clut_len = (size_t) num + dp->W;
		t->clut = malloc(t->clut_len * sizeof(htv_c16_t));
		if(!t->clut) { htv_tables_free(t); return(NULL); }
		d = 2.0 * M_PI * ((double) den / num);
		for(k = 0; k < t->clut_len; k++)
		{
			t->clut[k].i = round(cos(d * k) * INT16_MAX);
			t->clut[k].q = round(sin(d * k) * INT16_MAX);
		}

		if(c->colour_bw > 0)
		{
			double taps[HTV_MAX_CTAPS + 1];
			n = ((int) ceil(sample_rate / 1.35e6 / (c->colour_bw / 1.4e6))) | 1;
			if(n > HTV_MAX_CTAPS)
			{
				fprintf(stderr, "hacktv_b200: %d chroma taps exceed the supported %d\n", n, HTV_MAX_CTAPS);
				htv_tables_free(t);
				return(NULL);
			}
			gaussian(taps, n, sample_rate, c->colour_bw, 1);
			quantise(dp->chroma_taps, taps, n, 1);
			dp->chroma_ntaps = n;
			/* the kernel filters U/V across line boundaries in one window; that equals the
			 * reference's per-line zero padding as long as the picture keeps n/2 clear of both ends */
			if(n > 17 || dp->active_left < n / 2 || dp->active_left + dp->active_width + n / 2 > dp->W)
			{
				fprintf(stderr, "hacktv_b200: chroma filter (%d taps) / picture geometry not supported\n", n);
				htv_tables_free(t);
				return(NULL);
			}
		}
	}

	if(c->burst_level > 0 || c->colour_mode == HTV_SECAM)
	{
		/* burst / SECAM subcarrier envelope, ref video.c:2194-2214, 4017-4048, 4143-4151 */
		double rise = c->burst_rise * IRT1090;
		double lvl = c->colour_mode == HTV_SECAM ? 1.0 :
			c->burst_level * (c->white_level - c->blanking_level) / 2 * dp->vlevel;
		dp->burst_left = round(sample_rate * (c->burst_left - c->burst_rise / 2));
		dp->burst_width = t->burst_width = ceil(sample_rate * (c->burst_width + rise));
		t->burst_win = malloc(sizeof(int16_t) * (t->burst_width + 1));
		for(i = 0; i < t->burst_width; i++)
		{
			double tt = 1.0 / sample_rate * i;
			t->burst_win[i] = round(edge_window(tt, rise / 2, c->burst_width, rise) * lvl * INT16_MAX);
		}
		if(c->colour_mode == HTV_PAL)
		{
			double ph = 135.0 * (M_PI / 180.0);
			dp->burst_i = (int16_t) round(cos(ph) * INT16_MAX);
			dp->burst_q = (int16_t) round(sin(ph) * INT16_MAX);
		}
		else if(c->colour_mode == HTV_NTSC)
		{
			dp->burst_i = -INT16_MAX;
			dp->burst_q = 0;
		}
	}

	if(c->colour_mode == HTV_SECAM)
	{
		/* ref video.c:4075-4141 */
		double taps[51], a;
		int r;

		dp->secam_level = (int16_t) round(INT16_MAX * ((c->white_level - c->blanking_level) * dp->vlevel));
		t->secam_fm_lut = malloc(sizeof(htv_c32_t) * 65536);
		t->secam_bell = malloc(sizeof(htv_c16_t) * 65536);
		for(r = -32768; r <= 32767; r++)
		{
			double f0 = 4.286e6, f, lq, rq, dd;
			d = 2.0 * M_PI / sample_rate * (SECAM_FM_FREQ + (double) r / INT16_MAX * SECAM_FM_DEV);
			t->secam_fm_lut[r + 32768].i = lround(cos(d) * INT32_MAX);
			t->secam_fm_lut[r + 32768].q = lround(sin(d) * INT32_MAX);
			/* bell filter complex gain, ref video.c:2172-2185 */
			f = SECAM_FM_FREQ + (double) r * SECAM_FM_DEV / INT16_MAX;
			f = f / f0 - f0 / f;
			lq = 16.0 * f;
			rq = 1.26 * f;
			dd = 1.0 + rq * rq;
			t->secam_bell[(uint16_t) r].i = lround(0.115 * (1.0 + lq * rq) / dd * INT16_MAX);
			t->secam_bell[(uint16_t) r].q = lround(0.115 * (lq - rq) / dd * INT16_MAX);
		}
		dp->iir_a1 = -0.90456054; dp->iir_b0 = 2.90456054; dp->iir_b1 = -2.80912108;
		lowpass(taps, 15, sample_rate, 1.70e6, 1.0);
		quantise(dp->secam_lpf, taps, 15, 1);
		bandreject(taps, 51, sample_rate, SECAM_FM_FREQ - 1e6, SECAM_FM_FREQ + 1e6, 1.0);
		taps[51 / 2] += 0.5;
		for(a = 0, i = 0; i < 51; i++) a += taps[i];
		a = a / 1.0;
		for(i = 0; i < 51; i++) taps[i] /= a;
		quantise(dp->secam_notch, taps, 51, 1);
		/* secam_pad: the notch taps are symmetric after quantisation (the raster kernel folds them pairwise) */
		dp->secam_pad = 1;
		for(i = 0; i < 25; i++) if(dp->secam_notch[i] != dp->secam_notch[50 - i]) dp->secam_pad = 0;
		dp->secam_dmin[0] = lround((SECAM_CB_FREQ - SECAM_FM_FREQ - 350e3) / SECAM_FM_DEV * INT16_MAX);
		dp->secam_dmax[0] = lround((SECAM_CB_FREQ - SECAM_FM_FREQ + 506e3) / SECAM_FM_DEV * INT16_MAX);
		dp->secam_dmin[1] = lround((SECAM_CR_FREQ - SECAM_FM_FREQ - 506e3) / SECAM_FM_DEV * INT16_MAX);
		dp->secam_dmax[1] = lround((SECAM_CR_FREQ - SECAM_FM_FREQ + 350e3) / SECAM_FM_DEV * INT16_MAX);
	}

	if(c->vfilter)
	{
		/* ref video.c:3653-3764 */
		double lp[HTV_VF_NTAPS];
		if(c->modulation == HTV_FM)
		{
			/* ref video.c:3678-3740: a fixed CCIR-405 pre-emphasis table per standard and rate */
			const double *taps;
			#define FMT(a) do { taps = a; dp->fmv_ntaps = sizeof(a) / sizeof(double); } while(0)
			if(c->lines == 525)
			{
				if(sample_rate == 18000000) FMT(htv_fm_525_18_taps);
				else FMT(htv_fm_525_2025_taps);
			}
			else
			{
				if(sample_rate == 14000000) FMT(htv_fm_625_14_taps);
				else if(sample_rate == 20000000) FMT(htv_fm_625_20_taps);
				else if(sample_rate == 28000000) FMT(htv_fm_625_28_taps);
				else FMT(htv_fm_625_2025_taps);
			}
			#undef FMT
			quantise(dp->fmv_taps, taps, dp->fmv_ntaps, 1);
			dp->shift = dp->W;
		}
		else
		{
		if(c->modulation == HTV_VSB)
		{
			/* complex band-pass = low-pass shifted to the band centre, ref fir.c:230-255 */
			double taps[HTV_VF_NTAPS * 2];
			double freq = M_PI * (c->vsb_upper_bw + -c->vsb_lower_bw) / sample_rate;
			double phase = -freq * (HTV_VF_NTAPS >> 1);
			lowpass(lp, HTV_VF_NTAPS, sample_rate, (c->vsb_upper_bw - -c->vsb_lower_bw) / 2, 1);
			for(i = 0; i < HTV_VF_NTAPS; i++, phase += freq)
			{
				taps[i * 2 + 0] = lp[i] * cos(phase);
				taps[i * 2 + 1] = lp[i] * sin(phase);
			}
			quantise(dp->vf_i, taps + 0, HTV_VF_NTAPS, 2);
			quantise(dp->vf_q, taps + 1, HTV_VF_NTAPS, 2);
			dp->vf_type = 3;
		}
		else
		{
			lowpass(lp, HTV_VF_NTAPS, sample_rate, c->video_bw, 1);
			quantise(dp->vf_i, lp, HTV_VF_NTAPS, 1);
			dp->vf_type = 1;
		}
		/* the kernel folds the taps pairwise: I (and the real low-pass) symmetric, Q antisymmetric */
		for(i = 0; i < HTV_VF_NTAPS / 2; i++)
		{
			if(dp->vf_i[i] != dp->vf_i[HTV_VF_NTAPS - 1 - i] ||
			   (dp->vf_type == 3 && dp->vf_q[i] != -dp->vf_q[HTV_VF_NTAPS - 1 - i]))
			{
				fprintf(stderr, "hacktv_b200: video filter taps are not (anti)symmetric after quantisation\n");
				htv_tables_free(t);
				return(NULL);
			}
		}
		if(dp->vf_type == 3 && dp->vf_q[HTV_VF_NTAPS / 2] != 0)
		{
			fprintf(stderr, "hacktv_b200: VSB centre Q tap is not zero\n");
			htv_tables_free(t);
			return(NULL);
		}
		/* the filter's one-line pipeline delay makes the audio stages run one
		 * line ahead of the emitted stream (ref video.c:3244,3268; SURVEY.md §9 V2) */
		dp->shift = dp->W;
		}
	}

	if(c->modulation == HTV_FM)
	{
		/* ref video.c:4564-4570: carrier 0 Hz, deviation fm_deviation per unit of signal */
		dp->have_fmv = 1;
		dp->fmv_level = (int16_t) round(INT16_MAX * (c->fm_level * c->level));
		t->fmv_ang = malloc(sizeof(uint64_t) * 65536);
		build_fm_angles(t->fmv_ang, sample_rate, 0, c->fm_deviation);
	}

	/* audio subcarriers, ref video.c:4404-4558 */
	if(c->fm_mono_level > 0 && c->fm_mono_carrier != 0)
	{
		dp->have_fm = 1;
		dp->fm_level = (int16_t) round(INT16_MAX * (c->fm_mono_level * slevel));
		t->fm_ang = malloc(sizeof(uint64_t) * 65536);
		build_fm_angles(t->fm_ang, sample_rate, c->fm_mono_carrier, c->fm_mono_deviation);
		{
			/* (cos, sin) of 8 of those steps: the fused line kernel derives a lane's samples 8 apart from the first by rotation */
			int r;
			t->fm_rot8 = malloc(sizeof(float) * 2 * 65536);
			for(r = 0; r < 65536; r++)
			{
				long double a = (long double) (int64_t) (t->fm_ang[r] << 3) * 0x1p-64L * 2.0L * 3.14159265358979323846264338327950288L;
				t->fm_rot8[2 * r] = (float) cosl(a);
				t->fm_rot8[2 * r + 1] = (float) sinl(a);
			}
		}
		if(c->fm_mono_preemph)
		{
			const double *v = c->fm_mono_preemph == HTV_50US ? audio_50us :
			                  c->fm_mono_preemph == HTV_75US ? audio_75us : audio_j17;
			quantise(t->afir_v, v, HTV_AFIR_N, 1);
			quantise(t->afir_f, audio_flat, HTV_AFIR_N, 1);
			for(i = 0; i < HTV_LIM_W; i++)
			{
				t->lim_shape[i] = lround((1.0 - cos(2.0 * M_PI / (HTV_LIM_W + 1) * (i + 1))) * 0.5 * INT16_MAX);
			}
			dp->have_lim = 1;
		}
	}

	if(c->am_audio_level > 0 && c->am_mono_carrier != 0)
	{
		dp->have_am = 1;
		dp->am_level = (int16_t) round(INT16_MAX * (c->am_audio_level * slevel));
		dp->am_ang = carrier_angle(sample_rate, c->am_mono_carrier);
	}

	if(c->nicam_level > 0 && c->nicam_carrier != 0)
	{
		/* ref nicam728.c:257-326 */
		double sps = (double) sample_rate / 364000.0;
		unsigned int freq = (unsigned int) c->nicam_carrier;
		int64_t g;
		int x, h;

		dp->have_nicam = 1;
		t->nicam_ntaps = dp->nicam_ntaps = ((unsigned int) (sps * 5) + 1) | 1;
		t->nicam_taps = malloc(sizeof(int16_t) * t->nicam_ntaps);
		h = t->nicam_ntaps / 2;
		for(x = -h; x <= h; x++)
		{
			double xx = (double) x / h;
			double ham = (xx < -1 || xx > 1) ? 0 : 0.54 - 0.46 * cos((M_PI * (1.0 + xx)));
			double r = root_rc(((double) x) / sps, c->nicam_beta, 1.0) * ham;
			r *= M_SQRT1_2 * INT16_MAX * (c->nicam_level * slevel);
			t->nicam_taps[x + h] = lround(r);
		}
		g = gcd64(sample_rate, HTV_NICAM_SYMBOL_RATE);
		dp->nicam_F = sample_rate / g;         /* samples per ...            */
		dp->nicam_D = HTV_NICAM_SYMBOL_RATE / g; /* ... this many symbols      */
		/* padded pulse table the kernel stages in shared memory: 8 zeros, the pulse, zeros
		 * out to the farthest offset 7 overlapping symbols + 4 samples can ask for */
		dp->nicam_tpad_len = 8 + 8 * (int) ((sample_rate + HTV_NICAM_SYMBOL_RATE - 1) / HTV_NICAM_SYMBOL_RATE) + 8;
		if(dp->nicam_tpad_len < 8 + dp->nicam_ntaps + 8) dp->nicam_tpad_len = 8 + dp->nicam_ntaps + 8;
		{
			/* Pulse-shaping table. Symbols start every sps or sps-1 samples (ref nicam728.c:399-407)
			 * and the pulse spans < 6 symbol periods, so a sample's baseband value is decided by
			 * its offset into the current symbol, the polarities of the 6 latest symbols and where
			 * (if anywhere) the rarer of the two spacings occurs among the 5 gaps between them:
			 *   lut[(g * 64 + pattern) * sps + phi],  g = 0 none, 1..5 = that gap (1 = newest)
			 * pattern bit j = polarity of the j-th latest symbol (1 = +). Exact integers. */
			const int sps_i = (int) ((sample_rate + HTV_NICAM_SYMBOL_RATE - 1) / HTV_NICAM_SYMBOL_RATE);
			const int64_t gg = gcd64(sample_rate, HTV_NICAM_SYMBOL_RATE);
			const int D = (int) (HTV_NICAM_SYMBOL_RATE / gg), F = (int) (sample_rate / gg);
			const int nshort = sps_i * D - F;              /* gaps of sps-1 per D symbols */
			const int minor_is_short = nshort * 2 <= D;
			const int nminor = minor_is_short ? nshort : D - nshort;
			dp->nicam_sps = sps_i;
			dp->nicam_minor_short = minor_is_short;
			dp->nicam_lut_ok = nminor * 5 < D && t->nicam_ntaps <= 6 * (sps_i - 1) && sps_i >= 8;
			if(dp->nicam_lut_ok)
			{
				const int major = minor_is_short ? sps_i : sps_i - 1, minor = minor_is_short ? sps_i - 1 : sps_i;
				int gi, pat, phi, j;
				t->nicam_lut_len = 6 * 64 * sps_i;
				t->nicam_lut = calloc(t->nicam_lut_len + HTV_NICAM_LUT_PAD, sizeof(int16_t));
				for(gi = 0; gi < 6; gi++) for(pat = 0; pat < 64; pat++) for(phi = 0; phi < sps_i; phi++)
				{
					int off = 0, v = 0;
					for(j = 0; j < 6; j++)
					{
						if(j > 0) off += (gi == j) ? minor : major;
						if(phi + off < t->nicam_ntaps) v += ((pat >> j) & 1) ? t->nicam_taps[phi + off] : -t->nicam_taps[phi + off];
					}
					t->nicam_lut[(gi * 64 + pat) * sps_i + phi] = (int16_t) v;
				}
			}
		}
		dp->nicam_tpad_len = (dp->nicam_tpad_len + 7) & ~7;
		t->nicam_tpad = calloc(dp->nicam_tpad_len, sizeof(int16_t));
		memcpy(t->nicam_tpad + 8, t->nicam_taps, sizeof(int16_t) * t->nicam_ntaps);
		g = gcd64(sample_rate, freq);
		t->nicam_cc_len = dp->nicam_cc_len = sample_rate / g;
		/* W + 64 entries past the period, so a line can index it from (m0 mod period) without wrapping */
		t->nicam_cc = malloc(sizeof(htv_c16_t) * (t->nicam_cc_len + dp->W + 64));
		d = 2.0 * M_PI / t->nicam_cc_len * (freq / g);
		for(x = 0; x < t->nicam_cc_len; x++)
		{
			t->nicam_cc[x].i = round(cos(d * x) * 1.0 * INT16_MAX);
			t->nicam_cc[x].q = round(sin(d * x) * 1.0 * INT16_MAX);
		}
		for(x = t->nicam_cc_len; x < t->nicam_cc_len + dp->W + 64; x++) t->nicam_cc[x] = t->nicam_cc[x - t->nicam_cc_len];
		{
			/* PRN whitening sequence, ref nicam728.c:96-125 */
			int poly = 0x1FF, b;
			for(x = 0; x < 90; x++)
			{
				t->nicam_prn[x] = 0;
				for(b = 0; b < 8; b++)
				{
					uint8_t bit = (poly & 1) ^ ((poly >> 4) & 1);
					poly = (poly >> 1) | (bit << 8);
					t->nicam_prn[x] = (t->nicam_prn[x] << 1) | bit;
				}
			}
		}
	}

	if(c->offset != 0)
	{
		/* Frequency-offset mixer, ref video.c:3482-3515, 4592-4605. The reference
		 * starts its Q31 phasor at INT16_MAX (not INT32_MAX), so for the first
		 * 32767 samples `phase >> 16` is only 0 or -1; run that start-up exactly
		 * once here and hand the device the two sign bits per sample plus the
		 * phase the first renormalisation lands on. */
		htv_c32_t ph = { INT16_MAX, 0 }, dl;
		double dd = 2.0 * M_PI / sample_rate * c->offset;
		int k;
		dl.i = lround(cos(dd) * INT32_MAX);
		dl.q = lround(sin(dd) * INT32_MAX);
		dp->have_offset = 1;
		dp->offset_ang = turns_u64(atan2l((long double) dl.q, (long double) dl.i));
		t->offset_start_len = 32767;
		t->offset_start = malloc(32768);
		for(k = 0; k < 32767; k++)
		{
			int64_t ni = (int64_t) ph.i * dl.i - (int64_t) ph.q * dl.q;
			int64_t nq = (int64_t) ph.i * dl.q + (int64_t) ph.q * dl.i;
			ph.i = (int32_t) (ni >> 31);
			ph.q = (int32_t) (nq >> 31);
			t->offset_start[k] = ((ph.i >> 16) & 1) | (((ph.q >> 16) & 1) << 1);
		}
		dp->offset_phase0 = turns_u64(atan2l((long double) ph.q, (long double) ph.i));
	}

	return(t);
}

/* ref vid_init video.c:3839-3853 with pixel_rate != sample_rate, _init_vresampler video.c:3627-3651,
 * fir_int16_resampler_init fir.c:393-428, fir_int16_init fir.c:263-295 */
htv_tables_t *htv_tables_create2(const htv_config_t *conf, unsigned int sample_rate, unsigned int pixel_rate)
{
	htv_tables_t *t;
	double line_s, *taps;
	int64_t g;
	int ntaps, ph, col;

	if(pixel_rate == 0 || pixel_rate == sample_rate) return(htv_tables_create(conf, sample_rate));
	if(!conf || sample_rate == 0) return(NULL);
	if(conf->modulation == HTV_FM)
	{
		fprintf(stderr, "hacktv_b200: --pixelrate with FM video is not on the accelerated path\n");
		return(NULL);
	}
	t = htv_tables_create(conf, sample_rate);
	if(!t) return(NULL);
	line_s = (double) t->conf.frame_rate_den / t->conf.frame_rate_num / t->conf.lines;
	t->rs_wp = round((double) pixel_rate * line_s);
	g = gcd64(sample_rate, pixel_rate);
	t->rs_I = (int) (sample_rate / g);
	t->rs_D = (int) (pixel_rate / g);
	if(((int64_t) t->rs_wp * t->rs_I) % t->rs_D != 0 || (int64_t) t->rs_wp * t->rs_I / t->rs_D != t->dp.W)
	{
		/* the reference lets the line width vary from line to line then (fir_int16_process returns what
		 * the inputs of a line yield); the batched path needs one width */
		fprintf(stderr, "hacktv_b200: pixel rate %u -> sample rate %u does not keep the line width constant\n", pixel_rate, sample_rate);
		htv_tables_free(t);
		return(NULL);
	}
	ntaps = (21 * t->rs_I) | 1;
	taps = calloc(ntaps, sizeof(double));
	if(!taps) { htv_tables_free(t); return(NULL); }
	if(t->rs_I > t->rs_D) lowpass(taps, ntaps, t->rs_I, 0.45, t->rs_I);
	else lowpass(taps, ntaps, t->rs_I, 0.45 * t->rs_I / t->rs_D, t->rs_I);
	t->rs_ataps = (ntaps + t->rs_I - 1) / t->rs_I;
	t->rs_taps = calloc((size_t) t->rs_I * t->rs_ataps, sizeof(int16_t));
	if(!t->rs_taps) { free(taps); htv_tables_free(t); return(NULL); }
	for(ph = 0; ph < t->rs_I; ph++) for(col = 0; col < t->rs_ataps; col++)
	{
		/* fir.c:281-289: phase ph, column col holds tap[ntaps - I + ph - col I] */
		const int idx = ntaps - t->rs_I + ph - col * t->rs_I;
		if(idx >= 0 && idx < ntaps) t->rs_taps[ph * t->rs_ataps + col] = (int16_t) lround(taps[idx] * 32767.0);
	}
	free(taps);
	/* one more two-line stage in front of the sound carriers, the offset mixer and the passthru
	 * stream: they run a further line ahead (measured on the reference, DESIGN.md section 2) */
	t->dp.shift += t->dp.W;
	return(t);
}

void htv_tables_free(htv_tables_t *t)
{
	if(!t) return;
	free(t->rs_taps);
	free(t->codes); free(t->pulse_values); free(t->clut); free(t->burst_win);
	free(t->tmpl_out); free(t->tmpl_keep); free(t->tmpl_keep_any);
	free(t->fm_ang); free(t->fm_rot8); free(t->fmv_ang); free(t->nicam_taps); free(t->nicam_tpad); free(t->nicam_lut); free(t->nicam_cc);
	free(t->secam_fm_lut); free(t->secam_bell); free(t->offset_start); free(t->scratch);
	free(t);
}

/* ---- named views for tests --------------------------------------------- */

static const int32_t *view16(struct htv_tables_t *t, const int16_t *v, int n, int *count)
{
	int i;
	free(t->scratch);
	t->scratch = malloc(sizeof(int32_t) * (n > 0 ? n : 1));
	for(i = 0; i < n; i++) t->scratch[i] = v[i];
	*count = n;
	return(t->scratch);
}

static const int32_t *view32(struct htv_tables_t *t, const int32_t *v, int n, int *count)
{
	free(t->scratch);
	t->scratch = malloc(sizeof(int32_t) * (n > 0 ? n : 1));
	memcpy(t->scratch, v, sizeof(int32_t) * n);
	*count = n;
	return(t->scratch);
}

/* vid_t.white_level, black_level, blanking_level, sync_level (ref video.c:3877-3881; the conf copy was
 * already swapped for --invert-video) */
void htv_tables_levels(const htv_tables_t *t, int levels[4])
{
	const htv_config_t *c = &t->conf;
	levels[0] = (int16_t) round(c->white_level * t->dp.vlevel * INT16_MAX);
	levels[1] = (int16_t) round(c->black_level * t->dp.vlevel * INT16_MAX);
	levels[2] = t->dp.blank;
	levels[3] = (int16_t) round(c->sync_level * t->dp.vlevel * INT16_MAX);
}

const int32_t *htv_tables_get(htv_tables_t *t, const char *name, int *count)
{
	const htv_dparams_t *dp = &t->dp;
	int32_t tmp[8];
	*count = 0;
	if(strncmp(name, "sync", 4) == 0 && name[4] >= '0' && name[4] <= '4' && name[5] == 0)
	{
		int i = name[4] - '0';
		return(view16(t, t->pulse_values + dp->pulse_pos[i], dp->pulse_len[i], count));
	}
	if(!strcmp(name, "sync_off")) return(view32(t, dp->pulse_off, 5, count));
	if(!strcmp(name, "burst_win") && t->burst_win) return(view16(t, t->burst_win, t->burst_width, count));
	if(!strcmp(name, "chroma_taps") && dp->chroma_ntaps) return(view32(t, dp->chroma_taps, dp->chroma_ntaps, count));
	if(!strcmp(name, "vsb_itaps") && dp->vf_type) return(view32(t, dp->vf_i, HTV_VF_NTAPS, count));
	if(!strcmp(name, "fmv_taps") && dp->fmv_ntaps) return(view32(t, dp->fmv_taps, dp->fmv_ntaps, count));
	if(!strcmp(name, "vsb_qtaps") && dp->vf_type == 3) return(view32(t, dp->vf_q, HTV_VF_NTAPS, count));
	if(!strcmp(name, "nicam_taps") && t->nicam_taps) return(view16(t, t->nicam_taps, t->nicam_ntaps, count));
	if(!strcmp(name, "secam_lpf") && t->secam_bell) return(view32(t, dp->secam_lpf, 15, count));
	if(!strcmp(name, "secam_notch") && t->secam_bell) return(view32(t, dp->secam_notch, 51, count));
	if(!strcmp(name, "rs_taps") && t->rs_taps) return(view16(t, t->rs_taps, t->rs_I * t->rs_ataps, count));
	if(!strcmp(name, "rs_geometry") && t->rs_taps)
	{
		tmp[0] = t->rs_I; tmp[1] = t->rs_D; tmp[2] = t->rs_ataps; tmp[3] = t->rs_wp; tmp[4] = dp->shift;
		return(view32(t, tmp, 5, count));
	}
	if(!strcmp(name, "levels"))
	{
		htv_tables_levels(t, tmp);
		return(view32(t, tmp, 4, count));
	}
	if(!strcmp(name, "geometry"))
	{
		tmp[0] = dp->W; tmp[1] = dp->half_width; tmp[2] = dp->active_left;
		tmp[3] = dp->active_width; tmp[4] = dp->burst_left; tmp[5] = dp->burst_width;
		return(view32(t, tmp, 6, count));
	}
	if(!strcmp(name, "codes"))
	{
		int i;
		free(t->scratch);
		t->scratch = malloc(sizeof(int32_t) * t->ncodes);
		for(i = 0; i < t->ncodes; i++) t->scratch[i] = t->codes[i];
		*count = t->ncodes;
		return(t->scratch);
	}
	return(NULL);
}
