/* TEST INFRASTRUCTURE — the parity oracle. NOT part of the product.
 * See htv_oracle.h for scope, pinning and the rules on who may load this.
 *
 * "ref" in comments = /root/reference/src (fsphil/hacktv @ 80d98ea).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include "htv_oracle.h"
#include "fm_video_taps.h"

#define I16MAX 32767
#define I16MIN (-32768)
#define I32MAX 2147483647
#define ORC_RING 8      /* composite lines held: t - 1 .. t + 3 while line t is emitted (SECAM rasters one further) */

typedef struct { int16_t i, q; } c16_t;
typedef struct { int32_t i, q; } c32_t;

static inline int16_t sat16(int32_t a) { return(a < I16MIN ? I16MIN : (a > I16MAX ? I16MAX : a)); }

/* ------------------------------------------------------------------------ */
/* Maths helpers                                                            */
/* ------------------------------------------------------------------------ */

/* ref common.c:23-35 */
static int64_t gcd64(int64_t a, int64_t b)
{
	int64_t c;
	while((c = a % b)) { a = b; b = c; }
	return(b);
}

/* ref common.c:231-257 - integrated raised cosine window */
static double rc_window(double t, double left, double width, double rise)
{
	double r;
	t -= left + width / 2;
	t = fabs(t) - (width - rise) / 2;
	if(t <= 0) r = 1.0;
	else if(t < rise)
	{
		t = 1.0 - t / rise * 2;
		r = 0.5 * (1.0 + t + sin(M_PI * t) / M_PI);
	}
	else r = 0.0;
	return(r);
}

#define IRT1090 2.0738786 /* ref common.h:29 */

/* ref common.c:259-283 - root raised cosine */
static double rrc(double x, double b, double t)
{
	double r;
	if(x == 0)
	{
		r = (1.0 / t) * (1.0 + b * (4.0 / M_PI - 1));
	}
	else if(fabs(x) == t / (4.0 * b))
	{
		r = b / (t * sqrt(2.0)) * ((1.0 + 2.0 / M_PI) * sin(M_PI / (4.0 * b)) + (1.0 - 2.0 / M_PI) * cos(M_PI / (4.0 * b)));
	}
	else
	{
		double t1 = (4.0 * b * (x / t));
		double t2 = (sin(M_PI * (x / t) * (1.0 - b)) + 4.0 * b * (x / t) * cos(M_PI * (x / t) * (1.0 + b)));
		double t3 = (M_PI * (x / t) * (1.0 - t1 * t1));
		r = (1.0 / t) * (t2 / t3);
	}
	return(r);
}

/* ref common.h:80-89 - Q31 complex multiply, arithmetic >> (floor) */
static inline void c32_mul(c32_t *r, const c32_t *a, const c32_t *b)
{
	int64_t i = (int64_t) a->i * b->i - (int64_t) a->q * b->q;
	int64_t q = (int64_t) a->i * b->q + (int64_t) a->q * b->i;
	r->i = (int32_t) (i >> 31);
	r->q = (int32_t) (q >> 31);
}

/* ------------------------------------------------------------------------ */
/* FIR design (ref fir.c:31-255)                                            */
/* ------------------------------------------------------------------------ */

static double i_zero(double x)
{
	double sum, u, halfx, temp;
	int n;
	sum = u = n = 1;
	halfx = x / 2.0;
	do
	{
		temp = halfx / (double) n;
		n += 1;
		temp *= temp;
		u *= temp;
		sum += u;
	}
	while(u >= 1e-21 * sum);
	return(sum);
}

static void kaiser(double *taps, int ntaps, double beta)
{
	double i_beta = 1.0 / i_zero(beta);
	double inm1 = 1.0 / ((double) (ntaps - 1));
	int i;
	taps[0] = i_beta;
	for(i = 1; i < ntaps - 1; i++)
	{
		double temp = 2 * i * inm1 - 1;
		taps[i] = i_zero(beta * sqrt(1.0 - temp * temp)) * i_beta;
	}
	taps[ntaps - 1] = i_beta;
}

/* ref fir.c:89-137 (odd ntaps only here) */
static void design_low_pass(double *taps, int ntaps, double sample_rate, double cutoff, double gain)
{
	int n, M = (ntaps - 1) / 2;
	double fmax, fwT0 = 2.0 * M_PI * cutoff / sample_rate;
	kaiser(taps, ntaps, 7.0);
	for(n = -M; n <= M; n++)
	{
		if(n == 0) taps[n + M] *= fwT0 / M_PI;
		else taps[n + M] *= sin(n * fwT0) / (n * M_PI);
	}
	fmax = taps[0 + M];
	for(n = 1; n <= M; n++) fmax += 2 * taps[n + M];
	gain /= fmax;
	for(n = 0; n < ntaps; n++) taps[n] *= gain;
}

/* ref fir.c:179-228 */
static void design_band_reject(double *taps, int ntaps, double sample_rate, double lo, double hi, double gain)
{
	int n, M = (ntaps - 1) / 2;
	double fmax, fwT0 = 2.0 * M_PI * lo / sample_rate, fwT1 = 2.0 * M_PI * hi / sample_rate;
	kaiser(taps, ntaps, 7.0);
	for(n = -M; n <= M; n++)
	{
		if(n == 0) taps[n + M] *= 1.0 + (fwT0 - fwT1) / M_PI;
		else taps[n + M] *= (sin(n * fwT0) - sin(n * fwT1)) / (n * M_PI);
	}
	fmax = taps[0 + M];
	for(n = 1; n <= M; n++) fmax += 2 * taps[n + M];
	gain /= fmax;
	for(n = 0; n < ntaps; n++) taps[n] *= gain;
}

/* ref fir.c:139-177 */
static int gaussian_ntaps(double sample_rate, double cutoff)
{
	int ntaps = ceil(sample_rate / 1.35e6 / (cutoff / 1.4e6));
	return(ntaps | 1);
}

static void design_gaussian(double *taps, int ntaps, double sample_rate, double cutoff, double gain)
{
	double f = 13.5e6 / sample_rate;
	double s = 354372.0 / cutoff;
	double t, sum, r;
	int x, h = ntaps / 2;
	for(sum = x = 0; x <= h; x++)
	{
		t = (double) x / 5 * f;
		r = 1.0 / s * pow(2.0 * M_PI, 0.5) * pow(M_E, -pow(t, 2.0) / (2.0 * pow(s, 2)));
		sum += r * (x > 0 ? 2 : 1);
		taps[h + x] = taps[h - x] = r;
	}
	gain /= sum;
	for(x = 0; x < ntaps; x++) taps[x] *= gain;
}

/* ref fir.c:230-255 - taps[2*ntaps] out (interleaved re,im), odd ntaps */
static void design_complex_band_pass(double *taps, int ntaps, double sample_rate, double lo, double hi, double gain)
{
	double *lp = malloc(sizeof(double) * ntaps);
	double freq = M_PI * (hi + lo) / sample_rate;
	double phase = -freq * (ntaps >> 1);
	int i;
	design_low_pass(lp, ntaps, sample_rate, (hi - lo) / 2, gain);
	for(i = 0; i < ntaps; i++, phase += freq)
	{
		taps[i * 2 + 0] = lp[i] * cos(phase);
		taps[i * 2 + 1] = lp[i] * sin(phase);
	}
	free(lp);
}

/* ref fir.c:263-295 with interpolation 1: taps quantised with lround(t*32767)
 * and stored in application order (reversed) */
static int16_t *quantise_taps(const double *taps, int ntaps, int stride)
{
	int16_t *it = calloc(ntaps, sizeof(int16_t));
	int i;
	for(i = 0; i < ntaps; i++) it[i] = lround(taps[(ntaps - 1 - i) * stride] * 32767.0);
	return(it);
}

/* ref fir.c:357-375 + 304-355: block mode = centred FIR; the window starts
 * zeroed (left edge sees zeros) and the last ntaps/2 outputs read ntaps/2
 * samples PAST in[samples-1] - the caller's buffer defines what is there.
 * In-place safe (the reference's window holds copies). */
static void fir_block(const int16_t *it, int ntaps, int16_t *out, const int16_t *in, int samples, int step)
{
	int h = ntaps / 2, x, y;
	int16_t *copy = malloc(sizeof(int16_t) * (samples + ntaps));
	for(x = 0; x < h; x++) copy[x] = 0;
	for(x = 0; x < samples + h; x++) copy[h + x] = in[x * step];
	for(x = 0; x < samples; x++)
	{
		int32_t a = 0;
		for(y = 0; y < ntaps; y++) a += copy[x + y] * it[y];
		out[x * step] = sat16(a >> 15);
	}
	free(copy);
}

/* ------------------------------------------------------------------------ */
/* Data tables taken from the reference (filter coefficients / code tables) */
/* ------------------------------------------------------------------------ */

/* ref video.c:2118-2155 - 65-tap 32 kHz audio filters */
static const double fm_audio_flat_taps[65] = {
	 0.000000,-0.000793, 0.000318,-0.001297, 0.000756,-0.002084, 0.001341,-0.003091, 0.001926,-0.004059, 0.002173,
	-0.004543, 0.001586,-0.003982,-0.000386,-0.001819,-0.004219, 0.002351,-0.010158, 0.008641,-0.018108, 0.016785,
	-0.027575, 0.026122,-0.037697, 0.035663,-0.047356, 0.044249,-0.055360, 0.050742,-0.060650, 0.054238, 0.937500,
	 0.054238,-0.060650, 0.050742,-0.055360, 0.044249,-0.047356, 0.035663,-0.037697, 0.026122,-0.027575, 0.016785,
	-0.018108, 0.008641,-0.010158, 0.002351,-0.004219,-0.001819,-0.000386,-0.003982, 0.001586,-0.004543, 0.002173,
	-0.004059, 0.001926,-0.003091, 0.001341,-0.002084, 0.000756,-0.001297, 0.000318,-0.000793,-0.000000
};
static const double fm_audio_50us_taps[65] = {
	 0.001234,-0.002637, 0.002903,-0.004810, 0.005412,-0.008091, 0.008855,-0.012171, 0.012482,-0.015806, 0.014595,
	-0.016860, 0.012742,-0.012646, 0.004202,-0.000532,-0.013336, 0.021334,-0.041037, 0.053332,-0.078322, 0.093873,
	-0.122521, 0.139174,-0.168825, 0.183024,-0.210266, 0.214647,-0.236618, 0.196560,-0.226183,-0.606600, 2.497308,
	-0.606600,-0.226183, 0.196560,-0.236618, 0.214647,-0.210266, 0.183024,-0.168825, 0.139174,-0.122521, 0.093873,
	-0.078322, 0.053332,-0.041037, 0.021334,-0.013336,-0.000532, 0.004202,-0.012646, 0.012742,-0.016860, 0.014595,
	-0.015806, 0.012482,-0.012171, 0.008855,-0.008091, 0.005412,-0.004810, 0.002903,-0.002637, 0.001234
};
static const double fm_audio_75us_taps[65] = {
	 0.001981,-0.003755, 0.004472,-0.006942, 0.008239,-0.011739, 0.013420,-0.017690, 0.018901,-0.022955, 0.022160,
	-0.024370, 0.019556,-0.017960, 0.007049, 0.000170,-0.018791, 0.032752,-0.059706, 0.080325,-0.114856, 0.140480,
	-0.180353, 0.207455,-0.249292, 0.271550,-0.312119, 0.315065,-0.356561, 0.275266,-0.363286,-0.992136, 3.546394,
	-0.992136,-0.363286, 0.275266,-0.356561, 0.315065,-0.312119, 0.271550,-0.249292, 0.207455,-0.180353, 0.140480,
	-0.114856, 0.080325,-0.059706, 0.032752,-0.018791, 0.000170, 0.007049,-0.017960, 0.019556,-0.024370, 0.022160,
	-0.022955, 0.018901,-0.017690, 0.013420,-0.011739, 0.008239,-0.006942, 0.004472,-0.003755, 0.001981
};
static const double fm_audio_j17_taps[65] = {
	-0.000119,-0.000175,-0.000162,-0.000232,-0.000223,-0.000310,-0.000309,-0.000420,-0.000430,-0.000576,-0.000605,
	-0.000801,-0.000864,-0.001135,-0.001253,-0.001644,-0.001860,-0.002446,-0.002844,-0.003776,-0.004531,-0.006130,
	-0.007663,-0.010705,-0.014141,-0.020784,-0.029556,-0.046668,-0.072530,-0.124846,-0.211267,-0.400931, 2.279077,
	-0.400931,-0.211267,-0.124846,-0.072530,-0.046668,-0.029556,-0.020784,-0.014141,-0.010705,-0.007663,-0.006130,
	-0.004531,-0.003776,-0.002844,-0.002446,-0.001860,-0.001644,-0.001253,-0.001135,-0.000864,-0.000801,-0.000605,
	-0.000576,-0.000430,-0.000420,-0.000309,-0.000310,-0.000223,-0.000232,-0.000162,-0.000175,-0.000119
};

/* ref nicam728.c:35-42 - J.17 pre-emphasis, 32 kHz */
#define J17_NTAPS 83
static const int32_t j17_taps[J17_NTAPS] = {
	-1, 0, -1, -1, -1, -1, -1, -1, -1, -1, -2, -2, -3, -3, -3, -3, -5, -5,
	-6, -7, -9, -10, -13, -14, -18, -21, -27, -32, -42, -51, -69, -86, -120,
	-159, -233, -332, -524, -814, -1402, -2372, -4502, 25590, -4502, -2372,
	-1402, -814, -524, -332, -233, -159, -120, -86, -69, -51, -42, -32, -27,
	-21, -18, -14, -13, -10, -9, -7, -6, -5, -5, -3, -3, -3, -3, -2, -2, -1,
	-1, -1, -1, -1, -1, -1, -1, 0, -1
};

/* ref nicam728.c:45-68 */
static const int nicam_step[4] = { 0, 3, 1, 2 };
static const int nicam_syms[4] = { 0, 1, 3, 2 };
static const struct { int factor, shift; } nicam_scale[8] = {
	{ 0, 2 }, { 1, 2 }, { 2, 2 }, { 4, 2 }, { 3, 3 }, { 5, 4 }, { 6, 5 }, { 7, 6 },
};

#define SECAM_FM_DEV  1000e3  /* ref video.c:45-48 */
#define SECAM_FM_FREQ 4328125
#define SECAM_CB_FREQ 4250000
#define SECAM_CR_FREQ 4406250

/* ------------------------------------------------------------------------ */
/* State                                                                    */
/* ------------------------------------------------------------------------ */

typedef struct { int offset, length; int16_t *value; } pulse_t;

typedef struct {          /* ref video.h:90-104 _mod_fm_t (hot-path part) */
	int16_t level;
	int32_t counter;
	c32_t phase;
	c32_t *lut;
	int16_t sample;
} fm_t;

typedef struct {          /* ref video.h:106-114 _mod_am_t */
	int16_t level;
	int32_t counter;
	c32_t phase, delta;
	int16_t sample;
} am_t;

typedef struct {          /* ref fir.h:44-60 fir_int32_t, interpolation 1 */
	int ntaps;
	int32_t *taps;        /* application order */
	int32_t *win;         /* last ntaps inputs, oldest first */
} fir32_t;

typedef struct {          /* ref fir.h:105-123 limiter_t */
	fir32_t vfir, ffir;
	int width;
	int16_t *shape;
	int16_t level;
	int32_t *fix, *var;
	int16_t *att;
	int p, h;
} limiter_t;

typedef struct {          /* ref nicam728.h:50-96 */
	uint8_t mode, reserve;
	unsigned int frame;
	uint8_t prn[90];
	int fir_p;
	int16_t fir_l[J17_NTAPS], fir_r[J17_NTAPS];
	int16_t audio[64];
	int ntaps;
	int16_t *taps;
	int dsym;
	c16_t *bb; int bb_pos; int bb_len;
	int sps, ds, dsl, decimation;
	c16_t *cc; int cc_len, cc_pos;
	uint8_t fbytes[91];
	int frame_bit;
} nicam_t;

struct orc_t {
	orc_params_t p;
	int rate;
	int complex;

	/* geometry / levels: ref video.c:3844-3881 */
	int width, half_width, active_left, active_width;
	int16_t white, black, blank, sync;
	double vlevel, slevel;

	pulse_t syncs[5];

	double glut[256];
	/* memo of the per-colour result (the reference keeps a full 2^24-entry table) */
	uint32_t yuv_key[4096];
	int16_t yuv_val[4096][3];

	/* PAL/NTSC chroma: ref video.c:3961-4048 */
	unsigned int clut_width;
	c16_t *clut;
	int16_t *chroma;            /* 2*W (+pad, zero) U,V interleaved */
	int chroma_ntaps;
	int16_t *chroma_taps;
	c16_t burst_phase;
	int burst_left, burst_width;
	int16_t *burst_win;

	/* SECAM: ref video.c:4075-4162 */
	fm_t fm_secam;
	double iir_a[2], iir_b[2], iir_ix, iir_iy;
	int16_t *secam_lpf;         /* 15 taps */
	int16_t *secam_notch;       /* 51 taps */
	int16_t secam_dmin[2], secam_dmax[2];
	c16_t *secam_bell;          /* 65536 */
	/* The reference's line buffers (video.c:4642-4672) are a ring of `olines`, each with the zero heap's padding past
	 * its W samples. Where the burst window ends past the line (82 + 944 > 1024 at 16 Msps), the subcarrier loop adds
	 * into that padding (video.c:3228), and it is never cleared: what a ring buffer's past SECAM lines added there is
	 * what the luma notch of its next SECAM line reads through its taps ahead of centre, wherever the picture ends
	 * within 25 samples of the line's end (below about 15 Msps; it changes values below about 10). I of samples W, W + 1,
	 * ... per ring buffer. Restated only on request (orc_set_ref_heap) and without a resampler, whose wider output
	 * lines share the ring; otherwise the notch reads zeros past the line, as the CUDA path does. */
	int ref_heap, olines;
	int16_t secam_pad[32][8];

	/* video filter: ref video.c:3653-3764 */
	int vf_type;                /* 0 none, 1 real, 3 real->complex */
	int vf_ntaps;
	int16_t *vf_itaps, *vf_qtaps;

	/* audio: ref video.c:4404-4558 */
	int have_fm, have_am, have_nicam;
	fm_t fm_mono;
	limiter_t lim;
	int have_lim;
	am_t am_mono;
	nicam_t nicam;
	int interp;
	int16_t audio_lr[2];
	int16_t nicam_buf[64];
	int nicam_buf_len;

	/* offset mixer: ref video.c:4592-4605 */
	int32_t off_counter;
	c32_t off_phase, off_delta;

	/* sources */
	const uint32_t *frames; int nframes;
	const int16_t *pcm; size_t pcm_pairs; size_t pcm_pos;
	struct { int line, from, to, value; const int16_t *add; } vbi[64];
	int nvbi;
	int have_fmv; fm_t fm_video;                       /* FM video modulator (video.c:2299-2335) */
	const int16_t *pt; size_t pt_len; size_t pt_pos;   /* passthru stream (complex samples) */

	/* stream state */
	int64_t next_raster;        /* next line index to raster */
	int64_t next_secam;         /* next line index for the SECAM pass */
	int64_t next_emit;          /* next line index to emit */
	int16_t *ring[ORC_RING];    /* composite I, W + pad each */

	/* --pixelrate: the raster side (everything above) runs at `rate` / `width`, the stages from the
	 * resampler on at `srate` / `swidth` (ref video.c:3839-3853, 4361-4368). Equal without a resampler. */
	int srate, swidth;
	int rs_on, rs_I, rs_D, rs_ataps;
	int16_t *rs_taps;           /* [rs_I][rs_ataps], the order fir_int16_init lays them out */
	int16_t *rring[4];          /* resampled lines, swidth each */
	int64_t next_resamp;

	int32_t *tbl;               /* scratch for orc_table */
};

/* ------------------------------------------------------------------------ */
/* Sync pulse LUT: ref vbidata.c:36-81, video.c:3766-3810, 3885-3891        */
/* ------------------------------------------------------------------------ */

static void make_pulse(pulse_t *pl, double offset, double width, double rise, int level)
{
	int x1 = floor(offset - rise / 2);
	int x2 = ceil(offset + width + rise / 2);
	int n = x2 - x1 + 2;
	pl->value = calloc(n, sizeof(int16_t));
	pl->length = 0;
	pl->offset = 0;
	for(; x1 <= x2; x1++)
	{
		double h = rc_window(x1, offset, width, rise) * level;
		int value = round(h);
		if(value != 0)
		{
			if(pl->length == 0) pl->offset = x1;
			for(; pl->length < (x1 - pl->offset); pl->length++) pl->value[pl->length] = 0;
			pl->value[pl->length++] = value;
		}
	}
}

/* ------------------------------------------------------------------------ */
/* RGB -> YUV levels: ref video.c:3905-3959 (evaluated per pixel, not LUT)  */
/* ------------------------------------------------------------------------ */

static double dlimit(double v, double min, double max)
{
	if(v < min) return(min);
	if(v > max) return(max);
	return(v);
}

void orc_yuv(const orc_t *oc, uint32_t c, int16_t yuv[3])
{
	orc_t *o = (orc_t *) oc;
	const orc_params_t *p = &o->p;
	const unsigned int slot = (c ^ (c >> 12)) & 4095;
	if(o->yuv_key[slot] == (c | 0x80000000u))
	{
		yuv[0] = o->yuv_val[slot][0]; yuv[1] = o->yuv_val[slot][1]; yuv[2] = o->yuv_val[slot][2];
		return;
	}
	double level = o->vlevel;
	double r = o->glut[(c & 0xFF0000) >> 16];
	double g = o->glut[(c & 0x00FF00) >> 8];
	double b = o->glut[(c & 0x0000FF) >> 0];
	double y, u, v;

	y = r * p->rw_co
	  + g * p->gw_co
	  + b * p->bw_co;
	u = (b - y) * p->eu_co;
	v = (r - y) * p->ev_co;

	y = (p->black_level + (y * (p->white_level - p->black_level))) * level;

	if(p->colour_mode != ORC_COLOUR_SECAM)
	{
		u *= (p->white_level - p->black_level) * level;
		v *= (p->white_level - p->black_level) * level;
	}
	else
	{
		u = (u + SECAM_CB_FREQ - SECAM_FM_FREQ) / SECAM_FM_DEV;
		v = (v + SECAM_CR_FREQ - SECAM_FM_FREQ) / SECAM_FM_DEV;
	}

	yuv[0] = round(dlimit(y, -1, 1) * I16MAX);
	yuv[1] = round(dlimit(u, -1, 1) * I16MAX);
	yuv[2] = round(dlimit(v, -1, 1) * I16MAX);
	o->yuv_key[slot] = c | 0x80000000u;
	o->yuv_val[slot][0] = yuv[0]; o->yuv_val[slot][1] = yuv[1]; o->yuv_val[slot][2] = yuv[2];
}

/* ------------------------------------------------------------------------ */
/* Modulators                                                               */
/* ------------------------------------------------------------------------ */

/* ref video.c:2218-2243 */
static void fm_init(fm_t *fm, int sample_rate, double frequency, double deviation, double level)
{
	int r;
	fm->level = round(I16MAX * level);
	fm->counter = I16MAX;
	fm->phase.i = I32MAX;
	fm->phase.q = 0;
	fm->sample = 0;
	fm->lut = malloc(sizeof(c32_t) * 65536);
	for(r = I16MIN; r <= I16MAX; r++)
	{
		double d = 2.0 * M_PI / sample_rate * (frequency + (double) r / I16MAX * deviation);
		fm->lut[r - I16MIN].i = lround(cos(d) * I32MAX);
		fm->lut[r - I16MIN].q = lround(sin(d) * I32MAX);
	}
}

/* ref video.c:2259-2276 (phase step + the every-32767-samples renormalise) */
static inline void nco_renorm(c32_t *phase, int32_t *counter)
{
	if(--(*counter) == 0)
	{
		double ra = atan2(phase->q, phase->i);
		phase->i = lround(cos(ra) * I32MAX);
		phase->q = lround(sin(ra) * I32MAX);
		*counter = I16MAX;
	}
}

static inline void fm_add(fm_t *fm, int16_t *dst, int16_t sample)
{
	c32_mul(&fm->phase, &fm->phase, &fm->lut[sample - I16MIN]);
	dst[0] += ((fm->phase.i >> 16) * fm->level) >> 15;
	dst[1] += ((fm->phase.q >> 16) * fm->level) >> 15;
	nco_renorm(&fm->phase, &fm->counter);
}

/* ref video.c:2299-2335 without energy dispersal, 3452-3464: the line's I becomes the
 * modulating signal, I and Q are replaced by the phasor */
static void fmv_line(fm_t *fm, int16_t *iq, int W)
{
	int x;
	for(x = 0; x < W; x++)
	{
		int16_t *d = iq + x * 2;
		c32_mul(&fm->phase, &fm->phase, &fm->lut[d[0] - I16MIN]);
		d[0] = ((fm->phase.i >> 16) * fm->level) >> 15;
		d[1] = ((fm->phase.q >> 16) * fm->level) >> 15;
		nco_renorm(&fm->phase, &fm->counter);
	}
}

/* ref video.c:2278-2297 (SECAM only) */
static inline void fm_cgain(fm_t *fm, int16_t *dst, int16_t sample, const c16_t *g)
{
	c32_mul(&fm->phase, &fm->phase, &fm->lut[sample - I16MIN]);
	dst[0] = (((((fm->phase.i >> 16) * fm->level) >> 15) * g->i) >> 15)
	       - (((((fm->phase.q >> 16) * fm->level) >> 15) * g->q) >> 15);
	nco_renorm(&fm->phase, &fm->counter);
}

/* ref video.c:2343-2378 */
static void am_init(am_t *am, int sample_rate, double frequency, double level)
{
	double d;
	am->level = round(I16MAX * level);
	am->counter = I16MAX;
	am->phase.i = I32MAX;
	am->phase.q = 0;
	am->sample = 0;
	d = 2.0 * M_PI / sample_rate * frequency;
	am->delta.i = lround(cos(d) * I32MAX);
	am->delta.q = lround(sin(d) * I32MAX);
}

static inline void am_add(am_t *am, int16_t *dst, int16_t sample)
{
	c32_mul(&am->phase, &am->phase, &am->delta);
	sample = ((int32_t) sample - I16MIN) / 2;
	dst[0] += ((((am->phase.i >> 16) * sample) >> 15) * am->level) >> 15;
	dst[1] += ((((am->phase.q >> 16) * sample) >> 15) * am->level) >> 15;
	nco_renorm(&am->phase, &am->counter);
}

/* ------------------------------------------------------------------------ */
/* Soft limiter + its int32 FIRs: ref fir.c:623-694, 758-870                */
/* ------------------------------------------------------------------------ */

static void fir32_init(fir32_t *f, const double *taps, int ntaps)
{
	int i;
	f->ntaps = ntaps;
	f->taps = malloc(sizeof(int32_t) * ntaps);
	f->win = calloc(ntaps, sizeof(int32_t));
	for(i = 0; i < ntaps; i++) f->taps[i] = lround(taps[ntaps - 1 - i] * 32767.0);
}

static int32_t fir32_step(fir32_t *f, int32_t in)
{
	int64_t a = 0;
	int y;
	memmove(f->win, f->win + 1, sizeof(int32_t) * (f->ntaps - 1));
	f->win[f->ntaps - 1] = in;
	for(y = 0; y < f->ntaps; y++) a += (int64_t) f->win[y] * (int64_t) f->taps[y];
	a >>= 15;
	return(a < INT32_MIN ? INT32_MIN : (a > INT32_MAX ? INT32_MAX : a));
}

static void limiter_init(limiter_t *s, int16_t level, int width, const double *vtaps, const double *ftaps, int ntaps)
{
	int i;
	memset(s, 0, sizeof(*s));
	fir32_init(&s->vfir, vtaps, ntaps);
	fir32_init(&s->ffir, ftaps, ntaps);
	s->width = width | 1;
	s->shape = malloc(sizeof(int16_t) * s->width);
	for(i = 0; i < s->width; i++)
	{
		s->shape[i] = lround((1.0 - cos(2.0 * M_PI / (s->width + 1) * (i + 1))) * 0.5 * I16MAX);
	}
	s->level = level;
	s->att = calloc(sizeof(int16_t), s->width);
	s->fix = calloc(sizeof(int32_t), s->width);
	s->var = calloc(sizeof(int32_t), s->width);
	s->p = 0;
	s->h = s->width / 2;
}

/* One sample, vin == fin == the sample (as video.c:3322 calls it) */
static int16_t limiter_step(limiter_t *s, int16_t in)
{
	int j;
	int32_t a, b;

	s->var[s->p] = in;
	s->fix[s->p] = in;
	s->att[s->p] = 0;

	s->var[s->p] = fir32_step(&s->vfir, s->var[s->p]);
	s->fix[s->p] = fir32_step(&s->ffir, s->fix[s->p]);

	if(s->fix[s->p] < -s->level) s->fix[s->p] = -s->level;
	else if(s->fix[s->p] > s->level) s->fix[s->p] = s->level;

	s->var[s->p] -= s->fix[s->p];

	if(++s->p == s->width) s->p = 0;
	if(++s->h == s->width) s->h = 0;

	a = abs(s->var[s->h] + s->fix[s->h]);
	if(a > s->level)
	{
		/* int32 arithmetic as the reference's (wraps like -fwrapv on overflow) */
		a = I16MAX - (int32_t) ((uint32_t) (s->level + abs(s->var[s->h]) - a) * (uint32_t) I16MAX) / abs(s->var[s->h]);
		for(j = 0; j < s->width; j++)
		{
			b = (a * s->shape[j]) >> 15;
			if(b > s->att[s->p]) s->att[s->p] = b;
			if(++s->p == s->width) s->p = 0;
		}
	}

	a  = s->fix[s->p];
	a += ((int64_t) s->var[s->p] * (I16MAX - s->att[s->p])) >> 15;

	if(a < -s->level) a = -s->level;
	else if(a > s->level) a = s->level;

	return((int16_t) a);
}

/* ------------------------------------------------------------------------ */
/* NICAM-728: ref nicam728.c                                                */
/* ------------------------------------------------------------------------ */

/* ref nicam728.c:96-125 */
static void nicam_prn(uint8_t prn[90])
{
	int poly = 0x1FF, x, i;
	for(x = 0; x < 90; x++)
	{
		prn[x] = 0x00;
		for(i = 0; i < 8; i++)
		{
			uint8_t b = poly & 1;
			b ^= (poly >> 4) & 1;
			poly >>= 1;
			poly |= b << 8;
			prn[x] <<= 1;
			prn[x] |= b;
		}
	}
}

static uint8_t parity(unsigned int value)
{
	uint8_t p = 0;
	while(value) { p ^= value & 1; value >>= 1; }
	return(p);
}

/* ref nicam728.c:70-94 */
static int nicam_scale_index(const int16_t *pcm, int step)
{
	int i, b = 1;
	for(i = 0; b < 7 && i < 32; i++)
	{
		int16_t s = (*pcm < 0) ? ~*pcm : *pcm;
		while(b < 7 && s >> (b + 8)) b++;
		pcm += step;
	}
	return(b);
}

/* ref nicam728.c:140-249 */
static void nicam_encode_frame(nicam_t *s, const int16_t audio[64])
{
	int16_t d[64];
	int32_t l, r;
	int x, xi, sc[2];
	uint8_t *frame = s->fbytes;

	for(x = 0; x < 32; x++)
	{
		s->fir_l[s->fir_p] = audio[x * 2 + 0];
		s->fir_r[s->fir_p] = audio[x * 2 + 1];
		if(++s->fir_p == J17_NTAPS) s->fir_p = 0;
		for(l = r = xi = 0; xi < J17_NTAPS; xi++)
		{
			l += (int32_t) s->fir_l[s->fir_p] * j17_taps[xi];
			r += (int32_t) s->fir_r[s->fir_p] * j17_taps[xi];
			if(++s->fir_p == J17_NTAPS) s->fir_p = 0;
		}
		d[x * 2 + 0] = l >> 15;
		d[x * 2 + 1] = r >> 15;
	}

	sc[0] = nicam_scale_index(d + 0, 2);
	sc[1] = nicam_scale_index(d + 1, 2);

	for(x = 0; x < 64; x++)
	{
		d[x] = (d[x] >> nicam_scale[sc[x & 1]].shift) & 0x3FF;
		d[x] |= parity(d[x] >> 4) << 10;
		if(x < 54) d[x] ^= ((nicam_scale[sc[x & 1]].factor >> (2 - (x / 2 % 3))) & 1) << 10;
	}

	frame[0] = 0x4E;
	frame[1]  = (((~s->frame) >> 3) & 1) << 7;
	frame[1] |= ((s->mode >> 2) & 1) << 6;
	frame[1] |= ((s->mode >> 1) & 1) << 5;
	frame[1] |= ((s->mode >> 0) & 1) << 4;
	frame[1] |= (s->reserve & 1) << 3;
	for(x = 2; x < 91; x++) frame[x] = 0;

	for(xi = x = 0; x < 64; x++)
	{
		int b;
		for(b = 0; b < 11; b++, d[x] >>= 1)
		{
			if(d[x] & 1) frame[3 + (xi / 8)] |= 1 << (7 - (xi % 8));
			xi += 16;
			if(xi >= 728 - 24) xi -= 728 - 24 - 1;
		}
	}

	for(x = 0; x < 90; x++) frame[x + 1] ^= s->prn[x];
	s->frame++;
}

static double hamming(double x)
{
	if(x < -1 || x > 1) return(0);
	return(0.54 - 0.46 * cos((M_PI * (1.0 + x))));
}

/* ref nicam728.c:257-326 */
static void nicam_init(nicam_t *s, unsigned int sample_rate, unsigned int frequency, double beta, double level)
{
	double sps = (double) sample_rate / 364000.0;
	int x, n;

	memset(s, 0, sizeof(*s));
	s->mode = 0; /* NICAM_MODE_STEREO */
	s->reserve = 1;
	s->ntaps = ((unsigned int) (sps * 5) + 1) | 1;
	s->taps = malloc(sizeof(int16_t) * s->ntaps);
	n = s->ntaps / 2;
	for(x = -n; x <= n; x++)
	{
		double t = ((double) x) / sps;
		double r = rrc(t, beta, 1.0) * hamming((double) x / n);
		r *= M_SQRT1_2 * I16MAX * level;
		s->taps[x + n] = lround(r);
	}
	s->bb = calloc(s->ntaps, sizeof(c16_t));
	s->bb_pos = 0;
	s->bb_len = 0;

	n = gcd64(sample_rate, 364000);
	s->decimation = 364000 / n;
	s->sps = (sample_rate + 364000 - 1) / 364000;
	s->dsl = (s->sps * s->decimation) % (sample_rate / n);
	s->ds = 0;

	n = gcd64(sample_rate, frequency);
	s->cc_len = sample_rate / n;
	s->cc = malloc(sizeof(c16_t) * s->cc_len);
	{
		/* ref common.c:209-229 sin_cint16(length, cycles, 1.0) */
		double d = 2.0 * M_PI / s->cc_len * (frequency / n);
		for(x = 0; x < s->cc_len; x++)
		{
			s->cc[x].i = round(cos(d * x) * 1.0 * I16MAX);
			s->cc[x].q = round(sin(d * x) * 1.0 * I16MAX);
		}
	}
	s->cc_pos = 0;
	nicam_prn(s->prn);
	s->frame_bit = 728;
}

/* ref nicam728.c:342-411 */
static void nicam_output(nicam_t *s, int16_t *iq, int samples)
{
	c16_t *ciq = (c16_t *) iq;
	int x, i;

	for(x = 0; x < samples;)
	{
		for(; x < samples && s->bb_len; x++, s->bb_len--)
		{
			const c16_t *a = &s->bb[s->bb_pos], *b = &s->cc[s->cc_pos];
			int32_t ri = (int32_t) a->i * b->i - (int32_t) a->q * b->q;
			int32_t rq = (int32_t) a->i * b->q + (int32_t) a->q * b->i;
			ciq->i += ri >> 15;
			ciq->q += rq >> 15;
			ciq++;
			s->bb[s->bb_pos].i = 0;
			s->bb[s->bb_pos].q = 0;
			if(++s->bb_pos == s->ntaps) s->bb_pos = 0;
			if(++s->cc_pos == s->cc_len) s->cc_pos = 0;
		}
		if(s->bb_len > 0) break;

		if(s->frame_bit == 728)
		{
			nicam_encode_frame(s, s->audio);
			s->frame_bit = 0;
		}

		s->dsym += nicam_step[(s->fbytes[s->frame_bit >> 3] >> (6 - (s->frame_bit & 0x07))) & 0x03];
		s->dsym &= 0x03;
		s->frame_bit += 2;

		{
			int p = s->bb_pos;
			for(i = 0; i < s->ntaps; i++)
			{
				int16_t r = s->taps[i];
				s->bb[p].i += (nicam_syms[s->dsym] & 1 ? r : -r);
				s->bb[p].q += (nicam_syms[s->dsym] & 2 ? r : -r);
				if(++p == s->ntaps) p = 0;
			}
		}

		s->bb_len = s->sps;
		s->ds += s->dsl;
		if(s->ds >= s->decimation)
		{
			s->bb_len--;
			s->ds -= s->decimation;
		}
	}
}

/* ------------------------------------------------------------------------ */
/* Line codes: ref video.c:2447-2862                                        */
/* ------------------------------------------------------------------------ */

/* 4-char code: [0] first sync h/v/V/_, [1] burst 0/1/2/_, [2] left a/_, [3] right a/v/V/_ */
static const char *line_code(int type, int line)
{
	if(type == ORC_RASTER_625)
	{
		if(line >= 1 && line <= 2) return("V__V");
		if(line == 3) return("V__v");
		if(line >= 4 && line <= 5) return("v__v");
		if(line == 6) return("h1__");
		if(line >= 7 && line <= 22) return("h0__");
		if(line == 23) return("h0_a");
		if(line == 310) return("h1aa");
		if(line >= 311 && line <= 312) return("v__v");
		if(line == 313) return("v__V");
		if(line >= 314 && line <= 315) return("V__V");
		if(line >= 316 && line <= 317) return("v__v");
		if(line == 318) return("v___");
		if(line == 319) return("h2__");
		if(line >= 320 && line <= 335) return("h0__");
		if(line == 622) return("h1aa");
		if(line == 623) return("h_av");
		if(line >= 624 && line <= 625) return("v__v");
		return("h0aa");
	}
	else if(type == ORC_RASTER_525)
	{
		if(line >= 1 && line <= 3) return("v__v");
		if(line >= 4 && line <= 6) return("V__V");
		if(line >= 7 && line <= 9) return("v__v");
		if(line >= 10 && line <= 20) return("h0__");
		if(line == 263) return("h0av");
		if(line >= 264 && line <= 265) return("v__v");
		if(line == 266) return("v__V");
		if(line >= 267 && line <= 268) return("V__V");
		if(line == 269) return("V__v");
		if(line >= 270 && line <= 271) return("v__v");
		if(line == 272) return("v___");
		if(line >= 273 && line <= 282) return("h0__");
		if(line == 283) return("h0_a");
		return("h0aa");
	}
	return("____");
}

static int active_row(int type, int line)
{
	if(type == ORC_RASTER_625) return(line < 313 ? (line - 23) * 2 : (line - 336) * 2 + 1);
	if(type == ORC_RASTER_525) return(line < 265 ? (line - 23) * 2 : (line - 286) * 2 + 1);
	return(-1);
}

/* ref video.c:2886-2895 with our sources: vframe is exactly active_width x
 * active_lines (vframe_x = vframe_y = 0) and reports interlaced = 0 */
static int source_row(const orc_t *o, int line)
{
	int vy = active_row(o->p.type, line);
	if(vy >= 0 && o->p.interlaced != 0 && 0 != o->p.interlaced) vy += 1;
	if(vy < 0 || vy >= o->p.active_lines) vy = -1;
	return(vy);
}

static const uint32_t *frame_for(const orc_t *o, int frame /* 1-based */)
{
	if(!o->frames || o->nframes < 1) return(NULL);
	return(o->frames + (size_t) o->active_width * o->p.active_lines * ((frame - 1) % o->nframes));
}

/* ------------------------------------------------------------------------ */
/* Raster: ref video.c:2864-3066, vbidata.c:186-239                         */
/* ------------------------------------------------------------------------ */

static inline int16_t *ring_line(orc_t *o, int64_t L) { return(o->ring[((L % ORC_RING) + ORC_RING) % ORC_RING]); }

static void blank_line(orc_t *o, int16_t *l)
{
	/* ref video.c:2935-2939 blanks max_width samples: with a resampler that widens the line the
	 * buffer is longer than the raster line, and the block FIRs' reads past the line end
	 * (SURVEY.md section 8c) find the blanking level there instead of the heap */
	const int n = o->swidth > o->width ? o->swidth : o->width;
	int x;
	for(x = 0; x < n; x++) l[x] = o->blank;
}

static void raster_line(orc_t *o, int64_t L)
{
	const int W = o->width;
	int frame = L / o->p.lines + 1;
	int line = L % o->p.lines + 1;
	const char *seq = line_code(o->p.type, line);
	int vy = source_row(o, line);
	int pal = 0;
	int16_t *l = ring_line(o, L);
	const c16_t *lut = NULL;
	int x, b;
	uint8_t sc = 0;

	if(o->p.colour_mode == ORC_COLOUR_PAL || o->p.colour_mode == ORC_COLOUR_NTSC)
	{
		pal  = seq[1] == '0';
		pal |= seq[1] == '1' && (frame & 1) == 0;
		pal |= seq[1] == '2' && (frame & 1) == 1;

		/* video.c:2906-2910: offset advances by width per line, mod the LUT period */
		lut = &o->clut[(unsigned int) (((uint64_t) L * W) % o->clut_width)];

		if(o->p.colour_mode == ORC_COLOUR_PAL && pal && ((frame + line) & 1)) pal = -1;

		if(pal) memset(o->chroma, 0, sizeof(int16_t) * 2 * W);
	}

	/* video.c:2935-2939: the NEXT line is blanked now */
	blank_line(o, ring_line(o, L + 1));

	if(seq[0] == 'h')      sc |= 1 << 0;
	else if(seq[0] == 'v') sc |= 1 << 1;
	else if(seq[0] == 'V') sc |= 1 << 2;
	if(seq[3] == 'v')      sc |= 1 << 3;
	else if(seq[3] == 'V') sc |= 1 << 4;

	/* vbidata_render: add each selected pulse, spilling into the previous /
	 * next line; the very first line has no previous line (width 0 marks a
	 * boundary, vbidata.c:212-224) */
	for(b = 0; b < 5; b++)
	{
		const pulse_t *pl = &o->syncs[b];
		if(!(sc & (1 << b))) continue;
		for(x = 0; x < pl->length; x++)
		{
			int lx = pl->offset + x;
			if(lx < 0)
			{
				if(L == 0) continue;
				ring_line(o, L - 1)[W + lx] += pl->value[x];
			}
			else if(lx >= W) ring_line(o, L + 1)[lx - W] += pl->value[x];
			else l[lx] += pl->value[x];
		}
	}

	if(seq[2] == 'a' || seq[3] == 'a')
	{
		const uint32_t *fb = frame_for(o, frame);
		const uint32_t *row = (fb && vy >= 0) ? fb + (size_t) vy * o->active_width : NULL;
		int al = (seq[2] == 'a' ? o->active_left : (seq[3] == 'a' ? o->half_width : -1));
		int ar = (seq[3] == 'a' ? o->active_left + o->active_width : (seq[2] == 'a' ? o->half_width : -1));
		int16_t yuv[3], black[3];

		orc_yuv(o, 0x000000, black);

		for(x = al; x < o->active_left; x++) l[x] = black[0];
		for(; x < o->active_left + o->active_width && x < ar; x++)
		{
			uint32_t rgb = row ? (row[x - o->active_left] & 0xFFFFFF) : 0x000000;
			orc_yuv(o, rgb, yuv);
			l[x] = yuv[0];
			if(pal)
			{
				o->chroma[x * 2 + 0] = yuv[1];
				o->chroma[x * 2 + 1] = yuv[2];
			}
		}
		for(; x < ar; x++) l[x] = black[0];
	}

	if(pal)
	{
		int16_t *oc = o->chroma;

		if(o->chroma_taps)
		{
			fir_block(o->chroma_taps, o->chroma_ntaps, &oc[0], &oc[0], W, 2);
			fir_block(o->chroma_taps, o->chroma_ntaps, &oc[1], &oc[1], W, 2);
		}

		oc = &o->chroma[o->burst_left * 2];
		for(x = 0; x < o->burst_width; x++, oc += 2)
		{
			oc[0] = (o->burst_phase.i * o->burst_win[x]) >> 15;
			oc[1] = (o->burst_phase.q * o->burst_win[x]) >> 15;
		}

		oc = o->chroma;
		for(x = 0; x < W; x++, oc += 2)
		{
			l[x] += (lut[x].i * oc[1] * pal + lut[x].q * oc[0]) >> 15;
		}
	}
}

/* VBI stages (ref video.c:4213-4402) are registered behind the raster AND the SECAM stage, in front
 * of the video filter: they see - and WSS partly overwrites - the finished composite line */
static void vbi_line(orc_t *o, int64_t L)
{
	const int W = o->width;
	int line = L % o->p.lines + 1;
	int16_t *l = ring_line(o, L);
	int b, x;
	for(b = 0; b < o->nvbi; b++)
	{
		if(o->vbi[b].line != line) continue;
		for(x = o->vbi[b].from; x < o->vbi[b].to && x < W; x++) if(x >= 0) l[x] = (int16_t) o->vbi[b].value;
		if(o->vbi[b].add) for(x = 0; x < W; x++) l[x] = (int16_t) (l[x] + o->vbi[b].add[x]);
	}
}

/* ------------------------------------------------------------------------ */
/* SECAM chroma: ref video.c:3068-3233                                      */
/* ------------------------------------------------------------------------ */

/* The reference's line-buffer count: _add_lineprocess (video.c:3543-3579) over the stages vid_init adds
 * (video.c:4206-4638) for what the oracle restates, as (lines, threaded) in their order. A stage that is not threaded
 * shares its first line with the unthreaded stage before it. */
static int ref_olines(const orc_t *o)
{
	int st[12][2], n = 0, i, total = 0;
	st[n][0] = 3; st[n++][1] = 0;                                    /* raster */
	st[n][0] = 1; st[n++][1] = 1;                                    /* secam */
	if(o->nvbi) { st[n][0] = 1; st[n++][1] = 0; }                    /* wss */
	if(o->rs_on) { st[n][0] = 2; st[n++][1] = 1; }                   /* vresampler */
	if(o->vf_type)                                                   /* vfilter: 1 + its delay (video.c:3759) */
		{ st[n][0] = 1 + (o->vf_ntaps / 2 + o->swidth - 1) / o->swidth; st[n++][1] = 1; }
	st[n][0] = 1; st[n++][1] = 1;                                    /* audio */
	if(o->have_fmv) { st[n][0] = 1; st[n++][1] = 1; }                /* fmmod */
	if(o->p.swap_iq) { st[n][0] = 1; st[n++][1] = 0; }               /* swap_iq */
	if(o->p.offset != 0) { st[n][0] = 1; st[n++][1] = 1; }           /* offset */
	if(o->pt) { st[n][0] = 1; st[n++][1] = 0; }                      /* passthru */
	st[n][0] = 1; st[n++][1] = 0;                                    /* output */
	for(i = 0; i < n; i++) total += st[i][0] - (i == 0 || st[i][1] || st[i - 1][1] ? 0 : 1);
	return(total);
}

/* SECAM on raster line L of the stream (the two fill buffers in front of it are -2 and -1): L is what places it in the
 * reference's ring of line buffers, whose padding it reads and adds to */
static void secam_line(orc_t *o, int16_t *l, int64_t L, int frame, int line)
{
	const int W = o->width;
	const char *seq = line_code(o->p.type, line);
	int vy = source_row(o, line);
	int16_t *cb = o->chroma;
	int16_t *pad = o->secam_pad[((L % o->olines) + o->olines) % o->olines];
	int sl = 0, sr = 0, x;
	int dr = ((frame * o->p.lines) + line) & 1;

	if(line == 1 || line == o->p.hline) memset(cb, 0, sizeof(int16_t) * 2 * W);

	if(seq[2] == 'a' || seq[3] == 'a')
	{
		const uint32_t *fb = frame_for(o, frame);
		const uint32_t *row = (fb && vy >= 0) ? fb + (size_t) vy * o->active_width : NULL;
		int16_t yuv[3], black[3];
		int cur = dr ? 2 : 1, other = dr ? 1 : 2;

		orc_yuv(o, 0x000000, black);

		for(x = 0; x < o->active_left; x++) cb[x] = black[cur];
		for(; x < o->active_left + o->active_width; x++)
		{
			orc_yuv(o, row ? (row[x - o->active_left] & 0xFFFFFF) : 0x000000, yuv);
			cb[x] = (yuv[cur] + cb[W + x]) / 2;
			cb[W + x] = yuv[other];
		}
		for(; x < W; x++) cb[x] = black[cur];

		sl = o->burst_left;
		sr = seq[3] == 'a' ? sl + o->burst_width : o->half_width;
	}

	if(sr > sl)
	{
		int16_t dmin, dmax;

		/* luma notch over the active region, in place, step 1 here (I only); past the line it reads the padding */
		if(o->ref_heap) for(x = 0; x < 8; x++) l[W + x] = pad[x];
		fir_block(o->secam_notch, 51, l + o->active_left, l + o->active_left, o->active_width, 1);
		for(x = 0; x < 8; x++) l[W + x] = 0;
		fir_block(o->secam_lpf, 15, cb, cb, W, 1);

		/* ref fir.c:721-735 - double IIR, state carried across processed lines */
		for(x = 0; x < W; x++)
		{
			double in = (double) cb[x];
			double v;
			o->iir_iy = in * o->iir_b[0] + o->iir_ix * o->iir_b[1] - o->iir_iy * o->iir_a[1];
			o->iir_ix = in;
			v = o->iir_iy < I16MIN ? I16MIN : (o->iir_iy > I16MAX ? I16MAX : o->iir_iy);
			cb[x] = lround(v);
		}

		o->fm_secam.counter = I16MAX;
		o->fm_secam.phase.i = ((frame * o->p.lines) + line) % 3 == 0 ? I32MAX : -I32MAX;
		o->fm_secam.phase.q = 0;

		dmin = o->secam_dmin[dr];
		dmax = o->secam_dmax[dr];

		for(x = sl; x < sr; x++)
		{
			const c16_t *g;
			if(cb[x] < dmin) cb[x] = dmin;
			else if(cb[x] > dmax) cb[x] = dmax;
			g = &o->secam_bell[(uint16_t) cb[x]];
			fm_cgain(&o->fm_secam, &cb[x], cb[x], g);
			/* x can reach W, W+1 (burst window 82+944 > 1024): the reference
			 * then writes into the line buffer's padding (video.c:3228) */
			if(x < W) l[x] += (cb[x] * o->burst_win[x - o->burst_left]) >> 15;
			else if(x < W + 8) pad[x - W] += (cb[x] * o->burst_win[x - o->burst_left]) >> 15;
		}
	}
}

/* ------------------------------------------------------------------------ */
/* Audio: ref video.c:3261-3450                                             */
/* ------------------------------------------------------------------------ */

static void audio_line(orc_t *o, int16_t *iq /* interleaved, W samples */)
{
	int x;

	for(x = 0; x < o->swidth; x++)
	{
		int16_t add[2] = { 0, 0 };

		o->interp += 32000;
		if(o->interp >= o->srate)
		{
			int i;
			o->interp -= o->srate;

			if(o->pcm && o->pcm_pairs)
			{
				for(i = 0; i < 2; i++)
				{
					int32_t v = ((int32_t) o->pcm[o->pcm_pos * 2 + i] * o->p.volume + 128) >> 8;
					o->audio_lr[i] = sat16(v);
				}
				if(++o->pcm_pos == o->pcm_pairs) o->pcm_pos = 0;
			}
			else
			{
				o->audio_lr[0] = o->audio_lr[1] = 0;
			}

			if(o->have_am) o->am_mono.sample = (o->audio_lr[0] + o->audio_lr[1]) / 2;

			if(o->have_fm)
			{
				o->fm_mono.sample = (o->audio_lr[0] + o->audio_lr[1]) / 2;
				if(o->have_lim) o->fm_mono.sample = limiter_step(&o->lim, o->fm_mono.sample);
			}

			if(o->have_nicam)
			{
				o->nicam_buf[o->nicam_buf_len++] = o->audio_lr[0];
				o->nicam_buf[o->nicam_buf_len++] = o->audio_lr[1];
				if(o->nicam_buf_len == 64)
				{
					memcpy(o->nicam.audio, o->nicam_buf, sizeof(int16_t) * 64);
					o->nicam_buf_len = 0;
				}
			}
		}

		if(o->have_fm) fm_add(&o->fm_mono, add, o->fm_mono.sample);
		if(o->have_am) am_add(&o->am_mono, add, o->am_mono.sample);

		iq[x * 2 + 0] += add[0];
		iq[x * 2 + 1] += add[1];
	}

	if(o->have_nicam) nicam_output(&o->nicam, iq, o->swidth);
}

/* ref video.c:3482-3515 */
static void offset_line(orc_t *o, int16_t *iq)
{
	int x;
	for(x = 0; x < o->swidth; x++)
	{
		int32_t ai = iq[x * 2 + 0], aq = iq[x * 2 + 1], bi, bq;
		c32_mul(&o->off_phase, &o->off_phase, &o->off_delta);
		bi = o->off_phase.i >> 16;
		bq = o->off_phase.q >> 16;
		iq[x * 2 + 0] = (int16_t) ((ai * bi - aq * bq) >> 15);
		iq[x * 2 + 1] = (int16_t) ((ai * bq + aq * bi) >> 15);
		nco_renorm(&o->off_phase, &o->off_counter);
	}
}

/* ------------------------------------------------------------------------ */
/* Open: ref video.c:3812-4704                                              */
/* ------------------------------------------------------------------------ */

size_t orc_params_size(void) { return(sizeof(orc_params_t)); }

orc_t *orc_open(const orc_params_t *params, unsigned int sample_rate)
{
	return(orc_open2(params, sample_rate, 0));
}

/* vid_init with a pixel rate (ref video.c:3812, 3839): the raster is built at pixel_rate and a
 * polyphase FIR (ref _init_vresampler video.c:3627-3651, fir_int16_resampler_init fir.c:393-428)
 * brings it to sample_rate in front of the video filter. Only rate pairs that give every line the
 * same number of output samples are restated (the reference lets the line width vary otherwise);
 * FM video is not. */
orc_t *orc_open2(const orc_params_t *params, unsigned int sample_rate, unsigned int pixel_rate)
{
	orc_t *o = calloc(1, sizeof(orc_t));
	orc_params_t *p;
	double width, d;
	int i, c;

	if(!o) return(NULL);
	o->p = *params;
	p = &o->p;
	o->rate = pixel_rate ? pixel_rate : sample_rate;
	o->srate = sample_rate;

	if(p->type != ORC_RASTER_625 && p->type != ORC_RASTER_525) { free(o); return(NULL); }
	if(p->modulation == ORC_MOD_FM && p->fm_energy_dispersal != 0) { free(o); return(NULL); }

	/* video.c:3832-3837 defaults */
	if(p->hline <= 0 && p->interlaced != 0) p->hline = (p->lines + 1) / 2;
	if(p->gamma <= 0) p->gamma = 1.0;
	if(p->rw_co <= 0) p->rw_co = 0.299;
	if(p->gw_co <= 0) p->gw_co = 0.587;
	if(p->bw_co <= 0) p->bw_co = 0.114;

	o->complex = p->output_type == ORC_OUT_COMPLEX;

	/* video.c:3844-3853 */
	width = (double) p->frame_rate_den / p->frame_rate_num / p->lines;
	o->width = round((double) o->rate * width);
	o->half_width = round((double) o->rate * width / 2);
	o->active_left = round(o->rate * p->active_left);
	o->active_width = ceil(o->rate * p->active_width);
	if(o->active_width > o->width) o->active_width = o->width;
	o->swidth = o->width;
	if(o->srate != o->rate)
	{
		/* fir.c:393-428: r = out / in = I / D, (21 I) | 1 taps of a Kaiser low-pass at rate I, gain I;
		 * fir.c:263-295: ataps = ceil(ntaps / I) taps per phase, phase p column c = tap[ntaps - I + p - c I] */
		int64_t g = gcd64(o->srate, o->rate);
		int ntaps, ph, col;
		double *taps;
		o->rs_I = (int) (o->srate / g);
		o->rs_D = (int) (o->rate / g);
		o->swidth = round((double) o->srate * width);
		if(p->modulation == ORC_MOD_FM || ((int64_t) o->width * o->rs_I) % o->rs_D != 0 ||
		   (int64_t) o->width * o->rs_I / o->rs_D != o->swidth) { free(o); return(NULL); }
		ntaps = (21 * o->rs_I) | 1;
		taps = calloc(ntaps, sizeof(double));
		if(o->rs_I > o->rs_D) design_low_pass(taps, ntaps, o->rs_I, 0.45, o->rs_I);
		else design_low_pass(taps, ntaps, o->rs_I, 0.45 * o->rs_I / o->rs_D, o->rs_I);
		o->rs_ataps = (ntaps + o->rs_I - 1) / o->rs_I;
		o->rs_taps = calloc((size_t) o->rs_I * o->rs_ataps, sizeof(int16_t));
		for(ph = 0; ph < o->rs_I; ph++) for(col = 0; col < o->rs_ataps; col++)
		{
			int idx = ntaps - o->rs_I + ph - col * o->rs_I;
			if(idx >= 0 && idx < ntaps) o->rs_taps[ph * o->rs_ataps + col] = lround(taps[idx] * 32767.0);
		}
		free(taps);
		for(i = 0; i < 4; i++) o->rring[i] = calloc(o->swidth + 64, sizeof(int16_t));
		o->rs_on = 1;
	}

	/* video.c:3855-3881 */
	o->slevel = p->modulation == ORC_MOD_FM ? 1.0 : p->level;
	o->vlevel = p->video_level * o->slevel;

	if(p->invert_video)
	{
		double t = p->white_level;
		p->white_level = p->sync_level;
		p->sync_level = t;
		p->blanking_level = p->sync_level - (p->blanking_level - p->white_level);
		p->black_level = p->sync_level - (p->black_level - p->white_level);
	}

	o->white = round(p->white_level    * o->vlevel * I16MAX);
	o->black = round(p->black_level    * o->vlevel * I16MAX);
	o->blank = round(p->blanking_level * o->vlevel * I16MAX);
	o->sync  = round(p->sync_level     * o->vlevel * I16MAX);

	/* video.c:3883-3891; the level is truncated to int at the call (vbidata.c:62) */
	d = (p->sync_level - p->blanking_level) * o->vlevel * I16MAX;
	{
		const double sy[5][2] = {
			{ 0,         p->hsync_width },
			{ 0,         p->vsync_short_width },
			{ 0,         p->vsync_long_width },
			{ width / 2, p->vsync_short_width },
			{ width / 2, p->vsync_long_width },
		};
		for(i = 0; i < 5; i++)
		{
			make_pulse(&o->syncs[i], sy[i][0] * o->rate, sy[i][1] * o->rate, p->sync_rise * IRT1090 * o->rate, (int) d);
		}
	}

	for(c = 0; c < 256; c++) o->glut[c] = pow((double) c / 255, 1 / p->gamma);

	o->chroma = calloc(2 * o->width + 64, sizeof(int16_t));

	if(p->colour_mode == ORC_COLOUR_PAL || p->colour_mode == ORC_COLOUR_NTSC)
	{
		/* video.c:3961-3987: a = pixel_rate / colour_carrier, normalised */
		int64_t num = (int64_t) o->rate * p->colour_carrier_den;
		int64_t den = p->colour_carrier_num;
		int64_t e = gcd64(num, den);
		unsigned int n;
		num /= e; den /= e;
		o->clut_width = num;
		d = 2.0 * M_PI * ((double) den / num);
		o->clut = malloc(((size_t) o->clut_width + o->width) * sizeof(c16_t));
		for(n = 0; n < o->clut_width + o->width; n++)
		{
			o->clut[n].i = round(cos(d * n) * I16MAX);
			o->clut[n].q = round(sin(d * n) * I16MAX);
		}

		if(p->colour_bw > 0)
		{
			double *taps;
			o->chroma_ntaps = gaussian_ntaps(o->rate, p->colour_bw);
			taps = malloc(sizeof(double) * o->chroma_ntaps);
			design_gaussian(taps, o->chroma_ntaps, o->rate, p->colour_bw, 1);
			o->chroma_taps = quantise_taps(taps, o->chroma_ntaps, 1);
			free(taps);
		}
	}

	if(p->burst_level > 0)
	{
		/* video.c:4017-4048, 2194-2214 */
		double rise = p->burst_rise * IRT1090;
		double lvl = p->burst_level * (p->white_level - p->blanking_level) / 2 * o->vlevel;
		o->burst_left = round(o->rate * (p->burst_left - p->burst_rise / 2));
		o->burst_width = ceil(o->rate * (p->burst_width + rise));
		o->burst_win = malloc(sizeof(int16_t) * o->burst_width);
		for(i = 0; i < o->burst_width; i++)
		{
			double t = 1.0 / o->rate * i;
			o->burst_win[i] = round(rc_window(t, rise / 2, p->burst_width, rise) * lvl * I16MAX);
		}
		if(p->colour_mode == ORC_COLOUR_PAL)
		{
			double ph = 135.0 * (M_PI / 180.0);
			o->burst_phase.i = round(cos(ph) * I16MAX);
			o->burst_phase.q = round(sin(ph) * I16MAX);
		}
		else if(p->colour_mode == ORC_COLOUR_NTSC)
		{
			o->burst_phase.i = -I16MAX;
			o->burst_phase.q = 0;
		}
	}

	if(p->colour_mode == ORC_COLOUR_SECAM)
	{
		/* video.c:4075-4162 */
		double secam_level = (p->white_level - p->blanking_level) * o->vlevel;
		double taps[51];
		double rise = p->burst_rise * IRT1090;
		double a;
		int r;

		fm_init(&o->fm_secam, o->rate, SECAM_FM_FREQ, SECAM_FM_DEV, secam_level);
		o->iir_a[0] = 1.0; o->iir_a[1] = -0.90456054;
		o->iir_b[0] = 2.90456054; o->iir_b[1] = -2.80912108;
		o->iir_ix = o->iir_iy = 0;

		design_low_pass(taps, 15, o->rate, 1.70e6, 1.0);
		o->secam_lpf = quantise_taps(taps, 15, 1);

		design_band_reject(taps, 51, o->rate, SECAM_FM_FREQ - 1e6, SECAM_FM_FREQ + 1e6, 1.0);
		taps[51 / 2] += 0.5;
		for(a = i = 0; i < 51; i++) a += taps[i];   /* fir_normalise, fir.c:71-87 */
		a = a / 1.0;
		for(i = 0; i < 51; i++) taps[i] /= a;
		o->secam_notch = quantise_taps(taps, 51, 1);

		o->secam_dmin[0] = lround((SECAM_CB_FREQ - SECAM_FM_FREQ - 350e3) / SECAM_FM_DEV * I16MAX);
		o->secam_dmax[0] = lround((SECAM_CB_FREQ - SECAM_FM_FREQ + 506e3) / SECAM_FM_DEV * I16MAX);
		o->secam_dmin[1] = lround((SECAM_CR_FREQ - SECAM_FM_FREQ - 506e3) / SECAM_FM_DEV * I16MAX);
		o->secam_dmax[1] = lround((SECAM_CR_FREQ - SECAM_FM_FREQ + 350e3) / SECAM_FM_DEV * I16MAX);

		o->secam_bell = malloc(sizeof(c16_t) * 65536);
		for(r = I16MIN; r <= I16MAX; r++)
		{
			/* video.c:2172-2185 _secam_g */
			const double f0 = 4.286e6;
			double f = SECAM_FM_FREQ + (double) r * SECAM_FM_DEV / I16MAX;
			double lq, rq, dd;
			f = f / f0 - f0 / f;
			lq = 16.0 * f;
			rq = 1.26 * f;
			dd = 1.0 + rq * rq;
			o->secam_bell[(uint16_t) r].i = lround(0.115 * (1.0 + lq * rq) / dd * I16MAX);
			o->secam_bell[(uint16_t) r].q = lround(0.115 * (lq - rq) / dd * I16MAX);
		}

		o->burst_left = round(o->rate * (p->burst_left - p->burst_rise / 2));
		o->burst_width = ceil(o->rate * (p->burst_width + rise));
		o->burst_win = malloc(sizeof(int16_t) * o->burst_width);
		for(i = 0; i < o->burst_width; i++)
		{
			double t = 1.0 / o->rate * i;
			o->burst_win[i] = round(rc_window(t, rise / 2, p->burst_width, rise) * 1.0 * I16MAX);
		}
	}

	if(p->vfilter)
	{
		/* video.c:3653-3764 */
		if(p->modulation == ORC_MOD_VSB)
		{
			double taps[51 * 2];
			design_complex_band_pass(taps, 51, o->srate, -p->vsb_lower_bw, p->vsb_upper_bw, 1);
			o->vf_type = 3;
			o->vf_ntaps = 51;
			o->vf_itaps = quantise_taps(taps + 0, 51, 2);
			o->vf_qtaps = quantise_taps(taps + 1, 51, 2);
		}
		else if(p->modulation == ORC_MOD_FM)
		{
			/* video.c:3678-3740: a fixed pre-emphasis table per line standard and sample rate */
			const double *taps;
			int ntaps;
			#define FMT(t) do { taps = t; ntaps = sizeof(t) / sizeof(double); } while(0)
			if(p->lines == 525)
			{
				if(o->srate == 18000000) FMT(orc_fm_525_18_taps);
				else FMT(orc_fm_525_2025_taps);
			}
			else
			{
				if(o->srate == 14000000) FMT(orc_fm_625_14_taps);
				else if(o->srate == 20000000) FMT(orc_fm_625_20_taps);
				else if(o->srate == 28000000) FMT(orc_fm_625_28_taps);
				else FMT(orc_fm_625_2025_taps);
			}
			#undef FMT
			o->vf_type = 1;
			o->vf_ntaps = ntaps;
			o->vf_itaps = quantise_taps(taps, ntaps, 1);
		}
		else
		{
			double taps[51];
			design_low_pass(taps, 51, o->srate, p->video_bw, 1);
			o->vf_type = 1;
			o->vf_ntaps = 51;
			o->vf_itaps = quantise_taps(taps, 51, 1);
		}
	}

	/* audio: video.c:4404-4558 */
	if(p->fm_mono_level > 0 && p->fm_mono_carrier != 0)
	{
		o->have_fm = 1;
		fm_init(&o->fm_mono, o->srate, p->fm_mono_carrier, p->fm_mono_deviation, p->fm_mono_level * o->slevel);
		if(p->fm_mono_preemph)
		{
			const double *t = p->fm_mono_preemph == ORC_PREEMPH_50US ? fm_audio_50us_taps :
			                  p->fm_mono_preemph == ORC_PREEMPH_75US ? fm_audio_75us_taps : fm_audio_j17_taps;
			limiter_init(&o->lim, I16MAX, 21, t, fm_audio_flat_taps, 65);
			o->have_lim = 1;
		}
	}
	if(p->nicam_level > 0 && p->nicam_carrier != 0)
	{
		o->have_nicam = 1;
		nicam_init(&o->nicam, o->srate, (unsigned int) p->nicam_carrier, p->nicam_beta, p->nicam_level * o->slevel);
	}
	if(p->am_audio_level > 0 && p->am_mono_carrier != 0)
	{
		o->have_am = 1;
		am_init(&o->am_mono, o->srate, p->am_mono_carrier, p->am_audio_level * o->slevel);
	}

	if(p->modulation == ORC_MOD_FM)
	{
		/* video.c:4564-4585 */
		o->have_fmv = 1;
		fm_init(&o->fm_video, o->srate, 0, p->fm_deviation, p->fm_level * p->level);
	}

	if(p->offset != 0)
	{
		/* video.c:4592-4605 - note phase.i starts at INT16_MAX, as the reference does */
		o->off_counter = I16MAX;
		o->off_phase.i = I16MAX;
		o->off_phase.q = 0;
		d = 2.0 * M_PI / o->srate * p->offset;
		o->off_delta.i = lround(cos(d) * I32MAX);
		o->off_delta.q = lround(sin(d) * I32MAX);
	}

	/* the filter stage's delay is (ntaps / 2 + W - 1) / W lines (ref video.c:3759) and the render here assumes one: two
	 * lines below W = ntaps / 2 (25 at 51 taps). At W = ntaps / 2 the delay is one line, but the stream still differs from
	 * the reference's (51 taps, W = 25: not restated), so the refusal starts there. */
	if(o->vf_type && o->swidth <= o->vf_ntaps / 2)
	{
		orc_close(o);
		return(NULL);
	}

	for(i = 0; i < ORC_RING; i++)
	{
		o->ring[i] = calloc((o->swidth > o->width ? o->swidth : o->width) + 64, sizeof(int16_t));
		blank_line(o, o->ring[i]);
	}

	return(o);
}

void orc_close(orc_t *o)
{
	int i;
	if(!o) return;
	for(i = 0; i < 5; i++) free(o->syncs[i].value);
	for(i = 0; i < ORC_RING; i++) free(o->ring[i]);
	for(i = 0; i < 4; i++) free(o->rring[i]);
	free(o->rs_taps);
	free(o->clut); free(o->chroma); free(o->chroma_taps); free(o->burst_win);
	free(o->fm_secam.lut); free(o->secam_lpf); free(o->secam_notch); free(o->secam_bell);
	free(o->vf_itaps); free(o->vf_qtaps);
	free(o->fm_mono.lut);
	if(o->have_lim)
	{
		free(o->lim.vfir.taps); free(o->lim.vfir.win); free(o->lim.ffir.taps); free(o->lim.ffir.win);
		free(o->lim.shape); free(o->lim.att); free(o->lim.fix); free(o->lim.var);
	}
	free(o->nicam.taps); free(o->nicam.bb); free(o->nicam.cc);
	free(o->tbl);
	free(o);
}

void orc_set_ref_heap(orc_t *o, int on) { o->ref_heap = on && !o->rs_on; }
void orc_set_frames(orc_t *o, const uint32_t *rgb, int nframes) { o->frames = rgb; o->nframes = nframes; }
void orc_add_vbi_line(orc_t *o, int line, int replace_from, int replace_to, int replace_value, const int16_t *add)
{
	if(o->nvbi >= 64) return;
	o->vbi[o->nvbi].line = line; o->vbi[o->nvbi].from = replace_from; o->vbi[o->nvbi].to = replace_to;
	o->vbi[o->nvbi].value = replace_value; o->vbi[o->nvbi].add = add;
	o->nvbi++;
}

void orc_set_passthru(orc_t *o, const int16_t *iq, size_t ncomplex) { o->pt = iq; o->pt_len = ncomplex; o->pt_pos = 0; }
void orc_set_audio(orc_t *o, const int16_t *pcm, size_t npairs) { o->pcm = pcm; o->pcm_pairs = npairs; o->pcm_pos = 0; }

int orc_width(const orc_t *o) { return(o->swidth); }
int orc_raster_width(const orc_t *o) { return(o->width); }
int orc_active_width(const orc_t *o) { return(o->active_width); }
int orc_active_lines(const orc_t *o) { return(o->p.active_lines); }
int orc_is_complex(const orc_t *o) { return(o->complex); }

/* ------------------------------------------------------------------------ */
/* Render: the flattened vid_next_line loop                                 */
/* ------------------------------------------------------------------------ */

/* ref _vid_filter_process video.c:3235-3248 feeding fir_int16_process fir.c:304-355 with the
 * resampler's taps, in closed form of the global output index j: the newest input consumed is
 * i = floor(j D / I), the phase (j D) mod I, the window the rs_ataps inputs ending at i (zero
 * before the stream). Line L of the resampled stream needs raster lines L - 1 and L final. */
static void resample_line(orc_t *o, int64_t L)
{
	const int Wp = o->width, Ws = o->swidth, I = o->rs_I, D = o->rs_D, A = o->rs_ataps;
	int16_t *dst = o->rring[((L % 4) + 4) % 4];
	int k, c;
	for(k = 0; k < Ws; k++)
	{
		const int64_t j = L * Ws + k;
		const int64_t in = (j * D) / I;
		const int16_t *t = o->rs_taps + ((j * D) % I) * A;
		int32_t a = 0;
		for(c = 0; c < A; c++)
		{
			const int64_t n = in - A + 1 + c;
			if(n >= 0) a += ring_line(o, n / Wp)[n % Wp] * t[c];
		}
		dst[k] = sat16(a >> 15);
	}
}

size_t orc_render(orc_t *o, int nlines, int16_t *out)
{
	const int W = o->swidth;
	int16_t *iq = malloc(sizeof(int16_t) * 2 * W);
	size_t n = 0;
	int k, x, y;

	if(o->next_emit == 0 && o->next_raster == 0)
	{
		/* Pipeline fill, as the reference's threaded stages see it:
		 * - the SECAM stage runs on two fill buffers (line 0 of frame 1, an
		 *   all-black active line) before line 1 arrives (video.c:4665-4667,
		 *   window layout 4675-4688), pre-warming its IIR;
		 * - with a video filter the first filtered line lands in a fill buffer
		 *   whose width becomes W, so audio (and the offset mixer) consume one
		 *   full line of state before the first emitted sample (video.c:3244,
		 *   3268; SURVEY.md §9 V2). */
		if(o->p.colour_mode == ORC_COLOUR_SECAM)
		{
			int16_t *fill = calloc((o->swidth > o->width ? o->swidth : o->width) + 64, sizeof(int16_t));
			o->olines = ref_olines(o);
			for(k = 0; k < 2; k++)
			{
				blank_line(o, fill);
				secam_line(o, fill, k - 2, 1, 0);
			}
			free(fill);
		}
		if(o->rs_on)
		{
			/* the resampler is one more two-line stage: its first output line lands in a fill
			 * buffer too (width W from then on), so everything behind it runs one line earlier
			 * still - the sound carriers, the offset mixer and the passthru stream */
			memset(iq, 0, sizeof(int16_t) * 2 * W);
			audio_line(o, iq);
			if(o->p.offset != 0) offset_line(o, iq);
		}
		if(o->vf_type)
		{
			memset(iq, 0, sizeof(int16_t) * 2 * W);
			if(o->have_fmv)
			{
				/* the FM modulator integrates what is IN the fill line: the filter's output for
				 * the line before the stream - zero history, with the first samples of line 1
				 * reaching in through the taps ahead of centre */
				int h = o->vf_ntaps / 2;
				const int16_t *first;
				while(o->next_raster <= 1) raster_line(o, o->next_raster++);
				first = ring_line(o, 0);
				for(x = W - h; x < W; x++)
				{
					int32_t a = 0;
					for(y = 0; y < o->vf_ntaps; y++)
					{
						int j = x - h + y - W;             /* position in line 1 */
						if(j >= 0) a += first[j] * o->vf_itaps[y];
					}
					iq[x * 2] = sat16(a >> 15);
				}
			}
			audio_line(o, iq);
			if(o->have_fmv) fmv_line(&o->fm_video, iq, W);
			if(o->p.offset != 0) offset_line(o, iq);
			/* ... and the passthru stage spends its first line on that buffer too */
			if(o->pt) o->pt_pos = o->pt_len < (size_t) W ? o->pt_len : (size_t) W;
		}
		if(o->rs_on && o->pt)
		{
			size_t skip = (size_t) W * (o->vf_type ? 2 : 1);
			o->pt_pos = o->pt_len < skip ? o->pt_len : skip;
		}
	}

	for(k = 0; k < nlines; k++)
	{
		int64_t t = o->next_emit;
		int16_t *prev, *cur, *next;

		if(o->rs_on)
		{
			/* The emitted line t is line t + 1 of the resampled stream (the stage writes into
			 * the buffer one line back and, unlike the video filter, pads no delay), filtered
			 * across lines t and t + 2 of it. Raster lines are final once the next one is
			 * rastered (sync back-spill), SECAM and the VBI overlays have run on them. */
			while(o->next_resamp <= t + 2)
			{
				int64_t L = o->next_resamp;
				while(o->next_raster <= L + 1) raster_line(o, o->next_raster++);
				if(o->p.colour_mode == ORC_COLOUR_SECAM)
				{
					while(o->next_secam <= L)
					{
						int64_t M = o->next_secam++;
						secam_line(o, ring_line(o, M), M, M / o->p.lines + 1, M % o->p.lines + 1);
					}
				}
				if(o->nvbi) vbi_line(o, L);
				resample_line(o, L);
				o->next_resamp++;
			}
			prev = o->rring[t % 4];
			cur  = o->rring[(t + 1) % 4];
			next = o->rring[(t + 2) % 4];
		}
		else
		{
		/* raster through t+1 (sync back-spill, filter look-ahead) */
		while(o->next_raster <= t + 1) raster_line(o, o->next_raster++);

		/* SECAM sees a line only after the following line's raster. It runs ahead of the video filter in the
		 * reference's pipeline, so the filter's taps ahead of centre find line t + 1 with its subcarrier: below about
		 * 5 Msps the burst window starts within them (20 < 25 samples at 4 Msps). */
		if(o->p.colour_mode == ORC_COLOUR_SECAM)
		{
			while(o->next_raster <= t + 2) raster_line(o, o->next_raster++);
			while(o->next_secam <= t + 1)
			{
				int64_t L = o->next_secam++;
				secam_line(o, ring_line(o, L), L, L / o->p.lines + 1, L % o->p.lines + 1);
			}
		}

		if(o->nvbi) vbi_line(o, t);

		prev = ring_line(o, t - 1);
		cur  = ring_line(o, t);
		next = ring_line(o, t + 1);
		}

		if(o->vf_type)
		{
			/* video.c:3235-3248 + fir.c:304-355/564-615 as a centred FIR over
			 * the stream; samples before the first are zero (calloc'd window) */
			int h = o->vf_ntaps / 2;
			int32_t *win = malloc(sizeof(int32_t) * (W + 2 * h));
			for(x = 0; x < h; x++) win[x] = (t == 0 && !o->rs_on) ? 0 : prev[W - h + x];
			for(x = 0; x < W; x++) win[h + x] = cur[x];
			for(x = 0; x < h; x++) win[h + W + x] = next[x];
			for(x = 0; x < W; x++)
			{
				int32_t ai = 0, aq = 0;
				const int32_t *w = win + x;
				for(y = 0; y < o->vf_ntaps; y++) ai += w[y] * o->vf_itaps[y];
				if(o->vf_qtaps) for(y = 0; y < o->vf_ntaps; y++) aq += w[y] * o->vf_qtaps[y];
				iq[x * 2 + 0] = sat16(ai >> 15);
				iq[x * 2 + 1] = o->vf_qtaps ? sat16(aq >> 15) : 0;
			}
			free(win);
		}
		else
		{
			for(x = 0; x < W; x++)
			{
				iq[x * 2 + 0] = cur[x];
				iq[x * 2 + 1] = 0;
			}
		}

		if(o->have_fm || o->have_am || o->have_nicam) audio_line(o, iq);

		if(o->have_fmv) fmv_line(&o->fm_video, iq, W);

		if(o->p.swap_iq)
		{
			for(x = 0; x < W; x++)
			{
				int16_t tt = iq[x * 2 + 0];
				iq[x * 2 + 0] = iq[x * 2 + 1];
				iq[x * 2 + 1] = tt;
			}
		}

		if(o->p.offset != 0) offset_line(o, iq);

		/* ref _vid_passthru_process video.c:3517-3541: the last stage before the sink adds
		 * the external stream line by line, int16 wrap, whole lines only */
		if(o->pt && o->pt_pos + (size_t) W <= o->pt_len)
		{
			const int16_t *pl = o->pt + o->pt_pos * 2;
			for(x = 0; x < W * 2; x++) iq[x] = (int16_t) (iq[x] + pl[x]);
			o->pt_pos += W;
		}

		if(o->complex)
		{
			memcpy(out + n, iq, sizeof(int16_t) * 2 * W);
			n += 2 * W;
		}
		else
		{
			for(x = 0; x < W; x++) out[n++] = iq[x * 2];
		}

		o->next_emit++;
	}

	free(iq);
	return(n);
}

/* ------------------------------------------------------------------------ */
/* Table access for unit tests                                              */
/* ------------------------------------------------------------------------ */

static const int32_t *tbl16(orc_t *o, const int16_t *v, int n, int *count)
{
	int i;
	free(o->tbl);
	o->tbl = malloc(sizeof(int32_t) * (n > 0 ? n : 1));
	for(i = 0; i < n; i++) o->tbl[i] = v[i];
	*count = n;
	return(o->tbl);
}

const int32_t *orc_table(orc_t *o, const char *name, int *count)
{
	int16_t tmp[8];
	*count = 0;
	if(strncmp(name, "sync", 4) == 0 && name[4] >= '0' && name[4] <= '4' && name[5] == 0)
	{
		const pulse_t *pl = &o->syncs[name[4] - '0'];
		return(tbl16(o, pl->value, pl->length, count));
	}
	if(strcmp(name, "sync_off") == 0)
	{
		int i;
		for(i = 0; i < 5; i++) tmp[i] = o->syncs[i].offset;
		return(tbl16(o, tmp, 5, count));
	}
	if(strcmp(name, "rs_taps") == 0 && o->rs_on) return(tbl16(o, o->rs_taps, o->rs_I * o->rs_ataps, count));
	if(strcmp(name, "rs_geometry") == 0 && o->rs_on)
	{
		tmp[0] = o->rs_I; tmp[1] = o->rs_D; tmp[2] = o->rs_ataps; tmp[3] = o->width;
		return(tbl16(o, tmp, 4, count));
	}
	if(strcmp(name, "burst_win") == 0 && o->burst_win) return(tbl16(o, o->burst_win, o->burst_width, count));
	if(strcmp(name, "chroma_taps") == 0 && o->chroma_taps) return(tbl16(o, o->chroma_taps, o->chroma_ntaps, count));
	if(strcmp(name, "vsb_itaps") == 0 && o->vf_itaps) return(tbl16(o, o->vf_itaps, o->vf_ntaps, count));
	if(strcmp(name, "vsb_qtaps") == 0 && o->vf_qtaps) return(tbl16(o, o->vf_qtaps, o->vf_ntaps, count));
	if(strcmp(name, "nicam_taps") == 0 && o->have_nicam) return(tbl16(o, o->nicam.taps, o->nicam.ntaps, count));
	if(strcmp(name, "secam_lpf") == 0 && o->secam_lpf) return(tbl16(o, o->secam_lpf, 15, count));
	if(strcmp(name, "secam_notch") == 0 && o->secam_notch) return(tbl16(o, o->secam_notch, 51, count));
	if(strcmp(name, "levels") == 0)
	{
		tmp[0] = o->white; tmp[1] = o->black; tmp[2] = o->blank; tmp[3] = o->sync;
		return(tbl16(o, tmp, 4, count));
	}
	if(strcmp(name, "geometry") == 0)
	{
		tmp[0] = o->width; tmp[1] = o->half_width; tmp[2] = o->active_left;
		tmp[3] = o->active_width; tmp[4] = o->burst_left; tmp[5] = o->burst_width;
		return(tbl16(o, tmp, 6, count));
	}
	return(NULL);
}

/* ------------------------------------------------------------------------ */
/* Built-in test source: ref av_test.c:71-205                               */
/* ------------------------------------------------------------------------ */

void orc_test_pattern(int width, int height, uint32_t *video)
{
	static const uint32_t bars[8] = {
		0x000000, 0x0000BF, 0xBF0000, 0xBF00BF, 0x00BF00, 0x00BFBF, 0xBFBF00, 0xFFFFFF,
	};
	static const char *logo =
		"                                                "
		" ##  ##    ##     ####   ##  ##  ######  ##  ## "
		" ##  ##   ####   ##  ##  ## ##     ##    ##  ## "
		" ##  ##  ##  ##  ##      ####      ##    ##  ## "
		" ######  ######  ##      ###       ##    ##  ## "
		" ##  ##  ##  ##  ##      ####      ##    ##  ## "
		" ##  ##  ##  ##  ##  ##  ## ##     ##     ####  "
		" ##  ##  ##  ##   ####   ##  ##    ##      ##   "
		"                                                ";
	int c, x, y;

	for(y = 0; y < height; y++)
	{
		for(x = 0; x < width; x++)
		{
			if(y < height - 140) c = bars[7 - x * 8 / width];
			else if(y < height - 120) c = 0xBF0000;
			else if(y < height - 100)
			{
				c = x * 0xFF / (width - 1);
				c = c << 16 | c << 8 | c;
			}
			else
			{
				c = x * 0xFF / (width - 1);
				c &= 0xE0;
				c = c | (c >> 3) | (c >> 6);
				c = c << 16 | c << 8 | c;
			}
			video[y * width + x] = c;
		}
	}

	if(width >= 48 * 4 && height >= 9 * 4)
	{
		for(x = 0; x < 48 * 4; x++)
		{
			for(y = 0; y < 9 * 4; y++)
			{
				c = logo[y / 4 * 48 + x / 4] == ' ' ? 0x000000 : 0xFFFFFF;
				video[(height / 10 + y) * width + ((width - 48 * 4) / 2) + x] = c;
			}
		}
	}
}

size_t orc_test_tone_pairs(void) { return(32000 * 64 / 100 * 10); }

void orc_test_tone(int16_t *audio)
{
	double d = 1000.0 * 2 * M_PI * 1 / 32000;
	int y = 32000 / 1 * 64 / 100;
	int n = y * 10, x;

	for(x = 0; x < n; x++)
	{
		int16_t l = sin(x * d) * I16MAX * 0.1;
		if(x < y) { audio[x * 2 + 0] = 0; audio[x * 2 + 1] = l; }
		else if(x >= y * 2 && x < y * 3) { audio[x * 2 + 0] = l; audio[x * 2 + 1] = 0; }
		else if(x >= y * 4 && x < y * 5) { audio[x * 2 + 0] = l; audio[x * 2 + 1] = 0; }
		else { audio[x * 2 + 0] = l; audio[x * 2 + 1] = l; }
	}
}
