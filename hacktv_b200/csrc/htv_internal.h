/* hacktv_b200 internal definitions shared by the C host layer and the CUDA
 * translation unit. Not part of the public C-ABI (include/hacktv_b200.h). */
#ifndef HTV_INTERNAL_H
#define HTV_INTERNAL_H

#include <stdint.h>
#include <stddef.h>
#include "hacktv_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int16_t i, q; } htv_c16_t;
typedef struct { int32_t i, q; } htv_c32_t;

#define HTV_VF_NTAPS   51      /* ref video.c:3671,3744 */
#define HTV_FMV_MAXTAPS 72     /* FM video pre-emphasis: 67 or 71 taps (ref video.c:2016-2099) */
#define HTV_MAX_CTAPS  31      /* chroma Gaussian LPF taps we accept (13 @16M, 15 @20M, 11 @13.5M) */
#define HTV_AUDIO_RATE 32000   /* ref hacktv.h:30 */
#define HTV_NICAM_SYMBOL_RATE 364000
#define HTV_LIM_W      21      /* limiter width, ref video.c:4447 */
#define HTV_AFIR_N     65      /* audio FIR taps, ref video.c:2118 */
#define HTV_J17_N      83      /* ref nicam728.h:48 */
#define HTV_NICAM_LUT_PAD 256   /* zero entries behind the NICAM pulse table: lanes of a partial tile index past it */

/* Line code bits (one uint16 per line number, ref video.c:2447-2810 restated as a table) */
#define HTV_LC_SYNC_MASK  0x001F   /* 5-bit pulse mask fed to the sync renderer */
#define HTV_LC_BURST_SHIFT 5       /* 0 never, 1 always, 2 even frames ('1'), 3 odd frames ('2') */
#define HTV_LC_BURST_MASK (3 << HTV_LC_BURST_SHIFT)
#define HTV_LC_LEFT_ACTIVE  (1 << 7)
#define HTV_LC_RIGHT_ACTIVE (1 << 8)

/* Everything the kernels need by value. Passed as a __grid_constant__ kernel
 * parameter (constant bank): uniform reads of taps cost no registers. */
typedef struct {
	/* geometry */
	int32_t W, half_width, lines, hline;
	int32_t active_left, active_width, active_lines;
	int32_t raster, colour_mode, complex_out, interlaced;
	int32_t blank, black_y, black_u, black_v;

	/* sync pulses: values live in tables, here only the placement */
	int32_t pulse_off[5], pulse_len[5], pulse_pos[5];

	/* RGB -> YUV (ref video.c:3912-3959), evaluated in fp64 on the device */
	double rw, gw, bw, eu, ev;
	double black_level, white_minus_black, vlevel, uv_scale;

	/* PAL/NTSC chroma */
	int32_t chroma_ntaps;
	int32_t chroma_taps[HTV_MAX_CTAPS + 1];
	int32_t burst_left, burst_width, burst_i, burst_q;
	uint32_t clut_width;

	/* video filter */
	int32_t vf_type;               /* 0 none, 1 real low-pass, 3 real->complex (VSB) */
	int32_t vf_i[HTV_VF_NTAPS], vf_q[HTV_VF_NTAPS];

	/* audio subcarriers */
	int32_t rate;
	int32_t shift;                 /* audio-clock lead over the emitted stream, in samples (W with a filter) */
	int32_t volume;
	int32_t have_fm, fm_level, have_lim;
	int32_t have_am, am_level;
	uint64_t am_ang;               /* carrier step, turns * 2^64 */
	int32_t have_nicam, nicam_ntaps, nicam_F, nicam_D, nicam_cc_len, nicam_tpad_len;
	int32_t nicam_sps, nicam_minor_short, nicam_lut_ok;
	/* S-Video: the colour subcarrier goes to Q (k_line KL_SV); in what was this block's padding word, so that no field
	 * moves */
	int32_t s_video;

	/* SECAM */
	int32_t secam_level, secam_dmin[2], secam_dmax[2], secam_pad;
	int32_t secam_lpf[15], secam_notch[51];
	double iir_a1, iir_b0, iir_b1;

	/* FM video (ref video.c:2299-2335, 3452-3464, 3678-3740): the filtered composite + sound
	 * carriers become the modulating signal of a Q31 phasor; pre-emphasis taps in application order */
	int32_t have_fmv, fmv_level, fmv_ntaps;
	/* store: HTV_TYPE_* of the output stream (htv_sample_type.h), HTV_TYPE_INT16 unless htv_set_sample_type. It sits in
	 * what was this block's padding word, so that no other field (and no kernel parameter behind dp) moves */
	int32_t sample_type;
	int32_t fmv_taps[HTV_FMV_MAXTAPS];

	/* post mixers */
	int32_t swap_iq, have_offset;
	uint64_t offset_ang;           /* turns * 2^64 per sample */
	uint64_t offset_phase0;        /* phase after the first renormalisation (see htv_tables.c) */
} htv_dparams_t;

#ifdef __CUDACC__
#define HTV_HD __host__ __device__
#else
#define HTV_HD
#endif

/* The source picture row that line `line` (1 .. lines) of a frame shows, -1 none (ref video.c:2812-2895): a progressive
 * source on an interlaced raster shifts down one row. The device's line_numbers and the host's picture-row table
 * (htv_tables.c build_pic_rows) both take it from here. */
static inline HTV_HD int htv_line_vy(const htv_dparams_t *dp, int line)
{
	int vy;
	if(dp->raster == HTV_RASTER_625) vy = line < 313 ? (line - 23) * 2 : (line - 336) * 2 + 1;
	else vy = line < 265 ? (line - 23) * 2 : (line - 286) * 2 + 1;
	if(vy >= 0 && dp->interlaced != 0) vy += 1;
	return(vy >= 0 && vy < dp->active_lines ? vy : -1);
}

/* Host-built tables (ref video.c:3812-4704, restated). All arrays are owned. */
struct htv_tables_t {
	htv_config_t conf;
	unsigned int rate;
	htv_dparams_t dp;

	uint16_t *codes;        int ncodes;           /* lines + 1 */
	int16_t *pulse_values;  int npulse_values;
	int16_t *tmpl_out, *tmpl_keep;                 /* [tmpl_rows][W] line templates: blank + sync pulses (htv_tables.c) */
	uint8_t *tmpl_keep_any; int tmpl_rows;         /* lines + 2 */
	/* rows of the converted picture store, which the fused line kernel keeps for encoders whose colour subcarrier does not
	 * repeat within 4 frames (comp_phases = 0; htv_tables.c build_pic_rows): pic_rows[row] = line (1-based, 0: no line draws
	 * the row), al, ar, keep of the line that shows it; rows 0 .. active_lines - 1 are the picture rows, the rest the
	 * lines with a picture area and no source row (always black). line_row[line] = the row line `line` shows, -1: the
	 * line has no picture area. */
	int32_t *pic_rows;      int pic_nrows;
	int32_t *line_row;
	int comp_phases;        /* frames after which a line's colour subcarrier, V-switch and burst repeat (1, 2 or 4; 0: more:
	                         * no composite store, k_line's PS forms) */
	double glut[256];
	htv_c16_t *clut;        size_t clut_len;      /* clut_width + W */
	int16_t *burst_win;     int burst_width;

	uint64_t *fm_ang;                              /* 65536: effective angle of each FM LUT entry, turns * 2^64 */
	float *fm_rot8;                                /* 65536 x (cos, sin) of 8 steps of fm_ang */
	uint64_t *fmv_ang;                             /* the same for the FM video modulator's LUT */
	int32_t afir_v[HTV_AFIR_N], afir_f[HTV_AFIR_N]; /* audio FIR taps in application order */
	int16_t lim_shape[HTV_LIM_W];

	int16_t *nicam_taps;    int nicam_ntaps;
	int16_t *nicam_lut;     int nicam_lut_len;     /* pulse-shaping table, see htv_tables.c */
	int16_t *nicam_tpad;                           /* 8 zeros, the pulse, zeros up to dp.nicam_tpad_len (multiple of 8) */
	htv_c16_t *nicam_cc;    int nicam_cc_len;
	uint8_t nicam_prn[90];

	htv_c32_t *secam_fm_lut;                       /* 65536 */
	htv_c16_t *secam_bell;                         /* 65536 */

	uint8_t *offset_start;  int offset_start_len;  /* start-up quirk, 2 bits/sample packed 1 byte/sample */

	/* --pixelrate (htv_tables_create2): resampler in front of the video filter, ref fir.c:263-355, 393-428.
	 * rs_taps[phase * rs_ataps + c] multiplies the input (newest - rs_ataps + 1 + c). */
	int rs_I, rs_D, rs_ataps, rs_wp;               /* interpolation, decimation, taps per phase, raster line width */
	int16_t *rs_taps;
	int raster_only;                               /* tables of the raster side of a --pixelrate encoder: no modulator scratch */

	int32_t *scratch;                              /* htv_tables_get */
};

extern void htv_tables_levels(const struct htv_tables_t *t, int levels[4]);

/* ---- device layer (htv_kernels.cu), all C linkage ---------------------- */

typedef struct htv_dev_t htv_dev_t;


extern int htv_dev_count(void);
/* device: CUDA ordinal, or -1 for the calling thread's current device */
extern htv_dev_t *htv_dev_create(const struct htv_tables_t *t, int max_frame_slots, int device, char *err, size_t errlen);
extern int htv_dev_device(const htv_dev_t *d);
extern void htv_dev_destroy(htv_dev_t *d);
/* frame slot <- host RGB (active_width x active_lines), async on stream */
extern void *htv_dev_uploads_begin(htv_dev_t *d);
extern int htv_dev_uploads_end(htv_dev_t *d, void *stream);
extern int htv_dev_overlay_capacity(void);
extern int htv_dev_set_overlays(htv_dev_t *d, int n, const long long *line, const int *from, const int *to,
	const int *value, const int16_t *const *add);
extern int htv_dev_upload_frame(htv_dev_t *d, int slot, const uint32_t *rgb, void *stream);
extern int htv_dev_upload_frames(htv_dev_t *d, int slot, int count, const uint32_t *rgb, void *stream);
/* slot_of_frame[i] = slot holding frame (first_frame + i) for this launch */
extern int htv_dev_set_frame_map(htv_dev_t *d, const int32_t *slot_of_frame, int n, int64_t first_frame, void *stream);
/* raw audio ring <- host PCM pairs for absolute indices [j0, j0 + n) */
extern int htv_dev_upload_audio(htv_dev_t *d, int64_t j0, const int16_t *pcm, size_t npairs, void *stream);
/* audio-rate pre-pass for the absolute audio-clock sample range [m0, m1) */
extern int htv_dev_audio_prepass(htv_dev_t *d, int64_t m0, int64_t m1, void *stream);
/* the line kernel(s): render lines [line0, line0 + nlines) to d_out (device); r is NULL, or with --pixelrate the raster
 * context at the pixel rate, d then being the sample-rate context (htv_kernels.cu) */
extern int htv_dev_render_lines(htv_dev_t *d, htv_dev_t *r, int64_t line0, int nlines, int16_t *d_out,
	const int16_t *d_acc, int acc_lines, void *stream);
extern void *htv_dev_event_new_timed(htv_dev_t *d);
extern float htv_dev_event_elapsed(void *e0, void *e1);
extern int htv_dev_mix_add(int16_t *d_acc, const int16_t *d_in, size_t nvalues, void *stream);
/* the kernels of the new type's stores (before the first rendered line); HTV_ERROR with a message on stderr */
extern int htv_dev_set_sample_type(htv_dev_t *d, int type);
/* the alignment htv_render / htv_render_add need of d_out (bytes): the widest access of the plan's store and combiner */
extern int htv_dev_out_align(const htv_dev_t *d);
/* the name htv_line_kernel would report for an encoder of these tables writing this sample type, under the switches
 * (HTV_PATH, HTV_FIR, HTV_KL) in the environment; the kernel selection alone, without a CUDA call (CPU tests) */
extern int htv_dev_plan_name(const struct htv_tables_t *t, int sample_type, char *name, size_t len);
extern int htv_dev_convert(void *d_dst, int type, const int16_t *d_src, size_t nvalues, void *stream);
extern int htv_dev_memcpy_h2d(htv_dev_t *d, void *dst, const void *src, size_t bytes, void *stream);
extern int htv_dev_sync(htv_dev_t *d, void *stream);
extern int htv_dev_memcpy_d2h(htv_dev_t *d, void *dst, const void *src, size_t bytes, void *stream);
extern void *htv_dev_alloc(htv_dev_t *d, size_t bytes);
extern void htv_dev_free(htv_dev_t *d, void *p);
extern void *htv_dev_alloc_pinned(size_t bytes);
extern void htv_dev_free_pinned(void *p);
extern uint64_t htv_dev_launches(const htv_dev_t *d);
extern const char *htv_dev_line_kernel(const htv_dev_t *d);
extern void htv_dev_secam_chain(const htv_dev_t *d, htv_secam_chain_t *out);
extern void htv_dev_set_timing(htv_dev_t *d, int on);
extern float htv_dev_last_line_ms(htv_dev_t *d);
extern int htv_dev_last_line_count(const htv_dev_t *d);
extern size_t htv_dev_audio_ring_pairs(void);
extern void *htv_dev_stream_new(htv_dev_t *d);
extern void htv_dev_stream_free(void *s);
extern void *htv_dev_event_new(htv_dev_t *d);
extern void htv_dev_event_free(void *e);
extern int htv_dev_event_record(void *e, void *stream);
extern int htv_dev_event_wait(void *e);          /* host waits for the event */
extern int htv_dev_stream_wait(void *stream, void *e);

#ifdef __cplusplus
}
#endif

#endif
