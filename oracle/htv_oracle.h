/* TEST INFRASTRUCTURE — the parity oracle. NOT part of the product.
 *
 * A plain-C, single-threaded CPU restatement of the reference's (fsphil/hacktv)
 * composite-video -> IQ hot path, written from scratch against the reference's
 * behaviour. Every function in htv_oracle.c cites the reference file:line it
 * restates. Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load this library; the product (hacktv_b200/) never
 * does.
 *
 * Pinning: the reference has no tests or golden vectors of its own
 * (SURVEY.md §4). The oracle is pinned against outputs of the reference ITSELF,
 * built unmodified into oracle/_ref/ (oracle/Makefile, `make ref`) - bit-exact
 * on every BASELINE.json config (tests/test_oracle_vs_ref.py, and the committed
 * fixtures under tests/golden/ made by tests/golden/make_golden.py).
 *
 * Formulation: the reference runs a pthread pipeline over a ring of line
 * buffers (video.c:3543-3618, 4867-4952). The oracle restates the same
 * arithmetic as a flat stream: line t is rastered, SECAM-coloured, VSB-filtered
 * (a centred 51-tap FIR over the concatenated I stream with zero history -
 * SURVEY.md §9 V1) and given its audio subcarriers, in stream order, with the
 * reference's sequential recurrences (Q31 NCOs with renormalisation, limiter,
 * NICAM overlap-add ring, SECAM IIR) kept as recurrences.
 */
#ifndef HTV_ORACLE_H
#define HTV_ORACLE_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Values of the enumerated fields (reference video.h:49-87, rf.h:26-28) */
#define ORC_OUT_COMPLEX 0
#define ORC_OUT_REAL    1
#define ORC_MOD_NONE 0
#define ORC_MOD_AM   1
#define ORC_MOD_VSB  2
#define ORC_MOD_FM   3
#define ORC_RASTER_625 0
#define ORC_RASTER_525 1
#define ORC_COLOUR_NONE  0
#define ORC_COLOUR_PAL   1
#define ORC_COLOUR_NTSC  2
#define ORC_COLOUR_SECAM 3
#define ORC_PREEMPH_NONE 0
#define ORC_PREEMPH_50US 1
#define ORC_PREEMPH_75US 2
#define ORC_PREEMPH_J17  3

/* The hot-path subset of vid_config_t (reference video.h:125-292), same field
 * names and meaning. Plain doubles / ints only. */
typedef struct {
	int32_t output_type;
	int32_t modulation;
	double video_bw;
	double vsb_upper_bw;
	double vsb_lower_bw;
	double level;
	int32_t swap_iq;
	int32_t invert_video;
	int64_t offset;
	double video_level;
	double fm_mono_level;
	double am_audio_level;
	double nicam_level;
	int32_t type;
	int32_t lines;
	int64_t frame_rate_num;
	int64_t frame_rate_den;
	int32_t hline;
	int32_t interlaced;
	int32_t active_lines;
	int32_t vfilter;
	double hsync_width;
	double vsync_short_width;
	double vsync_long_width;
	double sync_rise;
	double white_level;
	double black_level;
	double blanking_level;
	double sync_level;
	double active_width;
	double active_left;
	double gamma;
	double rw_co;
	double gw_co;
	double bw_co;
	int32_t colour_mode;
	int32_t volume;
	int64_t colour_carrier_num;
	int64_t colour_carrier_den;
	double colour_bw;
	double burst_width;
	double burst_left;
	double burst_level;
	double burst_rise;
	double ev_co;
	double eu_co;
	double fm_mono_carrier;
	double fm_mono_deviation;
	int32_t fm_mono_preemph;
	int32_t reserved0;
	double nicam_carrier;
	double nicam_beta;
	double am_mono_carrier;
	/* FM video (modulation == ORC_MOD_FM; ref video.h:141-143). Energy dispersal is not modelled:
	 * no mode in scope enables it and the front end has no switch for it. */
	double fm_level;
	double fm_deviation;
	double fm_energy_dispersal;
} orc_params_t;

typedef struct orc_t orc_t;

extern size_t orc_params_size(void);

/* vid_init (reference video.c:3812-4704). sample_rate == pixel_rate (the
 * resampler, video.c:3627-3651, is out of scope). Returns NULL on bad params. */
extern orc_t *orc_open(const orc_params_t *p, unsigned int sample_rate);
/* vid_init with pixel_rate != sample_rate: the --pixelrate resampler (ref video.c:3627-3651, 4361-4368) */
extern orc_t *orc_open2(const orc_params_t *p, unsigned int sample_rate, unsigned int pixel_rate);
extern void orc_close(orc_t *o);

/* AV source (reference av.h:64-116 callbacks, flattened): frames are RGB32
 * active_width x active_lines, used cyclically one per video frame; audio is
 * 32 kHz stereo int16, used cyclically. Pointers are borrowed. */
/* SECAM: let the luma notch read what the reference's subcarrier loop left past the end of earlier lines in its line
 * buffers' zero-heap padding (ref video.c:3206, 3228), as the reference does, instead of zeros. Not with --pixelrate. */
extern void orc_set_ref_heap(orc_t *o, int on);
extern void orc_set_frames(orc_t *o, const uint32_t *rgb, int nframes);
extern void orc_set_audio(orc_t *o, const int16_t *pcm, size_t npairs);
/* External int16 complex stream added to the output (ref --passthru, video.c:3517-3541);
 * borrowed pointer, set before the first orc_render */
extern void orc_set_passthru(orc_t *o, const int16_t *iq, size_t ncomplex);

/* vid_next_line x nlines + the file sink (reference video.c:4936-4952,
 * rf_file.c:97-116,226-233): appends the next nlines scan lines of the emitted
 * stream to out - int16 I,Q interleaved for complex modes, I only for real
 * modes. Returns the number of samples written. */
/* VBI overlays (ref vbidata.c:186-239 adds int16 deltas into a line after the raster stage; wss.c:182-185
 * first overwrites part of line 23): applied to `line` (1-based) of every frame after its
 * raster and SECAM stages, before the video filter (the order video.c:4206-4357 registers
 * them in). `add` (W values, may be NULL) is borrowed. Overlays must leave the first 40 samples of
 * a line alone (this restatement filters line t before line t+1 has been overlaid). */
extern void orc_add_vbi_line(orc_t *o, int line, int replace_from, int replace_to, int replace_value, const int16_t *add);

extern size_t orc_render(orc_t *o, int nlines, int16_t *out);

/* Geometry (reference video.c:3844-3853 and friends) */
extern int orc_width(const orc_t *o);
extern int orc_raster_width(const orc_t *o);
extern int orc_active_width(const orc_t *o);
extern int orc_active_lines(const orc_t *o);
extern int orc_is_complex(const orc_t *o);

/* Named table access for unit tests: returns a pointer to int32 copies of the
 * table entries and their count, or NULL. Names: "sync0".."sync4" (values),
 * "sync_off" (5 offsets), "burst_win", "chroma_taps", "vsb_itaps",
 * "vsb_qtaps", "levels" (white, black, blank, sync), "nicam_taps",
 * "geometry" (width, half_width, active_left, active_width, burst_left,
 * burst_width). */
extern const int32_t *orc_table(orc_t *o, const char *name, int *count);

/* The reference's built-in test source (reference av_test.c:71-205) */
extern void orc_test_pattern(int width, int height, uint32_t *rgb);
extern size_t orc_test_tone_pairs(void);
extern void orc_test_tone(int16_t *pcm);

/* RGB -> (y,u,v) int16 levels (reference video.c:3912-3959) for one colour */
extern void orc_yuv(const orc_t *o, uint32_t rgb, int16_t yuv[3]);

#ifdef __cplusplus
}
#endif

#endif
