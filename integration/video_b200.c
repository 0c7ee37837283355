/* video_b200.c - the reference-side binding: hacktv's video.h entry points implemented
 * on top of the hacktv_b200 C-ABI (include/hacktv_b200.h).
 *
 * This file is what a hacktv maintainer adds to src/. It is compiled AGAINST THE
 * REFERENCE'S OWN HEADERS (video.h, av.h, rf.h - unmodified) and exports the symbols the
 * rest of hacktv links to: vid_init, vid_next_line, vid_free, vid_info,
 * vid_get_framebuffer_length (ref video.h:512-516). hacktv.c, av*.c, rf*.c stay untouched;
 * the stock encoder in video.c is kept as the fallback for every configuration the GPU
 * path does not cover (teletext, scramblers, MAC, energy dispersal, ...) by building it with
 *     -Dvid_init=cpu_vid_init -Dvid_next_line=cpu_vid_next_line -Dvid_free=cpu_vid_free
 *     -Dvid_info=cpu_vid_info -Dvid_get_framebuffer_length=cpu_vid_get_framebuffer_length
 * (see oracle/Makefile target `dropin`, which does exactly that without touching a source).
 *
 * It cannot be built outside a hacktv source tree and is not part of libhacktv_b200.so.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <time.h>
#include "video.h"
#include "hacktv_b200.h"

/* the stock CPU encoder, renamed at compile time */
extern int cpu_vid_init(vid_t *s, unsigned int sample_rate, unsigned int pixel_rate, const vid_config_t * const conf);
extern void cpu_vid_free(vid_t *s);
extern void cpu_vid_info(vid_t *s);
extern size_t cpu_vid_get_framebuffer_length(vid_t *s);
extern vid_line_t *cpu_vid_next_line(vid_t *s);

#define MAX_ENCODERS 16
#define MAX_VBI 64
static struct {
	vid_t *vid; htv_t *htv; vid_line_t line; uint32_t *packed; uint64_t serial;
	/* HACKTV_STATS=1: lines handed out and the wall time they took, printed by vid_free (bench.py drop-in figure) */
	long long stat_lines; struct timespec stat_t0;
	/* VBI stages: the reference's own code builds the waveforms, the encoder's overlay hook carries them */
	int16_t *vbi_scratch;           /* one line, I/Q interleaved, as the stock stages expect it */
	cint16_t *clut;                 /* the colour subcarrier table vits_render mixes its chroma with (ref video.c:3961-3987) */
	unsigned int clut_width;
	int16_t *vbi_add[MAX_VBI];
	htv_vbi_line_t vbi[MAX_VBI];
} _enc[MAX_ENCODERS];

static int _find(vid_t *s)
{
	int i;
	for(i = 0; i < MAX_ENCODERS; i++) if(_enc[i].vid == s) return(i);
	return(-1);
}

static void _translate(htv_config_t *h, const vid_config_t *c);

/* Can the accelerated path render this configuration bit for bit? (SURVEY.md section 8) */
static int _accelerated(const vid_config_t *c, unsigned int sample_rate, unsigned int pixel_rate)
{
	if(getenv("HACKTV_NO_B200")) return(0);
	if(c->type != VID_RASTER_625 && c->type != VID_RASTER_525) return(0);
	if(c->modulation == VID_FM && c->fm_energy_dispersal != 0) return(0);
	if(c->colour_mode != VID_NONE && c->colour_mode != VID_PAL && c->colour_mode != VID_NTSC && c->colour_mode != VID_SECAM) return(0);
	/* --pixelrate: PAL / NTSC / mono through the device resampler; SECAM, FM video and S-Video with a resampler,
	 * and rate pairs whose line width would vary, stay on the stock encoder (DESIGN.md section 8) */
	if(pixel_rate && pixel_rate != sample_rate)
	{
		htv_config_t hc;
		htv_tables_t *t;
		if(c->colour_mode == VID_SECAM || c->modulation == VID_FM) return(0);
		_translate(&hc, c);
		t = htv_tables_create2(&hc, sample_rate, pixel_rate);          /* host only: NULL when out of scope */
		if(!t) return(0);
		htv_tables_free(t);
	}
	if(c->s_video)
	{
		/* S-Video runs on the fused line kernels only: a chroma low-pass of fewer than 3 taps (PAL and NTSC at
		 * 1.25 Msps and below), which the split modulators take, stays on the stock encoder */
		htv_config_t hc;
		htv_tables_t *t;
		int ntaps = 0;
		_translate(&hc, c);
		t = htv_tables_create2(&hc, sample_rate, pixel_rate);
		if(!t) return(0);
		htv_tables_get(t, "chroma_taps", &ntaps);
		htv_tables_free(t);
		if(c->colour_mode != VID_SECAM && ntaps < 3) return(0);
	}
	if(c->videocrypt || c->videocrypt2 || c->videocrypts || c->syster ||
	   c->d11 || c->systercnr || c->acp || c->sis || c->eurocrypt) return(0);
	if(c->raw_bb_file || c->a2stereo || c->secam_field_id) return(0);
	if(c->fm_left_level > 0 || c->fm_right_level > 0 || c->dance_level > 0) return(0);
	if(c->interlace || c->frame_orientation) return(0);
	return(1);
}

static void _translate(htv_config_t *h, const vid_config_t *c)
{
	memset(h, 0, sizeof(*h));
#define CP(f) h->f = c->f
	CP(output_type); CP(modulation); CP(video_bw); CP(vsb_upper_bw); CP(vsb_lower_bw); CP(level);
	CP(swap_iq); CP(invert_video); CP(offset); CP(video_level); CP(fm_mono_level); CP(am_audio_level);
	CP(nicam_level); CP(type); CP(lines); CP(hline); CP(interlaced); CP(active_lines); CP(vfilter);
	CP(hsync_width); CP(vsync_short_width); CP(vsync_long_width); CP(sync_rise);
	CP(white_level); CP(black_level); CP(blanking_level); CP(sync_level); CP(active_width); CP(active_left);
	CP(gamma); CP(rw_co); CP(gw_co); CP(bw_co); CP(colour_mode); CP(volume); CP(colour_bw);
	CP(burst_width); CP(burst_left); CP(burst_level); CP(burst_rise); CP(ev_co); CP(eu_co);
	CP(fm_mono_carrier); CP(fm_mono_deviation); CP(fm_mono_preemph); CP(nicam_carrier); CP(nicam_beta);
	CP(am_mono_carrier); CP(fm_level); CP(fm_deviation); CP(fm_energy_dispersal); CP(s_video);
#undef CP
	h->frame_rate_num = c->frame_rate.num; h->frame_rate_den = c->frame_rate.den;
	h->colour_carrier_num = c->colour_carrier.num; h->colour_carrier_den = c->colour_carrier.den;
}

/* htv_av_t callbacks -> the reference's av_t (which hacktv.c fills in s->vid.av) */
static int _read_video(void *ctx, htv_frame_t *out)
{
	int i = _find((vid_t *) ctx), x, y;
	vid_t *s = ctx;
	av_frame_t f;
	if(i < 0 || av_read_video(&s->av, &f) != AV_OK || !f.framebuffer) return(HTV_ERROR);
	s->vframe = f;                                  /* WSS auto mode reads its pixel aspect ratio (wss.c:168-180) */
	out->width = f.width; out->height = f.height;
	out->serial = ++_enc[i].serial;                 /* a pulled frame may have changed: always upload */
	if(f.pixel_stride == 1 && f.line_stride == f.width) { out->framebuffer = f.framebuffer; return(HTV_OK); }
	if(!_enc[i].packed) _enc[i].packed = malloc(sizeof(uint32_t) * f.width * f.height);
	for(y = 0; y < f.height; y++)
		for(x = 0; x < f.width; x++)
			_enc[i].packed[y * f.width + x] = f.framebuffer[y * f.line_stride + x * f.pixel_stride];
	out->framebuffer = _enc[i].packed;
	return(HTV_OK);
}

static int _read_audio(void *ctx, const int16_t **samples, size_t *npairs)
{
	vid_t *s = ctx;
	int16_t *p = NULL;
	int r = av_read_audio(&s->av, &p, npairs);
	*samples = p;
	return(r == AV_OK ? HTV_OK : HTV_ERROR);
}

/* htv_read_vbi_t, once per frame: run the reference's own VBI stages (vid_lineprocess_process_t, ref
 * video.h:332), in the order vid_init registers them (ref video.c:4213-4357: ... wss ... vitc ... teletext),
 * line by line on an empty line buffer - exactly what they see in the stock pipeline, vbialloc included -
 * and hand what they drew to the encoder's overlay hook. Only WSS overwrites before it adds: part of line 23
 * is set to black (wss.c:182-185), which is passed on as the overlay's replace range. */
static int _read_vbi(void *ctx, int frame, const htv_vbi_line_t **lines, int *nlines)
{
	vid_t *s = ctx;
	int i = _find(s), n = 0, line, x, dirty = 1;
	const int W = s->width;
	if(i < 0) return(HTV_ERROR);
	s->frame = frame;
	for(line = 1; line <= s->conf.lines && n < MAX_VBI; line++)
	{
		vid_line_t l, *lp = &l;
		int rep_from = 0, rep_to = 0, rep_value = 0, any = 0;
		int16_t *add;
		if(dirty) memset(_enc[i].vbi_scratch, 0, sizeof(int16_t) * 2 * W);
		memset(&l, 0, sizeof(l));
		l.output = _enc[i].vbi_scratch; l.width = W; l.frame = frame; l.line = line;
		l.previous = l.next = &l;
		/* the line's place in the subcarrier table: the raster advances it by one line width per line (ref video.c:2904-2910) */
		if(_enc[i].clut)
		{
			const unsigned long long gl = (unsigned long long) (frame - 1) * s->conf.lines + (line - 1);
			l.lut = &_enc[i].clut[(gl * (unsigned long long) W) % _enc[i].clut_width];
		}
		if(s->conf.vits) vits_render(s, &s->vits, 1, &lp);
		if(s->conf.wss)
		{
			wss_render(s, &s->wss, 1, &lp);
			if(line == 23) { rep_from = s->half_width; rep_to = s->wss.blank_width; rep_value = s->black_level; }
		}
		if(s->conf.vitc) vitc_render(s, &s->vitc, 1, &lp);
		if(s->conf.cc608) cc608_render(s, &s->cc608, 1, &lp);
		if(s->conf.teletext) tt_render_line(s, &s->tt, 1, &lp);
		dirty = l.vbialloc;
		if(!l.vbialloc) continue;
		if(!_enc[i].vbi_add[n]) _enc[i].vbi_add[n] = malloc(sizeof(int16_t) * W);
		add = _enc[i].vbi_add[n];
		for(x = 0; x < W; x++)
		{
			add[x] = l.output[x * 2] - (x >= rep_from && x < rep_to ? rep_value : 0);
			any |= add[x];
		}
		if(!any && rep_from >= rep_to) continue;
		_enc[i].vbi[n++] = (htv_vbi_line_t) { line, rep_from, rep_to, rep_value, add };
	}
	*lines = _enc[i].vbi;
	*nlines = n;
	return(HTV_OK);
}

/* --passthru: the external stream as the reference reads it (video.c:3527-3533) */
static size_t _read_passthru(void *ctx, int16_t *iq, size_t ncomplex)
{
	FILE *f = ctx;
	size_t x = 0, i;
	while(x < ncomplex && (i = fread(iq + x * 2, sizeof(int16_t) * 2, ncomplex - x, f)) > 0) x += i;
	return(x);
}

int vid_init(vid_t *s, unsigned int sample_rate, unsigned int pixel_rate, const vid_config_t * const conf)
{
	htv_config_t hc;
	htv_t *h = NULL;
	FILE *pt = NULL;
	int i;

	if(!_accelerated(conf, sample_rate, pixel_rate)) return(cpu_vid_init(s, sample_rate, pixel_rate, conf));
	_translate(&hc, conf);
	if(htv_init(&h, sample_rate, pixel_rate, &hc) != HTV_OK)
	{
		/* an in-scope configuration never silently drops to the CPU: set HACKTV_NO_B200=1 to ask for it */
		fprintf(stderr, "video_b200: the GPU encoder could not be initialised\n");
		return(VID_ERROR);
	}
	i = _find(NULL);
	if(i < 0) { htv_free(h); return(VID_ERROR); }
	if(conf->passthru)
	{
		/* ref video.c:4607-4624 */
		pt = strcmp(conf->passthru, "-") == 0 ? stdin : fopen(conf->passthru, "rb");
		if(!pt) { perror(conf->passthru); htv_free(h); return(VID_ERROR); }
		htv_set_passthru(h, _read_passthru, pt);
	}

	/* the fields hacktv.c and the sinks read (ref hacktv.c:1447-1526) */
	memset(s, 0, sizeof(vid_t));
	s->conf = *conf;
	s->sample_rate = sample_rate;
	s->pixel_rate = pixel_rate ? pixel_rate : sample_rate;
	s->width = s->max_width = htv_samples_per_line(h);
	s->active_width = htv_active_width(h);
	{
		int lv[4];
		htv_signal_levels(h, lv);
		s->white_level = lv[0]; s->black_level = lv[1]; s->blanking_level = lv[2]; s->sync_level = lv[3];
		s->half_width = htv_half_line(h);
	}
	s->thread_abort = 1;                             /* no CPU stage threads to join */
	s->passthru = pt;
	_enc[i].vid = s; _enc[i].htv = h; _enc[i].serial = 0;
	if(conf->vits || conf->wss || conf->vitc || conf->cc608 || conf->teletext)
	{
		/* ref video.c:4216-4232, 4234-4242, 4305-4328, 4346-4358: the stock stages, initialised as vid_init does */
		if((conf->vits && vits_init(&s->vits, s->pixel_rate, s->width, s->conf.lines, s->conf.colour_mode == VID_PAL,
		                            s->white_level - s->blanking_level) != VID_OK) ||
		   (conf->wss && wss_init(&s->wss, s, conf->wss) != VID_OK) ||
		   (conf->vitc && vitc_init(&s->vitc, s) != VID_OK) ||
		   (conf->cc608 && cc608_init(&s->cc608, s) != VID_OK) ||
		   (conf->teletext && tt_init(&s->tt, s, conf->teletext) != VID_OK)) { _enc[i].vid = NULL; htv_free(h); return(VID_ERROR); }
		if(conf->vits && (conf->colour_mode == VID_PAL || conf->colour_mode == VID_NTSC))
		{
			/* vits_render adds its chroma through the line's subcarrier table (l->lut): the same table the raster
			 * uses, built as vid_init builds it (ref video.c:3961-3987) */
			r64_t a = r64_div((r64_t) { s->pixel_rate, 1 }, conf->colour_carrier);
			const double d = 2.0 * M_PI * ((double) a.den / a.num);
			int64_t c;
			_enc[i].clut_width = a.num;
			_enc[i].clut = malloc((a.num + s->width) * sizeof(cint16_t));
			if(!_enc[i].clut) { _enc[i].vid = NULL; htv_free(h); return(VID_OUT_OF_MEMORY); }
			for(c = 0; c < a.num + s->width; c++)
			{
				_enc[i].clut[c] = (cint16_t) { round(cos(d * c) * INT16_MAX), round(sin(d * c) * INT16_MAX) };
			}
		}
		_enc[i].vbi_scratch = malloc(sizeof(int16_t) * 2 * s->width);
		htv_set_vbi_source(h, _read_vbi, s);
	}
	htv_av(h)->ctx = s;
	htv_av(h)->read_video = _read_video;
	htv_av(h)->read_audio = _read_audio;
	return(VID_OK);
}

vid_line_t *vid_next_line(vid_t *s)
{
	int i = _find(s);
	htv_line_t *l;
	if(i < 0) return(cpu_vid_next_line(s));
	if(av_eof(&s->av)) return(NULL);
	if(_enc[i].stat_lines++ == 0)
	{
		clock_gettime(CLOCK_MONOTONIC, &_enc[i].stat_t0);
		/* HACKTV_B200_PREFETCH=1: let the encoder run one frame ahead of the consumer (htv_set_prefetch). It pulls the AV
		 * source one frame early, so it is for sources that do not end - the test pattern, live capture; at the end
		 * of a file av_eof() (ref av.c:84-87) would fire one frame too soon. */
		{
			const char *pf = getenv("HACKTV_B200_PREFETCH");
			if(pf && pf[0] == '1') htv_set_prefetch(_enc[i].htv, 1);
		}
	}
	l = htv_next_line(_enc[i].htv);
	if(!l) return(NULL);
	memset(&_enc[i].line, 0, sizeof(vid_line_t));
	_enc[i].line.output = l->output;
	_enc[i].line.width = l->width;
	_enc[i].line.frame = s->frame = l->frame;
	_enc[i].line.line = s->line = l->line;
	return(&_enc[i].line);
}

void vid_free(vid_t *s)
{
	int i = _find(s);
	if(i < 0) { cpu_vid_free(s); return; }
	if(getenv("HACKTV_STATS") && _enc[i].stat_lines > 0)
	{
		struct timespec t1;
		clock_gettime(CLOCK_MONOTONIC, &t1);
		fprintf(stderr, "{\"encoder\": \"hacktv_b200\", \"lines\": %lld, \"seconds\": %.6f}\n", _enc[i].stat_lines,
			(double) (t1.tv_sec - _enc[i].stat_t0.tv_sec) + 1e-9 * (double) (t1.tv_nsec - _enc[i].stat_t0.tv_nsec));
	}
	av_close(&s->av);
	if(s->passthru) fclose(s->passthru);             /* ref video.c:4743-4746 */
	htv_av(_enc[i].htv)->close = NULL;
	htv_free(_enc[i].htv);
	free(_enc[i].packed);
	if(s->conf.wss) wss_free(&s->wss);
	if(s->conf.vitc) vitc_free(&s->vitc);
	if(s->conf.teletext) tt_free(&s->tt);
	if(s->conf.vits) vits_free(&s->vits);
	if(s->conf.cc608) cc608_free(&s->cc608);
	free(_enc[i].clut);
	free(_enc[i].vbi_scratch);
	{ int k; for(k = 0; k < MAX_VBI; k++) free(_enc[i].vbi_add[k]); }
	memset(&_enc[i], 0, sizeof(_enc[i]));
	memset(s, 0, sizeof(vid_t));
}

void vid_info(vid_t *s)
{
	int i = _find(s);
	if(i < 0) { cpu_vid_info(s); return; }
	htv_info(_enc[i].htv);
	fprintf(stderr, "Encoder: %s\n", htv_version());
}

size_t vid_get_framebuffer_length(vid_t *s)
{
	int i = _find(s);
	if(i < 0) return(cpu_vid_get_framebuffer_length(s));
	return(htv_get_framebuffer_length(_enc[i].htv));
}
