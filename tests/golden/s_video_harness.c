/* TEST INFRASTRUCTURE - writes the reference's S-Video stream for tests/golden/make_golden_s_video.py.
 *
 * Drives the unmodified reference encoder (its objects as `make -C oracle ref` compiles them in place) the way
 * hacktv.c does for `--s-video`: mode lookup, the S-Video check and vid_conf.s_video = 1 (hacktv.c:1136-1148), the
 * in-scope overrides, vid_init, the test source or RGB32 pictures through the av_t callbacks, vid_next_line, and the
 * file sink's complex layout (hacktv.c:1493 opens it complex for S-Video: I,Q interleaved, rf_file.c:226-233).
 *
 *   s_video_harness -m MODE -s RATE [--filter] [--swap-iq] [--offset HZ] [--frames FILE.rgb32] --lines N -o FILE
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include <unistd.h>
#include "hacktv.h"
#include "av_test.h"

typedef struct { int width, height; uint32_t *frames; size_t nframes, cur; } pictures_t;

static int _read_video(void *ctx, av_frame_t *frame)
{
	pictures_t *p = ctx;
	uint32_t *fb = p->frames + (size_t) p->width * p->height * p->cur;
	p->cur = (p->cur + 1) % p->nframes;
	av_frame_init(frame, p->width, p->height, fb, 1, p->width);
	return(AV_OK);
}

int main(int argc, char **argv)
{
	static hacktv_t s;
	const vid_configs_t *vc;
	vid_config_t conf;
	const char *mode = NULL, *out = NULL, *frames_fn = NULL;
	unsigned int rate = 0;
	int filter = 0, swap_iq = 0, i;
	long long offset = 0, lines = 0, n;
	FILE *fo;

	for(i = 1; i < argc; i++)
	{
		if(!strcmp(argv[i], "-m") && i + 1 < argc) mode = argv[++i];
		else if(!strcmp(argv[i], "-s") && i + 1 < argc) rate = strtoul(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "--filter")) filter = 1;
		else if(!strcmp(argv[i], "--swap-iq")) swap_iq = 1;
		else if(!strcmp(argv[i], "--offset") && i + 1 < argc) offset = strtoll(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "--frames") && i + 1 < argc) frames_fn = argv[++i];
		else if(!strcmp(argv[i], "--lines") && i + 1 < argc) lines = strtoll(argv[++i], NULL, 10);
		else if(!strcmp(argv[i], "-o") && i + 1 < argc) out = argv[++i];
		else { fprintf(stderr, "s_video_harness: unknown argument %s\n", argv[i]); return(2); }
	}
	if(!mode || !rate || !out || lines <= 0) { fprintf(stderr, "s_video_harness: -m, -s, --lines and -o are required\n"); return(2); }

	for(vc = vid_configs; vc->id != NULL; vc++) if(strcmp(mode, vc->id) == 0) break;
	if(vc->id == NULL) { fprintf(stderr, "Unrecognised TV mode.\n"); return(2); }
	memcpy(&conf, vc->conf, sizeof(vid_config_t));

	/* hacktv.c:1136-1148 */
	if((conf.colour_mode != VID_PAL && conf.colour_mode != VID_SECAM && conf.colour_mode != VID_NTSC) ||
	   conf.output_type != RF_INT16_REAL)
	{
		fprintf(stderr, "S-Video is only available with PAL, SECAM, or NTSC baseband modes.\n");
		return(1);
	}
	conf.s_video = 1;
	if(filter) conf.vfilter = 1;
	conf.swap_iq = swap_iq;
	conf.offset = offset;
	conf.volume = 256;                                    /* hacktv.c's default --volume 1.0 */
	conf.raw_bb_white_level = INT16_MAX;

	memset(&s, 0, sizeof(s));
	if(vid_init(&s.vid, rate, 0, &conf) != VID_OK) { fprintf(stderr, "vid_init failed\n"); return(1); }

	/* hacktv.c:1503-1518 */
	s.vid.av = (av_t) {
		.frame_rate = (r64_t) { s.vid.conf.frame_rate.num * (s.vid.conf.interlace ? 2 : 1), s.vid.conf.frame_rate.den },
		.display_aspect_ratios = { s.vid.conf.frame_aspects[0], s.vid.conf.frame_aspects[1] },
		.fit_mode = AV_FIT_STRETCH,
		.width = s.vid.active_width,
		.height = s.vid.conf.active_lines,
		.sample_rate = (r64_t) { HACKTV_AUDIO_SAMPLE_RATE, 1 },
	};
	if(frames_fn)
	{
		pictures_t *p = calloc(1, sizeof(pictures_t));
		FILE *f = fopen(frames_fn, "rb");
		long len;
		if(!p || !f) { perror(frames_fn); return(2); }
		fseek(f, 0, SEEK_END);
		len = ftell(f);
		fseek(f, 0, SEEK_SET);
		p->width = s.vid.active_width;
		p->height = s.vid.conf.active_lines;
		p->nframes = (size_t) len / ((size_t) p->width * p->height * 4);
		p->frames = malloc(len);
		if(p->nframes < 1 || !p->frames || fread(p->frames, 1, len, f) != (size_t) len) { fprintf(stderr, "bad frame file\n"); return(2); }
		fclose(f);
		s.vid.av.av_source_ctx = p;
		s.vid.av.read_video = _read_video;
	}
	else if(av_test_open(&s.vid.av) != AV_OK) { fprintf(stderr, "av_test_open failed\n"); return(1); }

	fo = fopen(out, "wb");
	if(!fo) { perror(out); return(1); }
	for(n = 0; n < lines; n++)
	{
		vid_line_t *l = vid_next_line(&s.vid);
		if(l == NULL) break;
		fwrite(l->output, sizeof(int16_t) * 2, l->width, fo);
	}
	fclose(fo);
	/* no vid_free: the process ends here (the reference's thread shutdown can wait forever, see oracle/ref_harness.c) */
	fflush(NULL);
	_exit(n == lines ? 0 : 1);
}
