// hacktv_b200 - CUDA kernels (sm_90a) and the device layer behind the C-ABI.
//
// One CTA renders one scan line; a launch covers a run of lines (a field, a
// frame, or many frames). Every piece of state the reference carries from
// sample to sample (ref = fsphil/hacktv src/) is expressed as a closed form of
// the global sample index so lines are independent:
//
//   - raster (sync / blank / luma / PAL-NTSC chroma)   ref video.c:2864-3066
//   - VSB / low-pass video filter as a centred FIR     ref video.c:3235-3248, fir.c:304-355, 564-615
//   - FM / AM sound carriers: integer phase = prefix sum of exact per-sample
//     angles (audio-rate pre-pass), amplitude model of the Q31 recurrence   ref video.c:2259-2276, 2359-2378
//   - NICAM-728: frames encoded per millisecond in a pre-pass, pulse shaping by
//     direct evaluation of the <= 6 overlapping symbols per sample          ref nicam728.c:140-411
//   - frequency-offset mixer / IQ swap                  ref video.c:3466-3515
//
// The one dense contraction of the path, the 51-tap video filter, runs on the tensor cores as an exact
// int8 byte-split contraction (k_mod_mma, htv_mma_fir.h). The output is written once, with 128-bit
// streaming stores; all tables are L2/L1/shared resident.

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <stdarg.h>
#include <limits.h>
#include "htv_internal.h"
#include "htv_sample_type.h"
#include "htv_mma_fir.h"
#include "htv_resample.h"

#define HALO 25                       // (HTV_VF_NTAPS - 1) / 2
#define RA_BITS 20
#define RA (1 << RA_BITS)             // audio ring: pairs / processed samples / phase prefix
#define RS_BITS 23
#define RS (1 << RS_BITS)             // NICAM symbol ring
#define RF_BITS 14
#define RF (1 << RF_BITS)             // NICAM frame ring

#define CK(x) do { cudaError_t e_ = (x); if(e_ != cudaSuccess) { \
	fprintf(stderr, "hacktv_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return(HTV_ERROR); } } while(0)

// Every entry point that touches an encoder's device state runs with that encoder's device current
// and leaves the calling thread's current device as it found it: a host (hacktv itself, or any C
// program) can drive one encoder per GPU from one process, one thread per encoder or all from one.
struct DevGuard {
	int prev;
	bool switched;
	explicit DevGuard(int device) : prev(-1), switched(false)
	{
		if(cudaGetDevice(&prev) == cudaSuccess && prev != device) switched = cudaSetDevice(device) == cudaSuccess;
	}
	~DevGuard() { if(switched) cudaSetDevice(prev); }
};

// The record of audio index j for k_line's sound feed (htv_line.cuh), slot (j + 1) & (RA - 1): B(j), the phase
// accumulated before j's segment starts (for j = -1 one angle step less: see kl_lane_feed), the angle step of j's
// modulating sample and (cos, sin) of 8 of those steps (k_fm_scan_fix)
struct __align__(16) SegRec {
	ulonglong2 ba;                    // B(j), step
	float2 rot;
	float pad[2];
};

struct DevTables {
	const uint32_t *mma_atab;         // tap operand of the tensor-core video filter, fragment order (htv_mma_fir.h)
	const int16_t *tmpl_out, *tmpl_keep;   // line templates: blank + sync pulses (htv_tables.c build_templates)
	const uint8_t *tmpl_keep_any;
	const uint16_t *codes;
	const double *glut;
	const short4 *yuv_lut;            // [2^24] RGB -> (y, u, v, 0), the reference's yuv_level_lookup (video.c:3905-3960)
	const htv_c16_t *clut;
	const int16_t *burst_win;
	const uint64_t *fm_ang;
	const float2 *fm_rot8;            // (cos, sin) of 8 steps of fm_ang (fused line kernel)
	const uint32_t *notch_atab;       // SECAM luma notch as a tensor-core tap operand: [k-step][hi, lo][lane] x 4 registers
	const uint32_t *sec_lpf_atab;     // SECAM baseband low-pass, one k-step: [hi, lo][lane] x 4 registers
	const int16_t *sec_win;           // burst window by sample of the line (0 outside the subcarrier range), W rounded up to 8
	const int32_t *afir_v, *afir_f;
	const int16_t *lim_shape;
	const int16_t *nicam_taps;
	const int16_t *nicam_tpad;
	const int16_t *nicam_lut;
	const htv_c16_t *nicam_cc;
	const uint8_t *nicam_prn;
	const uint8_t *offset_start;
	const htv_c32_t *secam_fm_lut;
	const htv_c16_t *secam_bell;
	// frames
	const uint32_t *frames;           // slot-major, active_width * active_lines each
	const int32_t *frame_map;         // slot of frame (first_frame + i)
	int64_t frame_map_first;          // 0-based frame index of frame_map[0]
	int32_t frame_map_len;
	// composite store of the fused line kernel (k_compose): every line of the frame as the finished composite row before
	// the VBI overlay and the video filter, [slot][phase][line - 1][W], slot max_slots = black, phase = frame mod
	// comp_phases, then the two stream-start rows (comp_start: L < 0, comp_start + 1: L = 0); NULL on every other path
	int16_t *comp;
	int16_t *comp_q;                  // S-Video: the chroma term of each row (Q), same layout; NULL otherwise
	int32_t comp_phases, comp_black;  // colour-frame phases; the black slot
	int64_t comp_start;               // row of the first stream-start row
	// filtered store of the k_line forms with a video filter and a composite store (k_vf_rows): each composite-store row
	// of lines 2 .. lines - 1 after the video filter, as the line kernel holds it before the sound carriers - I | Q << 16,
	// S-Video's chroma added to Q - at the composite row's index; NULL on every other path
	uint32_t *filt;
	uint32_t *vfx;                    // the call's filtered rows of the lines vf_exception lists, [list index][W]
	int *vf_list;                     // [0]: how many; [1 + k]: raster descriptor entry of row k of vfx
	// converted picture store of the k_line encoders whose subcarrier does not repeat within 4 frames (k_picture; k_line's
	// PS forms): [slot][row][W], slot max_slots = black, row as htv_tables.c build_pic_rows; NULL on every other path
	const int4 *pic_rows;             // [pic_nrows] line (1-based, 0 none), al, ar, keep of the line that shows the row
	const int32_t *line_row;          // [lines + 1] the row line l shows, -1: no picture area
	int32_t pic_nrows, pic_black;     // rows per slot; the black slot
	int16_t *pic_val;                 // the line template outside [al, ar), Y + the template's keep part inside
	uint32_t *pic_cuv;                // U | V << 16 after the chroma low-pass (colour encoders; NULL for mono)
	// audio state rings
	const int16_t *pcm;               // RA stereo pairs, index j & (RA-1)
	int32_t *lim_var, *lim_fix;       // RA, index j & (RA-1)
	int16_t *fm_p;                    // RA, slot (j+1) & (RA-1): modulating sample in effect for audio index j
	uint64_t *fm_B;                   // RA, same slot: phase accumulated before that segment starts
	uint64_t *fm_inc;                 // RA, same slot: phase advance over the whole segment
	unsigned long long *scan_carry, *scan_tot;   // scratch of the two-pass phase scan
	uint8_t *nic_local;               // RS: inclusive prefix (mod 4) of the DQPSK steps inside the symbol's frame
	uint8_t *nic_ftot;                // RF: total step of frame k (mod 4)
	uint8_t *nic_fstart;              // RF: differential symbol state before frame k
	// records of k_line's sound feed (htv_line.cuh), written behind the pre-pass chains; NULL on the other paths
	SegRec *seg_rec;                  // RA, slot (j + 1) & (RA - 1): audio index j
	uint32_t *nic_rec;                // RS, slot s & (RS - 1): NICAM symbol s - pulse-table rows of its 6-symbol pattern,
	                                  // I (bits 0-8) and Q (9-17); its DQPSK polarities (18-19: symc's code); bit 20: no row
	// VBI overlays of the current launch sequence (sorted by global line index)
	int ov_n;
	const long long *ov_line;         // [ov_n] global line index
	const int4 *ov_meta;              // [ov_n] replace_from, replace_to, replace_value, row of ov_add or -1
	const int16_t *ov_add;            // [rows][W]
	// FM video
	const uint64_t *fmv_ang;          // 65536: effective rotation of each modulator LUT entry, turns * 2^64
	int16_t *fmv_base;                // [rows][W] modulating signal of the current sub-batch
	unsigned long long *fmv_tot;      // [rows] phase advance over each row
	unsigned long long *fmv_rowbase;  // [rows] phase before each row
	unsigned long long *fmv_carry;    // phase after the last row rendered so far
};

#define LOFF 33                       // luma window index = x + LOFF (aligned 128-bit loads at x0 - 25)
#define SEC_TAIL 8                    // low-pass outputs that see the two aliased words (7 used)

struct __align__(16) SecState {
	int A, B;                         // chrominance_buffer[W], [W + 1]
	int pad0, pad1;
	double ix, iy;                    // iir_int16_t state (ref fir.c:721-735)
};

struct __align__(16) SecChk {
	int pi, pq;                       // FM phasor before sample ck (valid: the FM loop came through there)
	int valid, pad;
	double ixm, iym;                  // IIR state before sample ck
};

struct SecScratch {
	int16_t *cbT;                     // [groups][rows][8] low-passed baseband without the aliased-tail terms
	int *tail;                        // [rows][SEC_TAIL]  raw sums of the last outputs
	SecState *st[2];                  // [rows] outgoing state, ping-pong between passes
	SecState *used;                   // [rows] the incoming state the line was last computed from ...
	SecState *outc;                   // [rows] ... and the outgoing state that computation gave
	SecState *carry;                  // state before the first line of the chain
	int *flags;                       // [0] outgoing states changed in the last pass, [2] lines recomputed, [3] work list length
	int16_t *yT;                      // [groups][rows][8] FM input: pre-emphasised, rounded, clamped baseband
	int *phT;                         // [groups][rows][8] phasor after each sample's step: (pi >> 16) & 0xFFFF | (pq >> 16) << 16
	double *iyc;                      // [W / 64 + 1][rows] IIR state iy before sample 64 k
	struct SecChk *chk;               // [rows] checkpoint before sample ck
	int *list;                        // [rows] lines whose FM recurrence must be re-run in full
	int rows;                         // row pitch of the transposed arrays
};

#define MAPBUFS 16
#define HTV_MAX_ALLOCS 128            // device tables owned by one encoder (about 50 for SECAM-L with AM + NICAM)
#define HTV_OV_CAP 2048                // VBI overlay lines per launch sequence

// The A/B and test switches, read from the environment once per encoder (dev_switches), beside HTV_SEC (sec_knobs)
struct DevSwitches {
	bool split;                       // HTV_PATH=split: the separate raster + modulator kernels where the fused ones would run
	bool scalar;                      // HTV_FIR=scalar: the scalar video filter and SECAM notch, not the tensor-core ones
	bool kl_general;                  // HTV_KL=general: never the k_line with the sound stages and width compiled in
	bool no_ahead;                    // HTV_AHEAD=0: the fused line kernel's sound pre-pass in the caller's stream order
	bool debug;                       // HTV_DEBUG: the SECAM chain's passes on stderr
};

// What an encoder launches (plan_kernels): chosen once from its tables, the switches and the sample type
enum { PATH_LINE, PATH_SEC_LINE, PATH_SPLIT, PATH_FMV, PATH_RS, PATH_RASTER };
struct KLine; struct KSec; struct KMod; struct KFmvBase; struct KFmvMod;
struct DevPlan {
	int path;                         // LINE: k_line; SEC_LINE: SECAM raster + chain + k_line<SRC>; SPLIT: raster (+ chain) +
	                                  // modulator; FMV: raster (+ chain) + FM video; RS / RASTER: the two sides of --pixelrate
	const KLine *kl;                  // LINE, SEC_LINE
	const KSec *ks;                   // SEC_LINE: the SECAM raster on the tensor cores; NULL: k_raster_secam
	const KMod *mod;                  // SPLIT, RS
	const KFmvBase *fmv_base;         // FMV
	const KFmvMod *fmv_mod;
	const void *raster;               // k_raster or k_raster_secam where this context launches one
	size_t raster_smem, kl_smem, ks_smem, mod_smem, fmv_smem;   // their dynamic shared memory
	int before, after;                // lines a call rasters before its first and after its last emitted line
	int line_threads;                 // CTA of the split kernels: a thread per 4 samples, whole warps, at least 64
	int kl_threads;                   // CTA of the fused kernels: a warp per tile of 128 samples
	int plane_pitch;                  // k_mod_mma: 0, the planes are the contiguous stream; else bytes per line row (htv_mma_fir.h)
	char kname[192];                  // what htv_line_kernel reports once a render has launched the plan
};

struct htv_dev_t {
	int device;
	const struct htv_tables_t *tab;   // the encoder's tables (they outlive it): plan_kernels again on a new sample type
	DevSwitches sw;
	DevPlan plan;
	htv_dparams_t dp;
	DevTables dt;
	size_t frame_pixels;
	int max_slots;
	void *alloc[HTV_MAX_ALLOCS];
	int nalloc, alloc_failed;
	uint32_t *d_frames;
	int32_t *d_frame_map;
	int frame_map_cap;
	// pinned staging for the frame map: a copy from pageable memory would make cudaMemcpyAsync
	// drain the stream first and stall the host behind the uploads it has just queued
	int32_t *h_map;
	cudaEvent_t ev_map[MAPBUFS];
	int map_i;
	int16_t *d_pcm;
	// VBI overlays: pinned staging + device copies, refilled per launch sequence
	long long *h_ov_line, *d_ov_line;
	int4 *h_ov_meta, *d_ov_meta;
	int16_t *h_ov_add, *d_ov_add;
	cudaEvent_t ev_ov;
	// carries
	int64_t fm_jc;                    // last audio index whose fm_B entry is valid (-1 at start)
	int64_t nic_kc;                   // first frame whose nic_fstart is valid for a restart
	int64_t fm_jr, nic_kr;            // last audio index / NICAM frame with records (dt.seg_rec, dt.nic_rec)
	uint64_t launches;
	int timing;
	cudaEvent_t ev0, ev1;
	cudaStream_t side;                // audio-rate pre-pass + sound descriptors run here, beside the raster
	cudaStream_t side2;               // the NICAM half of the pre-pass (independent of the FM chain until the descriptors)
	cudaEvent_t ev_nic;
	cudaStream_t up;                  // picture / PCM uploads: ahead of the previous chunk's kernels
	cudaEvent_t ev_up, ev_chunk[2];
	cudaStream_t pic;                 // the conversions (k_compose, k_picture), each behind its picture's copy but off the
	cudaEvent_t ev_pic;               // upload stream, so that the next copies do not queue behind the conversions
	cudaEvent_t ev_call;              // the caller's stream at the start of a render call that pulls device pictures or sound
	cudaEvent_t *ev_slot;             // [max_slots] the copy of each slot's last picture is done
	uint8_t *comp_valid;              // [max_slots] the phases of each slot's composite rows that hold its picture (bit p)
	int *vf_conv, vf_nconv;           // filtered store: the composite-store entries converted since the last k_vf_rows
	int pic_pending;                  // conversions were launched that the caller's stream has not waited for yet
	unsigned chunk_i;
	cudaEvent_t ev_in, ev_audio;
	cudaEvent_t ev_kl[2];             // the fused line kernel has read descriptor buffer 0 / 1
	int kl_buf, ahead;                // descriptor buffer of the next call; the sound pre-pass may run ahead of the caller's stream
	cudaStream_t side3;               // ... and so may the frame map and the raster descriptors, on a stream of their own
	cudaEvent_t ev_r2;
	int r2_armed;
	int side_armed;
	int ev_pending;
	void *d_desc_r;                   // raster descriptors [cap + before + after] (x 2 for the fused line kernel): LineS2 for
	                                  // SECAM, LineR2 for PAL / NTSC / mono
	void *d_desc_a2;                  // LineA2[cap + 1] (x 2 for the fused line kernel)
	uint32_t *d_vfx;                  // filtered store: the call's rows of the lines vf_exception lists, [vf_cap][W] x 2 ...
	int *d_vfl;                       // ... and their list, [1 + vf_cap] x 2, beside the raster descriptors
	int vf_cap;
	int desc_cap;                     // lines per call the descriptor buffers hold (desc_reserve)
	int kl_ctas;                      // persistent CTAs of the fused kernels (k_line, k_sec_raster)
	char kname[192];                  // the line kernel(s) the last render launched, with their template arguments (htv_line_kernel)
	SecScratch sec;                   // SECAM scratch (same sub-batch rows as d_comp)
	// the SECAM chain's switches (HTV_SEC, sec_knobs) and what it did since the encoder was created (htv_secam_chain)
	int sec_passes, sec_pred, sec_many, sec_repredict, sec_repredict_min, sec_sub;
	htv_secam_chain_t sec_stats;
	int *d_comp32;                    // int32 composite scratch for the TMA-fed modulator (4 | W, not SECAM)
	uint8_t *d_planes;                // high / low byte planes of the composite stream for k_mod_mma (video filter on)
	size_t plane_stride;
	// --pixelrate: this is the sample-rate side; the raster runs in a second context at the pixel rate
	int rs_I, rs_D, rs_ataps, rs_wp;
	int16_t *d_rs_taps;
	int mod_grid;                     // persistent CTAs of k_mod_tma / k_mod_mma
	int16_t *d_comp;                  // composite scratch, (sub + 3) lines, reused by every sub-batch (stays in L2)
	int16_t *d_compq;                 // SECAM with S-Video: the rows' Q (the subcarrier), beside d_comp; NULL otherwise
	int sub_lines;
	int last_mod_lines;
};

// ---------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------

__device__ __forceinline__ int sat16i(int a) { return(max(-32768, min(32767, a))); }
__device__ __forceinline__ int wrap16i(int a) { return((int) (short) a); }

// audio fetch count up to and including audio-clock sample m (ref video.c:3273-3276)
__host__ __device__ __forceinline__ int64_t fetches_by(int64_t m, int rate)
{
	return((int64_t) (((unsigned long long) (m + 1) * HTV_AUDIO_RATE) / (unsigned long long) rate));
}

// first audio-clock sample at which q fetches have happened
__host__ __device__ __forceinline__ int64_t first_with_fetches(int64_t q, int rate)
{
	if(q <= 0) return(0);
	return((int64_t) (((unsigned long long) q * (unsigned long long) rate + HTV_AUDIO_RATE - 1) / HTV_AUDIO_RATE) - 1);
}

// first audio-clock sample of the segment during which audio index j (>= -1) is in effect
__host__ __device__ __forceinline__ int64_t seg_start(int64_t j, int rate)
{
	return(j < 0 ? 0 : first_with_fetches(j + 1, rate));
}

// volume-scaled source sample (ref video.c:3291-3295); j < 0 -> silence
__device__ __forceinline__ int pcm_vol(const DevTables &dt, int64_t j, int ch, int volume)
{
	if(j < 0) return(0);
	int v = ((int) dt.pcm[((j & (RA - 1)) << 1) + ch] * volume + 128) >> 8;
	return(sat16i(v));
}

__device__ __forceinline__ int pcm_mono(const DevTables &dt, int64_t j, int volume)
{
	// (L + R) / 2 with C truncation toward zero (ref video.c:3314,3319)
	return((pcm_vol(dt, j, 0, volume) + pcm_vol(dt, j, 1, volume)) / 2);
}

// ---------------------------------------------------------------------------
// Audio-rate pre-pass, FM path (ref video.c:3319-3327, fir.c:655-694, 818-870)
// ---------------------------------------------------------------------------

// var/fix inputs of the soft limiter for audio index u: two 65-tap int FIRs of the mono mix. A CTA of 128
// consecutive audio indices stages the 192 mono samples it needs and both tap sets in shared memory.
__global__ void __launch_bounds__(128) k_fm_fir(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int64_t u0, int64_t u1)
{
	__shared__ int sx[128 + HTV_AFIR_N - 1];
	__shared__ int sv[HTV_AFIR_N], sf[HTV_AFIR_N];
	const int tid = threadIdx.x;
	const int64_t ub = u0 + (int64_t) blockIdx.x * 128;
	for(int i = tid; i < 128 + HTV_AFIR_N - 1; i += 128) sx[i] = pcm_mono(dt, ub - (HTV_AFIR_N - 1) + i, dp.volume);   // 0 before the stream
	if(tid < HTV_AFIR_N) { sv[tid] = dt.afir_v[tid]; sf[tid] = dt.afir_f[tid]; }
	__syncthreads();
	const int64_t u = ub + tid;
	if(u > u1) return;
	long long av = 0, af = 0;
	if(u >= 0)
	{
		#pragma unroll 13
		for(int y = 0; y < HTV_AFIR_N; y++)
		{
			const long long x = sx[tid + y];
			av += x * sv[y];
			af += x * sf[y];
		}
		av >>= 15; af >>= 15;
		av = av < INT32_MIN ? INT32_MIN : (av > INT32_MAX ? INT32_MAX : av);
		af = af < INT32_MIN ? INT32_MIN : (af > INT32_MAX ? INT32_MAX : af);
		// hard-limit the fixed path, the variable path is the remainder (fir.c:836-841)
		if(af < -32767) af = -32767; else if(af > 32767) af = 32767;
		av -= af;
	}
	dt.lim_var[u & (RA - 1)] = (int) av;
	dt.lim_fix[u & (RA - 1)] = (int) af;
}

__device__ __forceinline__ int lim_at(const int32_t *ring, int64_t u) { return(u < 0 ? 0 : ring[u & (RA - 1)]); }

// limiter output = modulating sample for audio index j, and its phase increment
__global__ void k_fm_limit(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int64_t j0, int64_t j1)
{
	int64_t j = j0 + (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if(j > j1) return;
	int p = 0;
	if(j >= 0)
	{
		if(!dp.have_lim) p = pcm_mono(dt, j, dp.volume);
		else
		{
			const int level = 32767;
			int64_t t = j - (HTV_LIM_W - 1);                 // the sample leaving the look-ahead window
			int att = 0;
			for(int q = 0; q < HTV_LIM_W; q++)
			{
				int64_t u = t + q - HTV_LIM_W / 2;           // sample examined at call t + q
				int var = lim_at(dt.lim_var, u), fix = lim_at(dt.lim_fix, u);
				int a = abs(var + fix);
				if(a > level)
				{
					a = 32767 - (int) ((unsigned) (level + abs(var) - a) * 32767u) / abs(var);
					int b = (a * dt.lim_shape[HTV_LIM_W - 1 - q]) >> 15;
					if(b > att) att = (short) b;
				}
			}
			int var = lim_at(dt.lim_var, t), fix = lim_at(dt.lim_fix, t);
			int a = fix + (int) (((long long) var * (32767 - att)) >> 15);
			p = a < -level ? -level : (a > level ? level : a);
		}
	}
	dt.fm_p[(j + 1) & (RA - 1)] = (short) p;
	// phase advance over the whole segment during which audio index j is in effect
	const unsigned long long cnt = (unsigned long long) (seg_start(j + 1, dp.rate) - seg_start(j, dp.rate));
	dt.fm_inc[(j + 1) & (RA - 1)] = cnt * dt.fm_ang[p + 32768];
}

// Phase prefix B(j+1) = B(j) + inc(j) over entries jc .. j1 (B(jc) is the carry from the
// previous batch). Two passes: per-block inclusive scans + block totals, then offsets.
#define SCAN_T 256
#define SCAN_PER 8
#define SCAN_BLK (SCAN_T * SCAN_PER)

__global__ void __launch_bounds__(SCAN_T) k_fm_scan_local(const DevTables dt, int64_t jc, int64_t j1)
{
	__shared__ unsigned long long part[SCAN_T];
	const int t = threadIdx.x;
	const int64_t a = jc + (int64_t) blockIdx.x * SCAN_BLK + t * SCAN_PER;
	unsigned long long v[SCAN_PER], sum = 0;
	if(blockIdx.x == 0 && t == 0) dt.scan_carry[0] = dt.fm_B[(jc + 1) & (RA - 1)];
	#pragma unroll
	for(int i = 0; i < SCAN_PER; i++)
	{
		const int64_t j = a + i;
		v[i] = j <= j1 ? dt.fm_inc[(j + 1) & (RA - 1)] : 0ull;
		sum += v[i];
	}
	part[t] = sum;
	__syncthreads();
	for(int o = 1; o < SCAN_T; o <<= 1)
	{
		const unsigned long long add = t >= o ? part[t - o] : 0ull;
		__syncthreads();
		part[t] += add;
		__syncthreads();
	}
	unsigned long long acc = part[t] - sum;                     // exclusive prefix of this thread's chunk
	#pragma unroll
	for(int i = 0; i < SCAN_PER; i++)
	{
		const int64_t j = a + i;
		if(j <= j1) dt.fm_B[(j + 1) & (RA - 1)] = acc;          // local value; k_fm_scan_fix adds the block offset
		acc += v[i];
	}
	if(t == SCAN_T - 1) dt.scan_tot[blockIdx.x] = part[t];
}

// Also the records of k_line's sound feed (dt.seg_rec) for the audio indices past jr, whose B(j) is final here
__global__ void __launch_bounds__(SCAN_T) k_fm_scan_fix(const DevTables dt, int64_t jc, int64_t j1, int64_t jr)
{
	__shared__ unsigned long long off;
	const int t = threadIdx.x;
	if(t == 0)
	{
		unsigned long long o = dt.scan_carry[0];
		for(unsigned int b = 0; b < blockIdx.x; b++) o += dt.scan_tot[b];
		off = o;
		if(blockIdx.x == gridDim.x - 1) dt.fm_B[(j1 + 2) & (RA - 1)] = o + dt.scan_tot[blockIdx.x];   // B(j1 + 1)
	}
	__syncthreads();
	const int64_t a = jc + (int64_t) blockIdx.x * SCAN_BLK + t * SCAN_PER;
	#pragma unroll
	for(int i = 0; i < SCAN_PER; i++)
	{
		const int64_t j = a + i;
		if(j > j1) continue;
		const unsigned long long B = dt.fm_B[(j + 1) & (RA - 1)] + off;
		dt.fm_B[(j + 1) & (RA - 1)] = B;
		if(dt.seg_rec && j > jr)
		{
			const int pi = (int) dt.fm_p[(j + 1) & (RA - 1)] + 32768;
			const unsigned long long ang = dt.fm_ang[pi];
			SegRec r;
			r.ba = make_ulonglong2(j < 0 ? B - ang : B, ang);
			r.rot = dt.fm_rot8[pi];
			r.pad[0] = r.pad[1] = 0.0f;
			dt.seg_rec[(j + 1) & (RA - 1)] = r;
		}
	}
}

// ---------------------------------------------------------------------------
// NICAM-728 frame encoder pre-pass (ref nicam728.c:140-249), one CTA per 1 ms frame
// ---------------------------------------------------------------------------

__constant__ int c_j17[HTV_J17_N] = {
	-1, 0, -1, -1, -1, -1, -1, -1, -1, -1, -2, -2, -3, -3, -3, -3, -5, -5,
	-6, -7, -9, -10, -13, -14, -18, -21, -27, -32, -42, -51, -69, -86, -120,
	-159, -233, -332, -524, -814, -1402, -2372, -4502, 25590, -4502, -2372,
	-1402, -814, -524, -332, -233, -159, -120, -86, -69, -51, -42, -32, -27,
	-21, -18, -14, -13, -10, -9, -7, -6, -5, -5, -3, -3, -3, -3, -2, -2, -1,
	-1, -1, -1, -1, -1, -1, -1, 0, -1
};
// scale-factor code and shift per coding range (ref nicam728.c:59-68)
__constant__ unsigned char c_nic_factor[8] = { 0, 1, 2, 4, 3, 5, 6, 7 };
__constant__ unsigned char c_nic_shift[8]  = { 2, 2, 2, 2, 3, 4, 5, 6 };
__constant__ unsigned char c_nic_step[4]   = { 0, 3, 1, 2 };   // ref nicam728.c:46

// First audio-clock sample of NICAM symbol s: ceil(s * F / D) (ref nicam728.c:301-307, 399-407)
__host__ __device__ __forceinline__ int64_t nic_sym_pos(int64_t s, int F, int D)
{
	return((int64_t) (((unsigned long long) s * (unsigned long long) F + (unsigned long long) D - 1) / (unsigned long long) D));
}

// Which 32-sample audio block frame k carries: the last block completed by the end of
// the scan line in which the frame's first symbol starts (ref video.c:3352-3363 vs
// 3435-3438); -1 = none yet (silence)
__device__ __forceinline__ int64_t nic_block_of(int64_t k, const htv_dparams_t &dp)
{
	if(k < 0) return(-1);
	int64_t p = nic_sym_pos(k * 364, dp.nicam_F, dp.nicam_D);
	int64_t line_end = (p / dp.W + 1) * dp.W - 1;
	return(fetches_by(line_end, dp.rate) / 32 - 1);
}

__global__ void __launch_bounds__(64) k_nicam_frames(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int64_t k0)
{
	__shared__ int64_t blk[4];
	__shared__ int rng[2];
	__shared__ unsigned int bits[23];          // 728 bits, MSB-first within bytes, packed big-endian
	__shared__ unsigned char steps[364];
	const int x = threadIdx.x;                 // sample slot: channel = x & 1, n = x >> 1
	const int64_t k = k0 + blockIdx.x;

	if(x < 4) blk[x] = nic_block_of(k - x, dp);
	if(x < 2) rng[x] = 1;
	if(x < 23) bits[x] = 0;
	__syncthreads();

	// J.17 pre-emphasis over the sequence of encoded blocks; history spans 3 earlier frames: the 32 + 82 samples
	// per channel this frame's filter sees are staged once (index t + 82, t relative to the frame's block)
	__shared__ short spcm[2][32 + HTV_J17_N - 1];
	for(int i = x; i < 2 * (32 + HTV_J17_N - 1); i += 64)
	{
		const int ch = i & 1;
		int t = (i >> 1) - (HTV_J17_N - 1);
		const int f = t < 0 ? (31 - t) >> 5 : 0;                        // how many frames back
		t += f << 5;
		const int64_t b = blk[f];
		spcm[ch][i >> 1] = (short) (b < 0 ? 0 : pcm_vol(dt, b * 32 + t, ch, dp.volume));
	}
	__syncthreads();
	int acc = 0;
	{
		const short *sp = spcm[x & 1] + (x >> 1);
		#pragma unroll
		for(int xi = 0; xi < HTV_J17_N; xi++) acc += (int) sp[xi] * c_j17[xi];
	}
	int d = (short) (acc >> 15);

	// coding range per channel: smallest b in 1..7 with |d| < 2^(b+8) (ref nicam728.c:70-94)
	{
		int s = d < 0 ? ~d : d;
		int need = 32 - __clz(s) - 8;
		need = need < 1 ? 1 : (need > 7 ? 7 : need);
		atomicMax(&rng[x & 1], need);
	}
	__syncthreads();
	{
		const int r = rng[x & 1];
		int v = (d >> c_nic_shift[r]) & 0x3FF;
		v |= (__popc(v >> 4) & 1) << 10;
		if(x < 54) v ^= ((c_nic_factor[r] >> (2 - (x / 2 % 3))) & 1) << 10;
		// 11 bits LSB first into the 16 x 44 interleaver (ref nicam728.c:220-239)
		for(int b = 0; b < 11; b++)
		{
			if((v >> b) & 1)
			{
				int q = x * 11 + b;
				int pos = 24 + 16 * (q % 44) + q / 44;
				atomicOr(&bits[pos >> 5], 0x80000000u >> (pos & 31));
			}
		}
	}
	__syncthreads();
	if(x < 23)
	{
		// header: FAW, C0 (toggles every 8 frames), mode 0, reserve flag 1; then the PRN
		unsigned int w = bits[x], prn = 0;
		if(x == 0) w |= (0x4Eu << 24) | ((((unsigned) (~k >> 3) & 1u) << 7 | (1u << 3)) << 16);
		for(int b = 0; b < 4; b++)
		{
			int byte = x * 4 + b;
			unsigned int pb = (byte >= 1 && byte <= 90) ? dt.nicam_prn[byte - 1] : 0;
			prn |= pb << (24 - 8 * b);
		}
		bits[x] = w ^ prn;
	}
	__syncthreads();
	for(int s = x; s < 364; s += 64)
	{
		int bit = 2 * s;
		unsigned int dibit = (bits[bit >> 5] >> (30 - (bit & 31))) & 3;
		steps[s] = c_nic_step[dibit];
	}
	__syncthreads();
	{
		// inclusive prefix (mod 4) of the 364 steps: 6 symbols per thread, then across the 64 threads
		__shared__ int wsum[2];
		const int64_t s0 = k * 364;
		int loc[6], sum = 0;
		#pragma unroll
		for(int i = 0; i < 6; i++)
		{
			const int s = x * 6 + i;
			sum += s < 364 ? steps[s] : 0;
			loc[i] = sum;
		}
		int inc = sum;
		#pragma unroll
		for(int o = 1; o < 32; o <<= 1)
		{
			const int v = __shfl_up_sync(0xFFFFFFFFu, inc, o);
			if((x & 31) >= o) inc += v;
		}
		if((x & 31) == 31) wsum[x >> 5] = inc;
		__syncthreads();
		const int base = inc - sum + (x >= 32 ? wsum[0] : 0);
		#pragma unroll
		for(int i = 0; i < 6; i++)
		{
			const int s = x * 6 + i;
			if(s < 364) dt.nic_local[(s0 + s) & (RS - 1)] = (unsigned char) ((base + loc[i]) & 3);
		}
		if(x == 63) dt.nic_ftot[k & (RF - 1)] = (unsigned char) ((wsum[0] + inc) & 3);
	}
}

// ---------------------------------------------------------------------------
// Per-line descriptors (one thread per scan line) and the line kernel
// ---------------------------------------------------------------------------

#define SPT 4                         // samples per thread: one 128-bit store of 4 complex int16 samples
#define EXT 32                        // composite samples staged either side of a line for the video filter (>= 25)
#define COFF (EXT + 1)                // composite window index = x + COFF: makes the filter's 128-bit loads aligned
#define UOFF (EXT + 8)                // chroma window index = x + UOFF
#define NIC_CAND 7                    // NICAM symbols that can overlap 4 consecutive samples
#define NIC_TPAD 8                    // zero entries in front of the padded NICAM pulse table
#define MAX_SEGS 6                    // audio samples overlapping one scan line (+1)
#define MAX_SYMS 48                   // NICAM symbols overlapping one scan line
#define MAX_BLKS 48                   // 32-sample blocks of a line (W <= 1536)

// Sound-carrier state of a line for the sound stage (htv_sound.cuh), built by k_line_desc_a2 (one warp per line)
struct __align__(16) LineA2 {
	unsigned long long seg_phase[MAX_SEGS], seg_ang[MAX_SEGS];   // FM phase at the line's sample 0 / per sample, per audio segment
	unsigned long long am_phase0, off_phase0;
	long long m0;                     // audio-clock index of the line's first sample
	int kk0, cc0;
	int seg_x[MAX_SEGS + 2];          // first sample (relative to the line) of each audio segment, INT_MAX behind the last
	int seg_am[MAX_SEGS];
	int nsym, nic_generic;            // nic_generic: some symbol in effect on this line has no pulse-table row
	// per 32-sample block b: the audio segment / NICAM symbol in effect at x = 32 b
	unsigned char fm_blk[MAX_BLKS], nic_blk[MAX_BLKS];
	// per symbol: x = pulse-table index bases, I | Q << 16 (row * sps - first sample + KL_BIAS), y = first sample
	// relative to the line; entry nsym is a sentinel (y = INT_MAX)
	uint2 symb[MAX_SYMS + 1];
	unsigned char symc[MAX_SYMS];     // bit 0: I polarity +, bit 1: Q polarity +
	float2 seg_rot[MAX_SEGS];         // (cos, sin) of 8 FM angle steps of the segment
	int pad[2];
};

// Raster descriptors: what the raster kernels need to know about a scan line, one form per colour system (64 bytes
// each, read as four int4). Blanking and sync come from the line templates (htv_tables.c build_templates): row `tmpl`
// of dt.tmpl_out outside the picture [al, ar), the picture value plus row `tmpl` of dt.tmpl_keep inside it.
// PAL / NTSC / mono (k_line, k_raster)
struct __align__(16) LineR2 {
	int valid;                        // 0: before the stream
	int tmpl;                         // row of the line templates
	int al, ar;                       // active sample range [al, ar), -1 if none
	int pal;                          // 0 no chroma, +1 / -1 V-switch
	int keep;                         // the template's keep part is non-zero somewhere
	// VBI overlay on this line (ref vbidata.c:186-239, wss.c:182-185): I[from, to) = value, then I += add
	int ov_any, ov_from;
	unsigned int clut_off;
	int ov_to, ov_value, ov_add;      // ov_add: row of dt.ov_add, -1 none; ov_from >= ov_to: no replace
	long long row_off;                // pixel offset of the source row in the frame store, -1 = black
	long long pic;                    // k_line: offset of the line's row in the composite store (dt.comp, dt.comp_q)
};
static_assert(sizeof(LineR2) == 64, "LineR2 is read as four int4");

// SECAM (k_sec_raster, k_raster_secam and the chrominance chain, ref video.c:3068-3233)
struct __align__(16) LineS2 {
	int valid;                        // 0: before the stream
	int tmpl;                         // row of the line templates
	int al, ar;                       // active sample range [al, ar), -1 if none
	int keep;                         // the template's keep part is non-zero somewhere
	int sec_proc, sec_dr;             // the line carries a subcarrier; 1: D'r line (uses v), 0: D'b (uses u)
	int sec_prev_kind;                // what the line-average store holds: 0 zeros, 1 black, 2 a picture row
	int sec_prev_comp;                // ... and which component of it: 1 u, 2 v
	int sec_sign;                     // subcarrier phase reset: +1 / -1
	int sec_sr;                       // end of the modulated range (start is burst_left)
	int sec_clear;                    // the line-average store is cleared at this line (line 1 / hline)
	long long row_off;                // pixel offset of the source row in the frame store, -1 = black
	long long sec_prev_row;           // pixel offset of the stored row
};
static_assert(sizeof(LineS2) == 64, "LineS2 is read as four int4");

static_assert(sizeof(LineA2) % 16 == 0, "descriptors are copied as int4");

// the picture slot of 0-based frame f0, -1: the source has no picture (black)
__device__ __forceinline__ int frame_slot(const DevTables &dt, int64_t f0)
{
	const int64_t fi = f0 - dt.frame_map_first;
	return(fi >= 0 && fi < dt.frame_map_len ? dt.frame_map[fi] : -1);
}

// frame / line / picture row of scan line L; L < 0 are the pipeline-fill lines the reference's
// SECAM stage sees before line 1 (frame 1, line 0: an all-black active line, ref video.c:4665-4667)
__device__ __forceinline__ void line_numbers(const htv_dparams_t &dp, const DevTables &dt, int64_t L,
	int &frame, int &line, int &code, long long &row_off)
{
	row_off = -1;
	if(L < 0) { frame = 1; line = 0; code = dt.codes[0]; return; }
	const int64_t f0 = L / dp.lines;
	frame = (int) (f0 + 1);
	line = (int) (L - f0 * dp.lines) + 1;
	code = dt.codes[line];
	const int vy = htv_line_vy(&dp, line);
	if(vy >= 0 && dt.frames)
	{
		const int slot = frame_slot(dt, f0);
		if(slot >= 0) row_off = ((long long) slot * dp.active_lines + vy) * (long long) dp.active_width;
	}
}

// the SECAM fields of line L, whose frame / line / code line_numbers gave
__device__ void line_secam(const htv_dparams_t &dp, const DevTables &dt, int64_t L, int frame, int line, int code, LineS2 &o)
{
	o.sec_proc = (code & (HTV_LC_LEFT_ACTIVE | HTV_LC_RIGHT_ACTIVE)) != 0;
	o.sec_dr = ((frame * dp.lines) + line) & 1;
	o.sec_sign = ((frame * dp.lines) + line) % 3 == 0 ? 1 : -1;
	o.sec_sr = (code & HTV_LC_RIGHT_ACTIVE) ? dp.burst_left + dp.burst_width : dp.half_width;
	o.sec_clear = L >= 0 && (line == 1 || line == dp.hline);
	o.sec_prev_kind = 0; o.sec_prev_comp = 1; o.sec_prev_row = -1;
	// what the vertical-average store holds when this line reads it (ref video.c:3149-3196):
	// the other component of the last processed line, unless a clearing line came in between
	for(int64_t M = L; M >= L - dp.lines; M--)
	{
		int f2, l2, c2; long long r2;
		line_numbers(dp, dt, M, f2, l2, c2, r2);
		if(M >= 0 && (l2 == 1 || l2 == dp.hline)) break;       // cleared at the start of line M
		if(M - 1 < -2) break;                                   // stream start: the store is zeroed
		line_numbers(dp, dt, M - 1, f2, l2, c2, r2);
		if(c2 & (HTV_LC_LEFT_ACTIVE | HTV_LC_RIGHT_ACTIVE))
		{
			o.sec_prev_kind = r2 >= 0 ? 2 : 1;
			o.sec_prev_row = r2;
			o.sec_prev_comp = (((f2 * dp.lines) + l2) & 1) ? 1 : 2;   // a D'r line stores u, a D'b line v
			break;
		}
	}
}

// the VBI overlay on scan line L (dt.ov_line is sorted): m = (replace from, replace to, replace value, row of dt.ov_add
// or -1); false, and m = (0, 0, 0, -1), on a line without one
__device__ __forceinline__ bool line_overlay(const DevTables &dt, int64_t L, int4 &m)
{
	m = make_int4(0, 0, 0, -1);
	if(dt.ov_n <= 0 || L < 0) return(false);
	int lo = 0, hi = dt.ov_n - 1;
	while(lo < hi) { const int mid = (lo + hi) >> 1; if(dt.ov_line[mid] < L) lo = mid + 1; else hi = mid; }
	if(dt.ov_line[lo] != L) return(false);
	m = dt.ov_meta[lo];
	return(true);
}

// the row of the composite store scan line L shows: of its frame's picture at its colour-frame phase, of the black slot
// where the frame has none; the stream-start rows for L <= 0
__device__ __forceinline__ long long comp_row(const htv_dparams_t &dp, const DevTables &dt, int64_t L)
{
	if(L <= 0) return(dt.comp_start + (L < 0 ? 0 : 1));
	const int64_t f0 = L / dp.lines;
	const int slot = frame_slot(dt, f0);
	return(((long long) (slot >= 0 ? slot : dt.comp_black) * dt.comp_phases + f0 % dt.comp_phases) * dp.lines + (L - f0 * dp.lines));
}

// The lines whose filtered row is not the filtered store's: the video filter of line L reads lines L - 1 .. L + 1
// (32-sample halos on the neighbours), which are rows of one (slot, phase) entry of the composite store, without
// overlays, unless L is the first or last line of its frame, reaches the stream-start rows (L <= 1), or an overlay line
// is among them. The one place that decides it (k_line_desc_r lists them, k_vf_rows filters the list).
__device__ __forceinline__ bool vf_exception(const htv_dparams_t &dp, const DevTables &dt, int64_t L)
{
	if(L <= 1) return(true);
	const int line = (int) (L % dp.lines);                        // 0-based
	if(line == 0 || line == dp.lines - 1) return(true);
	if(dt.ov_n <= 0) return(false);
	int lo = 0, hi = dt.ov_n;                                       // the first overlay line >= L - 1 (dt.ov_line is sorted)
	while(lo < hi) { const int mid = (lo + hi) >> 1; if(dt.ov_line[mid] < L - 1) lo = mid + 1; else hi = mid; }
	return(lo < dt.ov_n && dt.ov_line[lo] <= L + 1);
}

// The most lines of a call with `rows` raster descriptors from line line0 - before (line0 >= 0) that vf_exception can
// list: L <= 1 (before + 2 of them at most), the first and last line of every frame the rows touch, and each overlay line
// with its two neighbours
static int vf_list_bound(int rows, int before, int lines, int ov_n)
{
	const int n = before + 2 + 2 * (rows / lines + 2) + 3 * ov_n;
	return(n < rows ? n : rows);
}

// Raster descriptors of lines first .. first + n - 1, entry i <-> line first + i, one thread per line: LineS2 rows for
// SECAM, LineR2 rows for every other colour system. With a filtered store (dt.filt), pic is the line's filtered row,
// in the filtered store or, for the lines vf_exception lists (dt.vf_list, in no particular order), -1 - its index in
// the list, which is its row of dt.vfx.
__global__ void k_line_desc_r(const __grid_constant__ htv_dparams_t dp, const DevTables dt, void *out, int64_t first, int n)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= n) return;
	const int64_t L = first + i;
	int frame, line, code; long long row_off;
	line_numbers(dp, dt, L, frame, line, code, row_off);
	const int left = L >= 0 ? code & HTV_LC_LEFT_ACTIVE : 0, right = L >= 0 ? code & HTV_LC_RIGHT_ACTIVE : 0;
	const int al = left ? dp.active_left : (right ? dp.half_width : -1);
	const int ar = right ? dp.active_left + dp.active_width : (left ? dp.half_width : -1);
	const int tmpl = L < 0 ? dp.lines + 1 : (L == 0 ? dp.lines : line - 1);
	if(dp.colour_mode == HTV_SECAM)
	{
		LineS2 o;
		o.valid = L >= 0; o.tmpl = tmpl; o.al = al; o.ar = ar;
		o.keep = dt.tmpl_keep_any[tmpl];
		o.row_off = row_off;
		line_secam(dp, dt, L, frame, line, code, o);
		reinterpret_cast<LineS2 *>(out)[i] = o;
		return;
	}
	LineR2 o;
	o.valid = L >= 0; o.tmpl = tmpl; o.al = al; o.ar = ar;
	o.keep = dt.tmpl_keep_any[tmpl];
	o.pal = 0;
	o.clut_off = 0;
	if(L >= 0 && (dp.colour_mode == HTV_PAL || dp.colour_mode == HTV_NTSC))
	{
		const int b = (code & HTV_LC_BURST_MASK) >> HTV_LC_BURST_SHIFT;
		o.pal = b == 1 || (b == 2 && (frame & 1) == 0) || (b == 3 && (frame & 1) == 1);
		if(dp.colour_mode == HTV_PAL && o.pal && ((frame + line) & 1)) o.pal = -1;
		o.clut_off = (unsigned int) (((unsigned long long) L * (unsigned long long) dp.W) % dp.clut_width);
	}
	int4 m;
	o.ov_any = line_overlay(dt, L, m);
	o.ov_from = m.x; o.ov_to = m.y; o.ov_value = m.z; o.ov_add = m.w;
	o.row_off = row_off;
	// the composite row: of the frame's picture at its colour-frame phase, of the black slot where the frame has none
	o.pic = -1;
	if(dt.pic_val && al < ar)
	{
		const int row = dt.line_row[line];
		const int slot = row < dp.active_lines ? frame_slot(dt, frame - 1) : -1;
		o.pic = ((long long) (slot >= 0 ? slot : dt.pic_black) * dt.pic_nrows + row) * dp.W;
	}
	if(dt.comp) o.pic = comp_row(dp, dt, L) * dp.W;
	if(dt.filt && vf_exception(dp, dt, L))
	{
		const int k = atomicAdd(dt.vf_list, 1);
		dt.vf_list[1 + k] = i;
		o.pic = -1 - k;
	}
	reinterpret_cast<LineR2 *>(out)[i] = o;
}

// ---------------------------------------------------------------------------
// Sound descriptors (LineA2) for every modulator: ONE WARP per scan line. The closed forms of the sound
// carriers' state at the line's start, spread over the lanes: lane = audio segment, lane = NICAM symbol,
// lane = 32-sample block. 64-bit divisions by run-time constants go through fp64 (exact below 2^52, with
// the exact division behind it).
// ---------------------------------------------------------------------------

// floor(n / d) and the remainder for n < 2^63, 0 < d < 2^31
__device__ __forceinline__ unsigned long long kd_div(unsigned long long n, unsigned d, double inv, unsigned &rem)
{
	if(n >> 52) { const unsigned long long q = n / d; rem = (unsigned) (n - q * d); return(q); }
	long long q = __double2ll_rd(__dmul_rn((double) (long long) n, inv));
	long long r = (long long) n - q * (long long) d;
	if(r < 0) { q--; r += d; }
	else if(r >= (long long) d) { q++; r -= d; }
	rem = (unsigned) r;
	return((unsigned long long) q);
}

// DQPSK state before each frame k0 + 1 .. k1 + 1 - the state before k0 (valid from the previous batch, 0 at the stream
// start) plus the frame totals k0 .. k - 1, mod 4 - and, where k_line's sound feed reads them (dt.nic_rec), the records
// of the symbols of the frames from kr on (ref nicam728.c:342-411). One CTA per frame k0 .. k1.
// A record holds what the line descriptor's phase B (k_line_desc_a2) works out per symbol: its polarity code and the
// pulse-table rows of the 6-symbol patterns of symbols s - 5 .. s, with the spacing code of the 5 gaps between them
// (htv_tables.c); no row at the stream start (s < 5), with more than one gap of the rarer spacing, or without a table.
#define NR_T 384
__global__ void __launch_bounds__(NR_T) k_nicam_rec(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int64_t k0, int64_t k1,
	int64_t kr)
{
	__shared__ int red[NR_T / 32];
	__shared__ long long spos[364 + 5];       // first sample of symbols k 364 - 5 .. k 364 + 363
	__shared__ unsigned char scd[364 + 5];    // and their polarity codes
	const int t = threadIdx.x;
	const int64_t k = k0 + blockIdx.x;
	int sum = 0;
	for(int64_t i = k0 + t; i < k; i += NR_T) sum += dt.nic_ftot[i & (RF - 1)];
	#pragma unroll
	for(int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
	if((t & 31) == 0) red[t >> 5] = sum;
	__syncthreads();
	int fs = k0 == 0 ? 0 : dt.nic_fstart[k0 & (RF - 1)];
	#pragma unroll
	for(int w = 0; w < NR_T / 32; w++) fs += red[w];
	fs &= 3;                                  // the state before frame k
	if(t == 0) dt.nic_fstart[(k + 1) & (RF - 1)] = (unsigned char) ((fs + dt.nic_ftot[k & (RF - 1)]) & 3);
	if(!dt.nic_rec || k < kr) return;

	const unsigned F = (unsigned) dp.nicam_F, D = (unsigned) dp.nicam_D;
	const int64_t sb = k * 364 - 5;
	if(t < 364 + 5)
	{
		const int64_t s = sb + t;
		int cd = 0;
		long long pos = 0;
		if(s >= 0)
		{
			unsigned rem;
			pos = (long long) kd_div((unsigned long long) s * F + D - 1, D, 1.0 / (double) D, rem);
			const int st = t < 5 ? (fs - dt.nic_ftot[(k - 1) & (RF - 1)]) & 3 : fs;     // the state before s's frame
			const int sy = (st + dt.nic_local[s & (RS - 1)]) & 3;
			// ref nicam728.c:47,386-391: _syms = {0,1,3,2}; bit0 -> I polarity, bit1 -> Q polarity
			cd = sy == 2 ? 3 : (sy == 3 ? 2 : sy);
		}
		spos[t] = pos;
		scd[t] = (unsigned char) cd;
	}
	__syncthreads();
	if(t >= 364) return;
	const int i = t + 5;
	const int64_t s = sb + i;
	const int minor_adv = dp.nicam_minor_short ? dp.nicam_sps - 1 : dp.nicam_sps;
	unsigned rec = (unsigned) scd[i] << 18 | 1u << 20;
	if(dp.nicam_lut_ok && s >= 5)
	{
		// bit j of a pattern = the j-th latest symbol (0 = this one); bit j of gaps: the gap ending at symbol s - j is the
		// rarer spacing
		int patI = 0, patQ = 0, gaps = 0;
		#pragma unroll
		for(int j = 0; j < 6; j++)
		{
			patI |= (scd[i - j] & 1) << j;
			patQ |= ((scd[i - j] >> 1) & 1) << j;
			if(j < 5) gaps |= (spos[i - j] - spos[i - j - 1] == minor_adv) << j;
		}
		if(__popc(gaps) <= 1)
		{
			const int gg = gaps ? __ffs(gaps) : 0;                          // which gap (1 = newest) has the rarer spacing
			rec = (unsigned) (gg * 64 + patI) | (unsigned) (gg * 64 + patQ) << 9 | (unsigned) scd[i] << 18;
		}
	}
	dt.nic_rec[s & (RS - 1)] = rec;
}

// A warp takes KD_LINES consecutive lines. Phase A, lane = line: everything that is one value per line or per audio
// segment (the 64-bit divisions live here, once per line instead of once per lane). Phase B, for each of the
// lines in turn, lane = NICAM symbol: positions, DQPSK state, the 6-symbol polarity patterns and spacing
// codes through warp votes, then lane = 32-sample block for the "symbol in effect" table.
#define KD_WARPS 4
#define KD_LINES 8
// PART 1: audio segments, FM / AM / offset phases (needs the FM chain of the pre-pass); PART 2: NICAM symbols (needs the
// NICAM chain). The two halves write disjoint fields and run on the two side streams, each right behind its chain.
template<int PART>
__global__ void __launch_bounds__(32 * KD_WARPS)
k_line_desc_a2(const __grid_constant__ htv_dparams_t dp, const DevTables dt, LineA2 *out, int64_t line0, int nlines)
{
	__shared__ int s_blk[KD_WARPS][MAX_BLKS];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const int lbase = (blockIdx.x * KD_WARPS + wid) * KD_LINES;
	if(lbase >= nlines) return;
	const int W = dp.W;
	const int li = lbase + lane;
	const bool mine = lane < KD_LINES && li < nlines;
	const long long m0 = (line0 + (mine ? li : lbase)) * (long long) W + dp.shift;
	LineA2 &la = out[mine ? li : lbase];
	unsigned rem;

	// ---- phase A: lane = line ------------------------------------------------------------------------
	// NICAM scalars of the lane's line, handed to phase B by shuffles
	int a_ns = 0, a_dq = 0, a_ks0 = 0, a_generic = 0;
	int a_bk[MAX_SEGS - 1];
	unsigned a_r0 = 0;
	long long a_s0 = 0, a_k0 = 0;
	{
		int segx[MAX_SEGS + 2];
		#pragma unroll
		for(int k = 0; k < MAX_SEGS + 2; k++) segx[k] = 0x7FFFFFFF;
		if(PART == 1)
		{
			int kk0;
			kd_div((unsigned long long) m0, 32767u, 1.0 / 32767.0, rem); kk0 = (int) rem;
			if(mine)
			{
				la.m0 = m0; la.kk0 = kk0;
				la.am_phase0 = dp.am_ang * (unsigned long long) m0;
				la.off_phase0 = dp.offset_phase0 + dp.offset_ang * (unsigned long long) (m0 - 32767);
			}
		}
		else if(dp.have_nicam)
		{
			kd_div((unsigned long long) m0, (unsigned) dp.nicam_cc_len, 1.0 / (double) dp.nicam_cc_len, rem);
			if(mine) la.cc0 = (int) rem;
		}
		else if(mine) la.cc0 = 0;
		// audio segments: audio index j is in effect from seg_start(j) up to seg_start(j + 1)
		if(PART == 1 && (dp.have_fm || dp.have_am))
		{
			const double inv_ar = 1.0 / (double) HTV_AUDIO_RATE;
			const long long jf = (long long) kd_div((unsigned long long) (m0 + 1) * HTV_AUDIO_RATE, (unsigned) dp.rate, 1.0 / (double) dp.rate, rem) - 1;
			#pragma unroll
			for(int k = 0; k < MAX_SEGS; k++)
			{
				const long long j = jf + k;
				// seg_start(j) = j < 0 ? 0 : ceil((j + 1) rate / 32000) - 1
				long long st = 0;
				if(j >= 0) st = (long long) kd_div((unsigned long long) (j + 1) * (unsigned long long) dp.rate + HTV_AUDIO_RATE - 1, HTV_AUDIO_RATE, inv_ar, rem) - 1;
				unsigned long long ang = 0, ph = 0;
				float2 rot = make_float2(1.0f, 0.0f);
				int am = 0;
				if(st < m0 + W && (k == 0 || segx[k - 1] != 0x7FFFFFFF))
				{
					segx[k] = (int) max(0ll, st - m0);
					if(dp.have_fm)
					{
						const int pi = (int) dt.fm_p[(j + 1) & (RA - 1)] + 32768;
						ang = dt.fm_ang[pi];
						rot = dt.fm_rot8[pi];
						// phase at relative sample x = B(j) + (m0 + x - st + 1) * ang
						ph = dt.fm_B[(j + 1) & (RA - 1)] + ang * (unsigned long long) (m0 - st + 1);
					}
					if(dp.have_am) am = pcm_mono(dt, j, dp.volume);
				}
				if(mine) { la.seg_ang[k] = ang; la.seg_phase[k] = ph; la.seg_rot[k] = rot; la.seg_am[k] = am; }
			}
		}
		if(PART == 1 && mine)
		{
			#pragma unroll
			for(int k = 0; k < MAX_SEGS + 2; k++) la.seg_x[k] = segx[k];
		}
		// first block (32 samples) in which segment k >= 1 is in effect at the block start; phase B builds fm_blk
		#pragma unroll
		for(int k = 1; k < MAX_SEGS; k++) a_bk[k - 1] = segx[k] == 0x7FFFFFFF ? 0x7FFF : (segx[k] + 31) >> 5;
		if(PART == 2 && dp.have_nicam)
		{
			const unsigned F = (unsigned) dp.nicam_F, D = (unsigned) dp.nicam_D;
			const double inv_f = 1.0 / (double) F;
			// the symbols a sample of this line can see: from 6 before the one in effect at the line's first sample (the pulse
			// spans less than 6 symbol periods, and a pulse-table row needs the 5 predecessors) to the last one starting
			// on the line - at most 32 at any rate (a line is 23.3 symbol periods): one lane each
			const long long seff = (long long) kd_div((unsigned long long) m0 * D, F, inv_f, rem);
			const long long slast = (long long) kd_div((unsigned long long) (m0 + W - 1) * D, F, inv_f, rem);
			a_s0 = max(0ll, seff - 6);
			a_ns = (int) min(32ll, slast - a_s0 + 1);
			// pos(s0 + i) = ceil((s0 + i) F / D) = q0 + ceil((r0 + i F) / D)
			const long long q0 = (long long) kd_div((unsigned long long) a_s0 * F, D, 1.0 / (double) D, a_r0);
			unsigned ks0;
			a_k0 = (long long) kd_div((unsigned long long) a_s0, 364u, 1.0 / 364.0, ks0);
			a_ks0 = (int) ks0;
			a_dq = (int) (q0 - m0);                                     // |q0 - m0| < ntaps + W + a few symbols
			a_generic = !dp.nicam_lut_ok || dp.nicam_sps - 1 < 32 || a_ns < 1 || slast - a_s0 + 1 > 32;
		}
	}
	// ---- phase B: per line, lane = NICAM symbol (ref nicam728.c:342-411), then lane = block / table word ---------
	const unsigned F = (unsigned) dp.nicam_F, D = (unsigned) dp.nicam_D;
	const float inv_d = 1.0f / (float) D;
	const int minor_adv = dp.nicam_minor_short ? dp.nicam_sps - 1 : dp.nicam_sps;
	const int nl = min(KD_LINES, nlines - lbase);
	for(int l = 0; l < nl; l++)
	{
		LineA2 &lb = out[lbase + l];
		if(PART == 1)
		{
		if(dp.have_fm || dp.have_am)
		{
			// segment in effect at x = 32 b = number of segments k >= 1 whose first block is <= b; lane = word of four blocks
			int bk[MAX_SEGS - 1];
			#pragma unroll
			for(int k = 0; k < MAX_SEGS - 1; k++) bk[k] = __shfl_sync(0xFFFFFFFFu, a_bk[k], l);
			if(lane < MAX_BLKS / 4)
			{
				unsigned w = 0;
				#pragma unroll
				for(int e = 0; e < 4; e++)
				{
					int sg = 0;
					#pragma unroll
					for(int k = 0; k < MAX_SEGS - 1; k++) sg += bk[k] <= 4 * lane + e;
					w |= (unsigned) sg << (8 * e);
				}
				reinterpret_cast<unsigned *>(lb.fm_blk)[lane] = w;
			}
		}
		else if(lane < MAX_BLKS / 4) reinterpret_cast<unsigned *>(lb.fm_blk)[lane] = 0;
		continue;
		}
		if(!dp.have_nicam)
		{
			if(lane == 0) { lb.nsym = 0; lb.nic_generic = 0; lb.symb[0] = make_uint2(0u, 0x7FFFFFFFu); }
			continue;
		}
		const int ns = __shfl_sync(0xFFFFFFFFu, a_ns, l);
		const int dq = __shfl_sync(0xFFFFFFFFu, a_dq, l), ks0 = __shfl_sync(0xFFFFFFFFu, a_ks0, l);
		const unsigned r0 = __shfl_sync(0xFFFFFFFFu, a_r0, l);
		const long long s0 = __shfl_sync(0xFFFFFFFFu, a_s0, l), k0 = __shfl_sync(0xFFFFFFFFu, a_k0, l);
		int generic = __shfl_sync(0xFFFFFFFFu, a_generic, l);
		const int i = lane;                                             // window index = listed symbol index
		const bool valid = i < ns;
		// pos(s0 + i) - q0 = ceil((r0 + i F) / D): below 2^19, so one float multiply and a correction divide exactly
		const unsigned num = r0 + (unsigned) i * F + D - 1;
		unsigned p = (unsigned) __float2int_rz((float) num * inv_d);
		{
			const int rr = (int) num - (int) (p * D);
			if(rr < 0) p--; else if(rr >= (int) D) p++;
		}
		const unsigned pprev = __shfl_up_sync(0xFFFFFFFFu, p, 1);
		const bool minor = valid && i > 0 && (int) (p - pprev) == minor_adv;   // the window's first symbol: unknown, never used
		int ks = ks0 + i;
		long long k = k0;
		if(ks >= 364) { ks -= 364; k++; }
		int cd = 0;
		if(valid)
		{
			const int sy = (dt.nic_fstart[k & (RF - 1)] + dt.nic_local[(s0 + i) & (RS - 1)]) & 3;
			// ref nicam728.c:47,386-391: _syms = {0,1,3,2}; bit0 -> I polarity, bit1 -> Q polarity
			cd = sy == 2 ? 3 : (sy == 3 ? 2 : sy);
		}
		const unsigned MI = __ballot_sync(0xFFFFFFFFu, valid && (cd & 1)), MQ = __ballot_sync(0xFFFFFFFFu, valid && (cd & 2));
		const unsigned MG = __ballot_sync(0xFFFFFFFFu, minor);
		for(int b = lane; b < MAX_BLKS; b += 32) s_blk[wid][b] = 0;
		__syncwarp();
		int bad = 0, norow = 0;
		if(valid)
		{
			// bit j of a pattern = the j-th latest symbol (0 = this one): window bits i-5 .. i, reversed
			const unsigned wi = i >= 5 ? (MI >> (i - 5)) & 63u : (MI << (5 - i)) & 63u;
			const unsigned wq = i >= 5 ? (MQ >> (i - 5)) & 63u : (MQ << (5 - i)) & 63u;
			const unsigned wg = i >= 4 ? (MG >> (i - 4)) & 31u : (MG << (4 - i)) & 31u;
			const int patI = (int) (__brev(wi) >> 26), patQ = (int) (__brev(wq) >> 26), gaps = (int) (__brev(wg) >> 27);
			const int sx = dq + (int) p;
			int bI = 0xFFFF, bQ = 0xFFFF;
			// a row needs the 5 predecessors inside the window (and a stream that is 5 symbols old)
			const bool row_ok = dp.nicam_lut_ok && i >= 5 && s0 + i >= 5 && __popc(gaps) <= 1;
			if(row_ok)
			{
				const int gg = gaps ? __ffs(gaps) : 0;                      // which gap (1 = newest) has the rarer spacing
				bI = (gg * 64 + patI) * dp.nicam_sps - sx + 2048;
				bQ = (gg * 64 + patQ) * dp.nicam_sps - sx + 2048;
			}
			lb.symb[i] = make_uint2((unsigned) (bI & 0xFFFF) | ((unsigned) (bQ & 0xFFFF) << 16), (unsigned) sx);
			lb.symc[i] = (unsigned char) cd;
			// the symbol comes into effect at the first block that starts at or behind it
			const int bo = sx <= 0 ? 0 : (sx + 31) >> 5;
			if(bo < MAX_BLKS) atomicMax(&s_blk[wid][bo], i);
			if(i == 0 && sx > 0) bad = 1;
			norow = !row_ok;
		}
		if(lane == 0) lb.symb[ns] = make_uint2(0u, 0x7FFFFFFFu);
		__syncwarp();
		// running maximum over the blocks: blocks without a symbol start keep the previous symbol; block 0 gets the
		// LAST symbol starting at or before x = 0, the one in effect there
		int carry = 0, ib0 = 0;
		for(int b0 = 0; b0 < MAX_BLKS; b0 += 32)
		{
			const int b = b0 + lane;
			int v = b < MAX_BLKS ? s_blk[wid][b] : 0;
			#pragma unroll
			for(int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(0xFFFFFFFFu, v, o); if(lane >= o) v = max(v, u); }
			v = max(v, carry);
			if(b < MAX_BLKS) lb.nic_blk[b] = (unsigned char) v;
			if(b0 == 0) ib0 = __shfl_sync(0xFFFFFFFFu, v, 0);
			carry = __shfl_sync(0xFFFFFFFFu, v, 31);
		}
		// the table path needs a row for every symbol in effect on the line: those from nic_blk[0] on
		if(norow && i >= ib0) bad = 1;
		generic |= __any_sync(0xFFFFFFFFu, bad);
		if(lane == 0) { lb.nsym = ns; lb.nic_generic = generic; }
		__syncwarp();
	}
}

__device__ __forceinline__ int round_away(double v)
{
	// round() (half away from zero) from the round-to-nearest-even conversion
	int r = __double2int_rn(v);
	const double t = __dadd_rn(v, -(double) r);
	r += (t == 0.5 && v > 0.0) ? 1 : 0;
	r -= (t == -0.5 && v < 0.0) ? 1 : 0;
	return(r);
}

template<bool SECAM>
__device__ __forceinline__ void yuv_of(const htv_dparams_t &dp, const double *glut, unsigned int rgb, int &y, int &u, int &v)
{
	// ref video.c:3912-3959, same operation order, no FMA contraction. The reference clamps
	// to [-1, 1] before scaling; clamping the rounded integer to +-32767 is the same thing.
	const double r = glut[(rgb >> 16) & 0xFF], g = glut[(rgb >> 8) & 0xFF], b = glut[rgb & 0xFF];
	double yy = __dadd_rn(__dadd_rn(__dmul_rn(r, dp.rw), __dmul_rn(g, dp.gw)), __dmul_rn(b, dp.bw));
	double uu = __dmul_rn(__dadd_rn(b, -yy), dp.eu);
	double vv = __dmul_rn(__dadd_rn(r, -yy), dp.ev);
	yy = __dmul_rn(__dadd_rn(dp.black_level, __dmul_rn(yy, dp.white_minus_black)), dp.vlevel);
	if(!SECAM)
	{
		uu = __dmul_rn(uu, dp.uv_scale);
		vv = __dmul_rn(vv, dp.uv_scale);
	}
	else
	{
		uu = __ddiv_rn(__dadd_rn(__dadd_rn(uu, 4250000.0), -4328125.0), 1000e3);
		vv = __ddiv_rn(__dadd_rn(__dadd_rn(vv, 4406250.0), -4328125.0), 1000e3);
	}
	y = max(-32767, min(32767, round_away(__dmul_rn(yy, 32767.0))));
	u = max(-32767, min(32767, round_away(__dmul_rn(uu, 32767.0))));
	v = max(-32767, min(32767, round_away(__dmul_rn(vv, 32767.0))));
}

// The reference converts every pixel through a 2^24-entry table built once in vid_init
// (video.c:3905-3960, read at 2975-2992 / 3152-3190). Same here: 8 bytes per colour (134 MB of
// HBM; what a picture actually uses stays in L2), built on the device by the exact fp64 code.
template<bool SECAM>
__global__ void __launch_bounds__(256) k_yuv_lut(const __grid_constant__ htv_dparams_t dp, const double *glut_g, short4 *lut)
{
	__shared__ double glut[256];
	glut[threadIdx.x] = glut_g[threadIdx.x];
	__syncthreads();
	const unsigned int rgb = blockIdx.x * 256u + threadIdx.x;
	int y, u, v;
	yuv_of<SECAM>(dp, glut, rgb, y, u, v);
	lut[rgb] = make_short4((short) y, (short) u, (short) v, 0);
}

__device__ __forceinline__ void yuv_lookup(const DevTables &dt, unsigned int rgb, int &y, int &u, int &v)
{
	const short4 e = __ldg(dt.yuv_lut + rgb);
	y = e.x; u = e.y; v = e.z;
}

// Chroma low-pass for 4 consecutive samples with a compile-time tap count: the window is
// read with aligned 128-bit shared loads and the symmetric taps are folded.
template<int NT>
__device__ __forceinline__ void chroma_fir4(const htv_dparams_t &dp, const int *su, const int *sv, int x0, int cu[4], int cv[4])
{
	constexpr int H = NT / 2;
	static_assert(H <= 8, "window below assumes at most 17 taps");
	int wu[20], wv[20];
	const int4 *pu = reinterpret_cast<const int4 *>(su + x0 + UOFF - 8);
	const int4 *pv = reinterpret_cast<const int4 *>(sv + x0 + UOFF - 8);
	#pragma unroll
	for(int i = 0; i < 5; i++)
	{
		const int4 a = pu[i], b = pv[i];
		wu[4 * i] = a.x; wu[4 * i + 1] = a.y; wu[4 * i + 2] = a.z; wu[4 * i + 3] = a.w;
		wv[4 * i] = b.x; wv[4 * i + 1] = b.y; wv[4 * i + 2] = b.z; wv[4 * i + 3] = b.w;
	}
	#pragma unroll
	for(int k = 0; k < 4; k++)
	{
		int au = wu[k + 8] * dp.chroma_taps[H], av = wv[k + 8] * dp.chroma_taps[H];
		#pragma unroll
		for(int t = 0; t < H; t++)
		{
			au += (wu[k + 8 - H + t] + wu[k + 8 + H - t]) * dp.chroma_taps[t];
			av += (wv[k + 8 - H + t] + wv[k + 8 + H - t]) * dp.chroma_taps[t];
		}
		cu[k] = sat16i(au >> 15);
		cv[k] = sat16i(av >> 15);
	}
}

// A thread's composite values x0 .. x0 + 3 (x0 < W) of launch row blockIdx.x, stored where the split modulators read
// them: the byte planes when `planes` is set (pitched when plane_pitch is), else the int32 stream when `comp32` is, else
// the int16 stream. k_raster and k_resample both store through here, so every layout a plan can select is written.
__device__ __forceinline__ void store_line4(const int (&val)[SPT], int x0, int W, int16_t *comp, int *comp32,
	uint8_t *planes, size_t plane_stride, int plane_pitch)
{
	if(planes && plane_pitch)
	{
		// pitched byte planes (htv_mma_fir.h): one self-contained row per line, the first / last
		// MF_LEAD samples repeated in the halo of the previous / next row of this launch
		uint8_t *rowp = planes + (size_t) blockIdx.x * plane_pitch;
		if(x0 + SPT <= W)
		{
			*reinterpret_cast<unsigned *>(rowp + MF_LEAD + x0) = ((val[0] >> 8) & 0xFF) | (((val[1] >> 8) & 0xFF) << 8) |
				(((val[2] >> 8) & 0xFF) << 16) | ((unsigned) (val[3] >> 8) << 24);
			*reinterpret_cast<unsigned *>(rowp + plane_stride + MF_LEAD + x0) = (val[0] & 0xFF) | ((val[1] & 0xFF) << 8) |
				((val[2] & 0xFF) << 16) | ((unsigned) val[3] << 24);
		}
		const bool head = x0 < MF_LEAD && blockIdx.x > 0, tail = x0 + SPT > W - MF_LEAD && blockIdx.x + 1 < gridDim.x;
		if(head || tail || x0 + SPT > W)
		{
			#pragma unroll
			for(int k = 0; k < SPT; k++)
			{
				const int x = x0 + k;
				if(x >= W) break;
				const uint8_t hi = (uint8_t) ((val[k] >> 8) & 0xFF), lo = (uint8_t) (val[k] & 0xFF);
				if(x0 + SPT > W) { rowp[MF_LEAD + x] = hi; rowp[plane_stride + MF_LEAD + x] = lo; }
				if(head && x < MF_LEAD) { uint8_t *q = rowp - plane_pitch + MF_LEAD + W + x; q[0] = hi; q[plane_stride] = lo; }
				if(tail && x >= W - MF_LEAD) { uint8_t *q = rowp + plane_pitch + (x - (W - MF_LEAD)); q[0] = hi; q[plane_stride] = lo; }
			}
		}
		return;
	}
	if(planes)
	{
		// high / low byte planes for the tensor-core video filter (k_mod_mma): v = 256 hi + lo
		uint8_t *p = planes + (size_t) blockIdx.x * W + x0;
		*reinterpret_cast<unsigned *>(p) = ((val[0] >> 8) & 0xFF) | (((val[1] >> 8) & 0xFF) << 8) |
			(((val[2] >> 8) & 0xFF) << 16) | ((unsigned) (val[3] >> 8) << 24);
		*reinterpret_cast<unsigned *>(p + plane_stride) = (val[0] & 0xFF) | ((val[1] & 0xFF) << 8) |
			((val[2] & 0xFF) << 16) | ((unsigned) val[3] << 24);
		return;
	}
	if(comp32)
	{
		// int32 stream for the TMA-fed modulator (values are int16-wrapped as the reference's buffer is)
		*reinterpret_cast<int4 *>(comp32 + (size_t) blockIdx.x * W + x0) =
			make_int4(wrap16i(val[0]), wrap16i(val[1]), wrap16i(val[2]), wrap16i(val[3]));
		return;
	}
	int16_t *o = comp + (size_t) blockIdx.x * W + x0;
	if((W & 3) == 0)
	{
		int2 pk;
		pk.x = (val[0] & 0xFFFF) | (val[1] << 16);
		pk.y = (val[2] & 0xFFFF) | (val[3] << 16);
		*reinterpret_cast<int2 *>(o) = pk;
	}
	else
	{
		#pragma unroll
		for(int k = 0; k < SPT; k++) if(x0 + k < W) o[k] = (int16_t) val[k];
	}
}

// A thread's line values x0 .. x0 + 3 before the subcarrier (ref video.c:2864-2992): row `tmpl` of the line templates
// outside the picture area [al, ar), the picture's Y plus the template's keep part inside it; U, V inside it, 0 outside.
// rgb: the source row (pixel x at rgb[x - active_left]), NULL: black. k_raster and k_compose raster through here.
__device__ __forceinline__ void raster_pic4(const htv_dparams_t &dp, const DevTables &dt, int tmpl, int al, int ar, bool keep,
	const uint32_t *rgb, int x0, int (&val)[SPT], int (&uu)[SPT], int (&vv)[SPT])
{
	const int W = dp.W, trow = tmpl * W;
	#pragma unroll
	for(int k = 0; k < SPT; k++)
	{
		const int x = x0 + k;
		val[k] = x < W ? __ldg(dt.tmpl_out + trow + x) : 0; uu[k] = 0; vv[k] = 0;
		if(x >= al && x < ar)
		{
			yuv_lookup(dt, rgb ? (__ldg(rgb + (x - dp.active_left)) & 0xFFFFFF) : 0, val[k], uu[k], vv[k]);
			if(keep) val[k] += __ldg(dt.tmpl_keep + trow + x);           // the next line's leading edge
		}
	}
}

// The chroma low-pass of samples x0 .. x0 + 3 from the U, V windows su, sv (index x + UOFF, zero outside the picture)
__device__ __forceinline__ void chroma_lp4(const htv_dparams_t &dp, const int *su, const int *sv, int x0, int (&cu)[SPT], int (&cv)[SPT])
{
	// every tap count a raster up to the kernels' 1536-sample width has (7 at 9 MHz, 17 at 24 MHz); the lower ones only
	// the --pixelrate raster and the split path run
	switch(dp.chroma_ntaps)
	{
	case 1: chroma_fir4<1>(dp, su, sv, x0, cu, cv); break;
	case 3: chroma_fir4<3>(dp, su, sv, x0, cu, cv); break;
	case 5: chroma_fir4<5>(dp, su, sv, x0, cu, cv); break;
	case 7: chroma_fir4<7>(dp, su, sv, x0, cu, cv); break;
	case 9: chroma_fir4<9>(dp, su, sv, x0, cu, cv); break;
	case 11: chroma_fir4<11>(dp, su, sv, x0, cu, cv); break;
	case 13: chroma_fir4<13>(dp, su, sv, x0, cu, cv); break;
	case 15: chroma_fir4<15>(dp, su, sv, x0, cu, cv); break;
	case 17: chroma_fir4<17>(dp, su, sv, x0, cu, cv); break;
	default:                                                            // no chroma low-pass (chroma_ntaps = 0)
		for(int k = 0; k < SPT; k++) { cu[k] = su[x0 + k + UOFF]; cv[k] = sv[x0 + k + UOFF]; }
	}
}

// ---------------------------------------------------------------------------
// Raster kernel: one CTA per scan line, 4 samples per thread -> int16 composite stream
// (ref video.c:2864-3066 _vid_next_line_raster, vbidata.c:186-239). Low register count
// and high occupancy on purpose: the work is fp64 + gathers, i.e. latency bound.
// Launch covers lines first-1 .. first+n (one extra either side for the filter halo);
// line r of the launch lands at comp[r * W ..].
// ---------------------------------------------------------------------------

__global__ void __launch_bounds__(384, 4)
k_raster(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineR2 *lr, int16_t *comp, int *comp32,
	uint8_t *planes, size_t plane_stride, int plane_pitch)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W;
	const int W4 = (W + 3) & ~3;
	const int UW = W4 + 2 * UOFF;
	int *su = reinterpret_cast<int *>(smem_raw);                    // index = x + UOFF
	int *sv = su + UW;
	__shared__ LineR2 li;
	const int tid = threadIdx.x;

	if(tid < 4) reinterpret_cast<int4 *>(&li)[tid] = __ldg(reinterpret_cast<const int4 *>(lr + blockIdx.x) + tid);
	if(tid < 2 * UOFF)
	{
		// U,V outside the line read as zero (the reference filters each line on its own)
		const int j = tid < UOFF ? tid : W4 + tid;
		su[j] = 0; sv[j] = 0;
	}
	__syncthreads();

	const int x0 = tid * SPT;
	int val[SPT];
	if(x0 < W)
	{
		// ---- blanking and sync from the line template, luma, unfiltered U,V ------
		int uu[SPT], vv[SPT];
		raster_pic4(dp, dt, li.tmpl, li.al, li.ar, li.keep, li.row_off >= 0 ? dt.frames + li.row_off : NULL, x0, val, uu, vv);
		if(li.pal)
		{
			*reinterpret_cast<int4 *>(su + x0 + UOFF) = make_int4(uu[0], uu[1], uu[2], uu[3]);
			*reinterpret_cast<int4 *>(sv + x0 + UOFF) = make_int4(vv[0], vv[1], vv[2], vv[3]);
		}
	}
	if(li.pal)
	{
		__syncthreads();
		// ---- chroma low-pass, burst, subcarrier (ref video.c:3011-3040) ------------
		if(x0 < W)
		{
			const int h = dp.chroma_ntaps / 2;
			const bool near_pic = x0 + SPT - 1 + h >= li.al && x0 - h < li.ar;
			const bool near_burst = x0 + SPT - 1 >= dp.burst_left && x0 < dp.burst_left + dp.burst_width;
			if(near_pic || near_burst)
			{
				int cu[SPT] = { 0, 0, 0, 0 }, cv[SPT] = { 0, 0, 0, 0 };
				if(near_pic) chroma_lp4(dp, su, sv, x0, cu, cv);
				#pragma unroll
				for(int k = 0; k < SPT; k++)
				{
					const int x = x0 + k;
					if(x >= W) break;
					if(x >= dp.burst_left && x < dp.burst_left + dp.burst_width)
					{
						const int w = dt.burst_win[x - dp.burst_left];
						cu[k] = (dp.burst_i * w) >> 15;
						cv[k] = (dp.burst_q * w) >> 15;
					}
					const htv_c16_t c = dt.clut[li.clut_off + x];
					val[k] += ((int) c.i * cv[k] * li.pal + (int) c.q * cu[k]) >> 15;
				}
			}
		}
	}
	if(x0 >= W) return;
	if(li.ov_any)
	{
		// VBI stages run on the finished line (ref video.c:4213-4357 register them behind the raster)
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			const int x = x0 + k;
			if(x >= li.ov_from && x < li.ov_to) val[k] = li.ov_value;
			if(li.ov_add >= 0 && x < W) val[k] = wrap16i(val[k]) + dt.ov_add[(size_t) li.ov_add * W + x];
		}
	}
	store_line4(val, x0, W, comp, comp32, planes, plane_stride, plane_pitch);
}

// ---------------------------------------------------------------------------
// Converted picture store of the fused line kernel's PS forms (encoders whose subcarrier does not repeat within 4
// frames): the part of a line that depends on the picture and on the line's place in the frame only - the line
// template, Y, and U / V through the chroma low-pass - converted once per picture when it arrives
// (htv_dev_upload_frame[s]), not on every line that shows it. One CTA per row `blockIdx.x` of picture
// slot `slot0 + blockIdx.y` (slot max_slots, the black slot: from zero RGB), 4 samples per thread, as k_raster's first
// half; the line of the row and its geometry come from the host (htv_tables.c build_pic_rows). What k_line takes from
// here is what k_raster computes up to the burst: dt.pic_val = val[], dt.pic_cuv = (cu, cv) over the whole line.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(384)
k_picture(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int slot0)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W, W4 = (W + 3) & ~3;
	int *su = reinterpret_cast<int *>(smem_raw);                    // index = x + UOFF
	int *sv = su + W4 + 2 * UOFF;
	const int tid = threadIdx.x, row = blockIdx.x, slot = slot0 + blockIdx.y;
	const int4 g = __ldg(dt.pic_rows + row);                        // line, al, ar, keep
	if(g.x == 0) return;                                            // no line shows this row
	const bool black = slot == dt.pic_black;
	if(tid < 2 * UOFF)
	{
		const int j = tid < UOFF ? tid : W4 + tid;
		su[j] = 0; sv[j] = 0;
	}
	const int x0 = tid * SPT;
	const size_t at = ((size_t) slot * dt.pic_nrows + row) * W + x0;
	int val[SPT], uu[SPT], vv[SPT];
	if(x0 < W)
	{
		const uint32_t *rgb = black ? NULL : dt.frames + ((size_t) slot * dp.active_lines + row) * dp.active_width;
		raster_pic4(dp, dt, g.x - 1, g.y, g.z, g.w, rgb, x0, val, uu, vv);
		#pragma unroll
		if((W & 3) == 0)                                            // at is a multiple of 4: one 8-byte store
			*reinterpret_cast<uint2 *>(dt.pic_val + at) = make_uint2((val[0] & 0xFFFF) | (val[1] << 16), (val[2] & 0xFFFF) | (val[3] << 16));
		else for(int k = 0; k < SPT; k++) if(x0 + k < W) dt.pic_val[at + k] = (int16_t) val[k];
		*reinterpret_cast<int4 *>(su + x0 + UOFF) = make_int4(uu[0], uu[1], uu[2], uu[3]);
		*reinterpret_cast<int4 *>(sv + x0 + UOFF) = make_int4(vv[0], vv[1], vv[2], vv[3]);
	}
	if(!dt.pic_cuv) return;
	__syncthreads();
	if(x0 >= W) return;
	int cu[SPT], cv[SPT];
	chroma_lp4(dp, su, sv, x0, cu, cv);
	#pragma unroll
	unsigned w[SPT];
	#pragma unroll
	for(int k = 0; k < SPT; k++) w[k] = ((unsigned) cu[k] & 0xFFFFu) | ((unsigned) cv[k] << 16);
	if((W & 3) == 0) *reinterpret_cast<uint4 *>(dt.pic_cuv + at) = make_uint4(w[0], w[1], w[2], w[3]);
	else for(int k = 0; k < SPT; k++) if(x0 + k < W) dt.pic_cuv[at + k] = w[k];
}

// ---------------------------------------------------------------------------
// Composite store of the fused line kernel: everything of a line that depends on the picture, the line's place in the
// frame and the colour-frame phase only - the line template, Y, U / V through the chroma low-pass, burst and subcarrier
// (ref video.c:2864-3040) - converted once per (picture, phase) the frames that show the picture need
// (htv_dev_set_frame_map), not on every line of every frame. The subcarrier offset (L W mod clut_width), V-switch and
// burst code of line `line` of frame f0 (0-based) depend on f0 mod comp_phases only (htv_tables.c).
// One CTA per line `blockIdx.x + 1` of slot `slot` at phase `phase` (slot max_slots, the black slot: from zero RGB), 4
// samples per thread, as k_raster. start: the two stream-start rows instead (block 0: the lines before the stream, block
// 1: stream line 0, which has templates of their own; neither has a picture area, htv_dev_create checks).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(384)
k_compose(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int slot, int phase, int start)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W, W4 = (W + 3) & ~3;
	int *su = reinterpret_cast<int *>(smem_raw);                    // index = x + UOFF
	int *sv = su + W4 + 2 * UOFF;
	const int tid = threadIdx.x;
	const int line = start ? 1 : blockIdx.x + 1, frame = phase + 1;
	const int code = start && blockIdx.x == 0 ? 0 : dt.codes[line];
	const int left = code & HTV_LC_LEFT_ACTIVE, right = code & HTV_LC_RIGHT_ACTIVE;
	const int al = left ? dp.active_left : (right ? dp.half_width : -1);
	const int ar = right ? dp.active_left + dp.active_width : (left ? dp.half_width : -1);
	const int tmpl = start ? dp.lines + 1 - blockIdx.x : line - 1;
	const int vy = htv_line_vy(&dp, line);
	const uint32_t *rgb = slot == dt.comp_black || vy < 0 ? NULL : dt.frames + ((size_t) slot * dp.active_lines + vy) * dp.active_width;
	// V-switch and subcarrier offset as k_line_desc_r has them for a line of a frame f0 with f0 mod comp_phases = phase
	int pal = 0;
	unsigned clut_off = 0;
	if(code && (dp.colour_mode == HTV_PAL || dp.colour_mode == HTV_NTSC))
	{
		const int b = (code & HTV_LC_BURST_MASK) >> HTV_LC_BURST_SHIFT;
		pal = b == 1 || (b == 2 && (frame & 1) == 0) || (b == 3 && (frame & 1) == 1);
		if(dp.colour_mode == HTV_PAL && pal && ((frame + line) & 1)) pal = -1;
		const unsigned long long cw = dp.clut_width;
		clut_off = (unsigned) (((unsigned long long) phase * ((unsigned long long) dp.lines * W % cw) + (unsigned long long) (line - 1) * W) % cw);
	}
	if(tid < 2 * UOFF)
	{
		const int j = tid < UOFF ? tid : W4 + tid;
		su[j] = 0; sv[j] = 0;
	}
	const int x0 = tid * SPT;
	const size_t at = (start ? (size_t) dt.comp_start + blockIdx.x : ((size_t) slot * dt.comp_phases + phase) * dp.lines + line - 1) * W + x0;
	int val[SPT], uu[SPT], vv[SPT], cq[SPT] = { 0, 0, 0, 0 };
	if(x0 < W)
	{
		raster_pic4(dp, dt, tmpl, al, ar, dt.tmpl_keep_any[tmpl], rgb, x0, val, uu, vv);
		*reinterpret_cast<int4 *>(su + x0 + UOFF) = make_int4(uu[0], uu[1], uu[2], uu[3]);
		*reinterpret_cast<int4 *>(sv + x0 + UOFF) = make_int4(vv[0], vv[1], vv[2], vv[3]);
	}
	if(pal)
	{
		__syncthreads();
		// ---- chroma low-pass (saturating, int16), burst, subcarrier (ref video.c:3011-3040) ----
		if(x0 < W)
		{
			int cu[SPT] = { 0, 0, 0, 0 }, cv[SPT] = { 0, 0, 0, 0 };
			if(al < ar)
			{
				chroma_lp4(dp, su, sv, x0, cu, cv);
				#pragma unroll
				for(int k = 0; k < SPT; k++) { cu[k] = (int) (short) cu[k]; cv[k] = (int) (short) cv[k]; }
			}
			#pragma unroll
			for(int k = 0; k < SPT; k++)
			{
				const int x = x0 + k;
				if(x >= W) break;
				if(x >= dp.burst_left && x < dp.burst_left + dp.burst_width)
				{
					const int w = dt.burst_win[x - dp.burst_left];
					cu[k] = (dp.burst_i * w) >> 15;
					cv[k] = (dp.burst_q * w) >> 15;
				}
				const htv_c16_t c = dt.clut[clut_off + x];
				cq[k] = ((int) c.i * cv[k] * pal + (int) c.q * cu[k]) >> 15;
				if(!dt.comp_q) val[k] += cq[k];
			}
		}
	}
	if(x0 >= W) return;
	if((W & 3) == 0)                                                // at is a multiple of 4: one 8-byte store
	{
		*reinterpret_cast<uint2 *>(dt.comp + at) = make_uint2((val[0] & 0xFFFF) | (val[1] << 16), (val[2] & 0xFFFF) | (val[3] << 16));
		if(dt.comp_q) *reinterpret_cast<uint2 *>(dt.comp_q + at) = make_uint2((cq[0] & 0xFFFF) | (cq[1] << 16), (cq[2] & 0xFFFF) | (cq[3] << 16));
	}
	else for(int k = 0; k < SPT; k++) if(x0 + k < W)
	{
		dt.comp[at + k] = (int16_t) val[k];
		if(dt.comp_q) dt.comp_q[at + k] = (int16_t) cq[k];
	}
}

// ---------------------------------------------------------------------------
// SECAM (ref video.c:3068-3233). Three parts:
//   k_raster_secam  one CTA per line: luma / sync as k_raster, the luma notch FIR, the
//                   line's colour-difference baseband (vertical average with the previous
//                   line) and its 15-tap low-pass - everything that is parallel in x.
//   k_secam_seq     one THREAD per line: the sample-serial tail of the reference - the
//                   double-precision pre-emphasis IIR and the Q31 FM recurrence with the
//                   bell-filter gain - exactly as the reference computes them.
//   cross-line state (IIR state; the two words at chrominance_buffer[W], [W+1] that the
//                   reference's FM loop overruns into and the next line's low-pass reads
//                   back) is resolved by iteration: every line is computed from a guess of
//                   its predecessor's state and recomputed while that guess was wrong. The
//                   chain is contracting, so a handful of passes reaches the fixed point,
//                   which is the sequential result bit for bit.
// ---------------------------------------------------------------------------

// mma.sync.m16n8k32 in its four signedness mixes (htv_mma_fir.h: the byte-split int16 FIR)
#define MMA_I8(NAME, AT, BT) \
__device__ __forceinline__ void NAME(int (&d)[4], const uint4 &a, const uint2 &b) \
{ \
	asm("mma.sync.aligned.m16n8k32.row.col.s32." AT "." BT ".s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};" \
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) \
		: "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b.x), "r"(b.y)); \
}
MMA_I8(mma_ss, "s8", "s8")
MMA_I8(mma_su, "s8", "u8")
MMA_I8(mma_us, "u8", "s8")
MMA_I8(mma_uu, "u8", "u8")

__global__ void __launch_bounds__(384, 3)
k_raster_secam(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineS2 *lr, int16_t *comp, SecScratch ss)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W;
	const int W4 = (W + 3) & ~3;
	const int LW = W4 + 2 * LOFF + 14;
	int *line = reinterpret_cast<int *>(smem_raw);                  // index = x + LOFF
	int *cbin = line + ((LW + 3) & ~3);                             // index = x + 8
	// luma as high / low byte planes for the notch on the tensor cores: byte i = sample i - MF_LEAD, zero outside 0 .. W-1
	const int RBn = mf_row_bytes(W);
	unsigned char *pl = reinterpret_cast<unsigned char *>(cbin + W4 + 32);
	__shared__ LineS2 li;
	const int tid = threadIdx.x;

	if(tid < 4) reinterpret_cast<int4 *>(&li)[tid] = __ldg(reinterpret_cast<const int4 *>(lr + blockIdx.x) + tid);
	for(int i = tid; i < LOFF; i += blockDim.x) { line[i] = 0; line[W4 + LOFF + i] = 0; }
	if(tid < 16) { cbin[tid < 8 ? tid : W4 + tid] = 0; }
	if(dt.notch_atab)
	{
		for(int i = tid; i < MF_LEAD / 4; i += blockDim.x) { reinterpret_cast<unsigned *>(pl)[i] = 0; reinterpret_cast<unsigned *>(pl + RBn)[i] = 0; }
		for(int i = (MF_LEAD + W4) / 4 + tid; i < RBn / 4; i += blockDim.x) { reinterpret_cast<unsigned *>(pl)[i] = 0; reinterpret_cast<unsigned *>(pl + RBn)[i] = 0; }
	}
	__syncthreads();

	const int x0 = tid * SPT;
	const int cur = li.sec_dr ? 2 : 1;                              // 1: u, 2: v
	if(x0 < W4)
	{
		int val[SPT], cbv[SPT];
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			const int x = x0 + k;
			val[k] = 0;
			cbv[k] = cur == 1 ? dp.black_u : dp.black_v;
			int y = 0, u = 0, v = 0;
			const bool inpic = x >= dp.active_left && x < dp.active_left + dp.active_width;
			if((x >= li.al && x < li.ar) || (li.sec_proc && inpic))
			{
				const unsigned int rgb = li.row_off >= 0 ? (__ldg(dt.frames + li.row_off + (x - dp.active_left)) & 0xFFFFFF) : 0;
				yuv_lookup(dt, rgb, y, u, v);
			}
			if(x >= li.al && x < li.ar) val[k] = y;
			if(li.sec_proc && inpic)
			{
				// average with what the previous line left in the store (C division: toward zero)
				int st = 0;
				if(li.sec_prev_kind == 1) st = li.sec_prev_comp == 1 ? dp.black_u : dp.black_v;
				else if(li.sec_prev_kind == 2)
				{
					int y2, u2, v2;
					const unsigned int rgb2 = __ldg(dt.frames + li.sec_prev_row + (x - dp.active_left)) & 0xFFFFFF;
					yuv_lookup(dt, rgb2, y2, u2, v2);
					st = li.sec_prev_comp == 1 ? u2 : v2;
				}
				cbv[k] = ((cur == 1 ? u : v) + st) / 2;
			}
		}
		// blanking and sync from the line template (the samples from W to W4 are zero)
		const int trow = li.tmpl * W;
		unsigned ph4 = 0, pl4 = 0;
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			const int x = x0 + k;
			int lv = 0;
			if(x < W)
			{
				const bool act = x >= li.al && x < li.ar;
				lv = act ? val[k] : __ldg(dt.tmpl_out + trow + x);
				if(act && li.keep) lv = wrap16i(lv + __ldg(dt.tmpl_keep + trow + x));
			}
			line[x + LOFF] = lv;
			cbin[x + 8] = x < W ? cbv[k] : 0;
			// the notch reads samples left of the picture as zero (ref fir.c:357-375)
			const int nv = x >= dp.active_left ? lv : 0;
			ph4 |= ((unsigned) (nv >> 8) & 0xFFu) << (8 * k);
			pl4 |= ((unsigned) nv & 0xFFu) << (8 * k);
		}
		if(dt.notch_atab && li.sec_proc)
		{
			*reinterpret_cast<unsigned *>(pl + MF_LEAD + x0) = ph4;
			*reinterpret_cast<unsigned *>(pl + RBn + MF_LEAD + x0) = pl4;
		}
	}
	__syncthreads();
	if(dt.notch_atab && li.sec_proc)
	{
		// luma notch over the picture region (ref video.c:3082-3090, fir.c:304-355): the 51-tap FIR as the byte-split
		// int8 contraction of htv_mma_fir.h, one tile of 128 samples per warp; results replace the line's samples
		const int a0 = dp.active_left, a1 = dp.active_left + dp.active_width;
		const int lane = tid & 31;
		const uint4 *at = reinterpret_cast<const uint4 *>(dt.notch_atab);
		for(int w = tid >> 5; w < mf_tiles(W); w += blockDim.x >> 5)
		{
			if(MF_TILE * w >= a1 || MF_TILE * (w + 1) <= a0) continue;
			const unsigned char *ph = pl + mf_b_offset(w, 0, lane), *plo = ph + RBn;
			int hh[4] = { 0, 0, 0, 0 }, mid[4] = { 0, 0, 0, 0 }, ll[4] = { 0, 0, 0, 0 };
			#pragma unroll
			for(int s = 0; s < MF_KSTEPS; s++)
			{
				const uint2 xh = *reinterpret_cast<const uint2 *>(ph + 32 * s);
				const uint2 xl = *reinterpret_cast<const uint2 *>(plo + 32 * s);
				const uint4 ah = __ldg(at + (s * 2 + 0) * 32 + lane), al = __ldg(at + (s * 2 + 1) * 32 + lane);
				mma_ss(hh, ah, xh); mma_su(mid, ah, xl); mma_us(mid, al, xh); mma_uu(ll, al, xl);
			}
			#pragma unroll
			for(int ci = 0; ci < 4; ci++)
			{
				const int x = mf_out_x(w, lane, ci);
				if(x >= a0 && x < a1) line[x + LOFF] = sat16i(mf_combine(hh[ci], mid[ci], ll[ci]) >> 15);
			}
		}
		__syncthreads();
	}
	if(x0 >= W) return;

	int outv[SPT];
	#pragma unroll
	for(int k = 0; k < SPT; k++) outv[k] = line[x0 + k + LOFF];
	if(li.sec_proc)
	{
		// without the tensor-core operand (never on the shipped path): the scalar notch
		const int a0 = dp.active_left, a1 = dp.active_left + dp.active_width;
		if(!dt.notch_atab && x0 + SPT - 1 >= a0 && x0 < a1)
		{
			if(dp.secam_pad)
			{
				// symmetric taps (checked on the host): the window of 4 outputs in registers, taps folded pairwise
				int c[56];
				const int4 *pc = reinterpret_cast<const int4 *>(line + x0 - 25 + LOFF);
				#pragma unroll
				for(int i = 0; i < 14; i++)
				{
					const int4 a = pc[i];
					c[4 * i] = a.x; c[4 * i + 1] = a.y; c[4 * i + 2] = a.z; c[4 * i + 3] = a.w;
				}
				#pragma unroll
				for(int i = 0; i < 56; i++) if(x0 - 25 + i < a0) c[i] = 0;
				#pragma unroll
				for(int k = 0; k < SPT; k++)
				{
					int acc = c[k + 25] * dp.secam_notch[25];
					#pragma unroll
					for(int y = 0; y < 25; y++) acc += (c[k + y] + c[k + 50 - y]) * dp.secam_notch[y];
					if(x0 + k >= a0 && x0 + k < a1) outv[k] = sat16i(acc >> 15);
				}
			}
			else
			{
				#pragma unroll
				for(int k = 0; k < SPT; k++)
				{
					const int x = x0 + k;
					if(x < a0 || x >= a1) continue;
					int acc = 0;
					for(int t = 0; t < 51; t++)
					{
						const int j = x - 25 + t;
						acc += (j >= a0 ? line[j + LOFF] : 0) * dp.secam_notch[t];
					}
					outv[k] = sat16i(acc >> 15);
				}
			}
		}
		// 15-tap low-pass of the colour-difference baseband; the two aliased words past the
		// end of the line are added by the chain (sec_tail), so the last 7 outputs are kept as raw sums;
		// cbT is the chain's transposed layout ([group of 8][row][8])
		const size_t row = (size_t) blockIdx.x;
		int cbo[SPT];
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			const int x = x0 + k;
			cbo[k] = 0;
			if(x >= W) break;
			int acc = 0;
			#pragma unroll
			for(int t = 0; t < 15; t++) acc += cbin[x - 7 + t + 8] * dp.secam_lpf[t];
			cbo[k] = sat16i(acc >> 15);
			if(x >= W - 7) ss.tail[row * SEC_TAIL + (x - (W - 7))] = acc;
		}
		// 4 samples = half a group of the transposed layout
		if(x0 < W) *reinterpret_cast<int2 *>(ss.cbT + ((((size_t) (x0 >> 3) * ss.rows + row) << 3) + (x0 & 7))) =
			make_int2((cbo[0] & 0xFFFF) | (cbo[1] << 16), (cbo[2] & 0xFFFF) | (cbo[3] << 16));
	}
	const size_t o = (size_t) blockIdx.x * W + x0;
	#pragma unroll
	for(int k = 0; k < SPT; k++)
	{
		if(x0 + k < W) comp[o + k] = (int16_t) outv[k];
	}
}

#include "htv_secam.cuh"

// SECAM: the VBI stages sit behind the SECAM stage (ref video.c:4211-4357), so an overlay line is
// folded in once k_sec_out has added the line's subcarrier to the composite row: replace / add in place. One CTA per row
// (row 0 is scan line line_r0), a handful of rows per frame do work.
__global__ void __launch_bounds__(256) k_overlay_secam(const __grid_constant__ htv_dparams_t dp, const DevTables dt, int64_t line_r0, int16_t *comp)
{
	int4 m;
	if(!line_overlay(dt, line_r0 + blockIdx.x, m)) return;
	const int W = dp.W;
	const size_t o = (size_t) blockIdx.x * W;
	for(int x = threadIdx.x; x < W; x += blockDim.x)
	{
		int v = comp[o + x];
		if(x >= m.x && x < m.y) v = m.z;
		if(m.w >= 0) v += dt.ov_add[(size_t) m.w * W + x];
		comp[o + x] = (int16_t) v;
	}
}

// ---------------------------------------------------------------------------
// Modulator kernel: one CTA per scan line, 4 samples per thread. Stages the line's
// composite samples (+-32 from the contiguous stream, so neighbours need no special
// case) in shared memory, applies the video filter as a centred 51-tap FIR (ref
// video.c:3235-3248, fir.c:304-355/564-615), adds the sound carriers (ref
// video.c:3261-3450, nicam728.c:342-411), the optional mixers (ref video.c:3466-3515)
// and writes int16 IQ with 128-bit streaming stores.
// ---------------------------------------------------------------------------

#include "htv_sound.cuh"

// Mixers after the modulation (htv_sound.cuh), the channel combiner and the store of 4 consecutive samples.
// TY: the output has another sample type than int16 (dp.sample_type, htv_sample_type.h). The kernels that share this store
// take it as a template argument, so that their int16 instantiations compile as if the conversion did not exist.
template<bool TY>
__device__ __forceinline__ void mod_store(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	int x0, int row, int (&oi)[SPT], int (&oq)[SPT], int16_t *out, const int16_t *acc)
{
	const int W = dp.W;
	kl_mix<-1, 1>(dp, dt, la, x0, oi, oq);

	// ---- store (ref rf_file.c:97-116, 226-233 layout) ------------------------
	// `acc` (same layout as `out`, may alias it): the stream to add this one into, int16 wrap per
	// component - ref _vid_passthru_process video.c:3536-3539, the channel combiner.
	const size_t lbase = (size_t) row * (size_t) W;
	if constexpr(TY)
	{
		// another sample type: the int16 sum, then the conversion, one sample at a time; `acc` is int16 in the output
		// layout, never `out` itself (htv_render_add refuses other types)
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			if(x0 + k >= W) continue;
			const size_t s = lbase + x0 + k;
			if(dp.complex_out) htv_st_put2(out, s, dp.sample_type, wrap16i(oi[k] + (acc ? acc[2 * s] : 0)), wrap16i(oq[k] + (acc ? acc[2 * s + 1] : 0)));
			else htv_st_put(out, s, dp.sample_type, wrap16i(oi[k] + (acc ? acc[s] : 0)));
		}
		return;
	}
	if(dp.complex_out)
	{
		int16_t *o = out + (lbase + x0) * 2;
		if((W & 3) == 0)
		{
			int4 pk;
			pk.x = (oi[0] & 0xFFFF) | (oq[0] << 16);
			pk.y = (oi[1] & 0xFFFF) | (oq[1] << 16);
			pk.z = (oi[2] & 0xFFFF) | (oq[2] << 16);
			pk.w = (oi[3] & 0xFFFF) | (oq[3] << 16);
			if(acc)
			{
				const int4 a = __ldcs(reinterpret_cast<const int4 *>(acc + (lbase + x0) * 2));
				pk.x = __vadd2(pk.x, a.x); pk.y = __vadd2(pk.y, a.y); pk.z = __vadd2(pk.z, a.z); pk.w = __vadd2(pk.w, a.w);
			}
			__stcs(reinterpret_cast<int4 *>(o), pk);
		}
		else
		{
			#pragma unroll
			for(int k = 0; k < SPT; k++)
			{
				if(x0 + k < W)
				{
					unsigned v = (oi[k] & 0xFFFF) | (oq[k] << 16);
					if(acc) v = __vadd2(v, __ldcs(reinterpret_cast<const unsigned *>(acc + (lbase + x0) * 2) + k));
					__stcs(reinterpret_cast<unsigned *>(o) + k, v);
				}
			}
		}
	}
	else
	{
		int16_t *o = out + lbase + x0;
		if((W & 3) == 0)
		{
			int2 pk;
			pk.x = (oi[0] & 0xFFFF) | (oi[1] << 16);
			pk.y = (oi[2] & 0xFFFF) | (oi[3] << 16);
			if(acc)
			{
				const int2 a = __ldcs(reinterpret_cast<const int2 *>(acc + lbase + x0));
				pk.x = __vadd2(pk.x, a.x); pk.y = __vadd2(pk.y, a.y);
			}
			__stcs(reinterpret_cast<int2 *>(o), pk);
		}
		else
		{
			#pragma unroll
			for(int k = 0; k < SPT; k++) if(x0 + k < W) o[k] = (int16_t) (oi[k] + (acc ? acc[lbase + x0 + k] : 0));
		}
	}
}

// Everything k_mod does for 4 consecutive samples once the composite window is in shared
// memory. cwin[j] = composite sample x0 - 25 - CSKEW + j (16-byte aligned).
template<int CSKEW, bool TY>
__device__ __forceinline__ void mod_body(const htv_dparams_t &dp, const DevTables &dt, const LineA2 *la,
	const int *cwin, const short *ntp, int x0, int row, int16_t *out, const int16_t *acc)
{
	const int W = dp.W;
	int oi[SPT], oq[SPT];
	if(dp.vf_type)
	{
		// c[j] = composite sample x0 - 25 + j
		int c[(SPT + 2 * HALO + 2 + CSKEW + 3) / 4 * 4];
		const int4 *pc = reinterpret_cast<const int4 *>(cwin);
		#pragma unroll
		for(int i = 0; i < (SPT + 2 * HALO + 2 + CSKEW + 3) / 4; i++)
		{
			const int4 a = pc[i];
			c[4 * i] = a.x; c[4 * i + 1] = a.y; c[4 * i + 2] = a.z; c[4 * i + 3] = a.w;
		}
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			int ai = c[k + HALO + CSKEW] * dp.vf_i[HALO], aq = 0;
			// VSB: I taps symmetric, Q taps antisymmetric (complex band-pass of a real low-pass)
			#pragma unroll
			for(int y = 0; y < HALO; y++)
			{
				ai += (c[k + y + CSKEW] + c[k + 2 * HALO - y + CSKEW]) * dp.vf_i[y];
				aq += (c[k + y + CSKEW] - c[k + 2 * HALO - y + CSKEW]) * dp.vf_q[y];
			}
			oi[k] = sat16i(ai >> 15);
			oq[k] = sat16i(aq >> 15);                               // vf_q is all zero for the real low-pass
		}
	}
	else
	{
		#pragma unroll
		for(int k = 0; k < SPT; k++) { oi[k] = cwin[k + HALO + CSKEW]; oq[k] = 0; }
	}

	kl_sound<-1, 1>(dp, dt, la, ntp, x0, oi, oq);
	mod_store<TY>(dp, dt, la, x0, row, oi, oq, out, acc);
}


// ---------------------------------------------------------------------------
// FM video (ref _vid_fmmod_process video.c:3452-3464, _fm_modulator 2299-2335; modes pal-fm,
// ntsc-fm, secam-fm). The reference multiplies a Q31 phasor, once per output sample, by the LUT
// entry the sample's baseband value selects - a recurrence over the whole stream. Closed form,
// as for the sound carriers: phase(n) = sum over samples <= n of the rotation each LUT entry
// actually applies (dt.fmv_ang, 0.64 turns), amplitude from the renormalisation counter. Three
// launches per sub-batch:
//   k_fmv_base  one CTA per line: pre-emphasis FIR (optional, 67/71 taps, asymmetric) over the
//               composite stream + sound carriers -> baseband int16 (kept in L2) and the line's
//               total rotation;
//   k_fmv_scan  one CTA: exclusive prefix of the line totals on top of the carried phase;
//   k_fmv_mod   one CTA per line: per-sample prefix inside the line, sin/cos, level, then the
//               common post stage (IQ swap, offset mixer, combiner, 128-bit stores).
// With a pre-emphasis filter the reference's modulator also integrates the pipeline's fill line
// (the filter output for the line before the stream); that row is computed and scanned like
// any other and simply not stored (out_row0 = -1).
// ---------------------------------------------------------------------------

#define FOFF 40                       // baseband window index = x + FOFF (>= 35 = 71 / 2)

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long *sm)
{
	#pragma unroll
	for(int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
	const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	if(lane == 0) sm[w] = v;
	__syncthreads();
	if(w == 0)
	{
		v = lane < (int) ((blockDim.x + 31) >> 5) ? sm[lane] : 0;
		#pragma unroll
		for(int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
	}
	return(v);                                                      // valid in thread 0
}

template<int NT>
__global__ void __launch_bounds__(384)
k_fmv_base(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineA2 *lap, const int16_t *comp, int pre)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W;
	const int W4 = (W + 3) & ~3;
	const int CW = W4 + 2 * FOFF;
	int *cw = reinterpret_cast<int *>(smem_raw);                    // index = x + FOFF
	short *ntp = reinterpret_cast<short *>(cw + CW);
	__shared__ LineA2 la;
	__shared__ unsigned long long red[12];
	const int tid = threadIdx.x;

	{
		const int4 *sa = reinterpret_cast<const int4 *>(lap + blockIdx.x);
		int4 *da = reinterpret_cast<int4 *>(&la);
		for(int i = tid; i < (int) (sizeof(LineA2) / 16); i += blockDim.x) da[i] = __ldg(sa + i);
	}
	if(dp.have_nicam)
	{
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	{
		// the launch's composite stream starts one line early: row b begins at (b + 1) * W - or at
		// b * W when row 0 is the pipeline's fill line (`pre`), whose history is zero
		const size_t r = (size_t) blockIdx.x + 1 - pre;
		const int16_t *cs = comp + r * W;
		const bool first = pre && blockIdx.x == 0;
		for(int i = tid; i < CW; i += blockDim.x)
		{
			const int x = i - FOFF;
			cw[i] = first && x < 0 ? 0 : __ldg(cs + x);
		}
	}
	__syncthreads();

	const int x0 = tid * SPT;
	unsigned long long rot = 0;
	if(x0 < W)
	{
		int oi[SPT], oq[SPT];
		if(NT > 0)
		{
			// out[x] = sat16(sum_y win[x - NT/2 + y] * taps[y] >> 15), ref fir.c:304-355 as a centred FIR
			int a0 = 0, a1 = 0, a2 = 0, a3 = 0;
			const int *w = cw + x0 - NT / 2 + FOFF;
			int w0 = w[0], w1 = w[1], w2 = w[2];
			#pragma unroll
			for(int y = 0; y < NT; y++)
			{
				const int w3 = w[y + 3], t = dp.fmv_taps[y];
				a0 += w0 * t; a1 += w1 * t; a2 += w2 * t; a3 += w3 * t;
				w0 = w1; w1 = w2; w2 = w3;
			}
			oi[0] = sat16i(a0 >> 15); oi[1] = sat16i(a1 >> 15); oi[2] = sat16i(a2 >> 15); oi[3] = sat16i(a3 >> 15);
		}
		else
		{
			#pragma unroll
			for(int k = 0; k < SPT; k++) oi[k] = cw[x0 + k + FOFF];
		}
		#pragma unroll
		for(int k = 0; k < SPT; k++) oq[k] = 0;
		kl_sound<-1, 1, true>(dp, dt, &la, ntp, x0, oi, oq);         // only the I sum modulates (ref video.c:3460)
		int16_t *b = dt.fmv_base + (size_t) blockIdx.x * W + x0;
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			if(x0 + k < W)
			{
				const int v = wrap16i(oi[k]);
				b[k] = (int16_t) v;
				rot += __ldg(dt.fmv_ang + v + 32768);
			}
		}
	}
	rot = block_sum_u64(rot, red);
	if(tid == 0) dt.fmv_tot[blockIdx.x] = rot;
}

__global__ void __launch_bounds__(1024) k_fmv_scan(const DevTables dt, int nrows)
{
	__shared__ unsigned long long part[1024];
	const int tid = threadIdx.x;
	const int per = (nrows + 1023) / 1024;
	const int r0 = tid * per, r1 = min(nrows, r0 + per);
	unsigned long long sum = 0;
	for(int r = r0; r < r1; r++) sum += dt.fmv_tot[r];
	part[tid] = sum;
	__syncthreads();
	for(int o = 1; o < 1024; o <<= 1)
	{
		const unsigned long long v = tid >= o ? part[tid - o] : 0;
		__syncthreads();
		part[tid] += v;
		__syncthreads();
	}
	unsigned long long run = *dt.fmv_carry + part[tid] - sum;      // exclusive
	for(int r = r0; r < r1; r++) { dt.fmv_rowbase[r] = run; run += dt.fmv_tot[r]; }
	__syncthreads();
	if(tid == 1023) *dt.fmv_carry += part[1023];
}

template<bool TY>
__global__ void __launch_bounds__(384)
k_fmv_mod(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineA2 *lap, int16_t *out,
	const int16_t *acc, int acc_rows, int out_row0)
{
	__shared__ LineA2 la;
	__shared__ unsigned long long wsum[12];
	const int W = dp.W, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	{
		const int4 *sa = reinterpret_cast<const int4 *>(lap + blockIdx.x);
		int4 *da = reinterpret_cast<int4 *>(&la);
		for(int i = tid; i < (int) (sizeof(LineA2) / 16); i += blockDim.x) da[i] = __ldg(sa + i);
	}
	const int x0 = tid * SPT;
	unsigned long long p[SPT];
	unsigned long long run = 0;
	{
		const int16_t *b = dt.fmv_base + (size_t) blockIdx.x * W + x0;
		#pragma unroll
		for(int k = 0; k < SPT; k++)
		{
			if(x0 + k < W) run += __ldg(dt.fmv_ang + (int) b[k] + 32768);
			p[k] = run;                                             // inclusive inside the thread
		}
	}
	// exclusive prefix of the thread totals across the CTA
	unsigned long long inc = run;
	#pragma unroll
	for(int o = 1; o < 32; o <<= 1)
	{
		const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, inc, o);
		if(lane >= o) inc += v;
	}
	if(lane == 31) wsum[wid] = inc;
	__syncthreads();
	unsigned long long before = dt.fmv_rowbase[blockIdx.x] + inc - run;
	for(int w = 0; w < wid; w++) before += wsum[w];

	const int row = (int) blockIdx.x + out_row0;
	if(x0 >= W || row < 0) return;
	int oi[SPT], oq[SPT];
	int kk = la.kk0 + x0; if(kk >= 32767) kk -= 32767;
	#pragma unroll
	for(int k = 0; k < SPT; k++, kk++)
	{
		if(kk >= 32767) kk -= 32767;
		// amplitude of the Q31 phasor kk+1 multiplications after a renormalisation (as the sound carriers)
		const float amp = 32767.99998f - (float) (kk + 1) * 1.52587890625e-5f;
		const unsigned long long ph = before + p[k];
		float sn, cs;
		__sincosf((float) (int) (ph >> 32) * 1.4629180792671596e-9f, &sn, &cs);       // pi / 2^31
		oi[k] = (min((int) floorf(amp * cs), 32767) * dp.fmv_level) >> 15;    // pi >> 16 <= 32767
		oq[k] = (min((int) floorf(amp * sn), 32767) * dp.fmv_level) >> 15;
	}
	mod_store<TY>(dp, dt, &la, x0, row, oi, oq, out, row < acc_rows ? acc : NULL);
}

template<int MAXT, int MINB, bool TY = false>
__global__ void __launch_bounds__(MAXT, MINB)
k_mod(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineA2 *lap, const int16_t *comp, int16_t *out,
	const int16_t *acc, int acc_rows)
{
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int W = dp.W;
	const int W4 = (W + 3) & ~3;
	const int CW = W4 + 2 * EXT + 16;
	int *cw = reinterpret_cast<int *>(smem_raw);                    // index = x + COFF
	short *ntp = reinterpret_cast<short *>(cw + CW);                // padded NICAM pulse table
	__shared__ LineA2 la;
	const int tid = threadIdx.x;

	{
		const int4 *sa = reinterpret_cast<const int4 *>(lap + blockIdx.x);
		int4 *da = reinterpret_cast<int4 *>(&la);
		for(int i = tid; i < (int) (sizeof(LineA2) / 16); i += blockDim.x) da[i] = __ldg(sa + i);
	}
	if(dp.have_nicam)
	{
		// the zero-padded pulse table (8 zeros, the pulse, zeros) is prepared on the host
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	{
		// the launch's composite stream starts one line early: this line begins at (b + 1) * W
		const int16_t *cs = comp + ((size_t) blockIdx.x + 1) * W;
		const int nquads = (W4 + 2 * EXT) / 4;
		for(int q = tid; q < nquads; q += blockDim.x)
		{
			const int xe0 = q * 4 - EXT;
			int v[4];
			if((W & 3) == 0)
			{
				const int2 p = __ldg(reinterpret_cast<const int2 *>(cs + xe0));
				v[0] = (int) (short) p.x; v[1] = p.x >> 16; v[2] = (int) (short) p.y; v[3] = p.y >> 16;
			}
			else
			{
				#pragma unroll
				for(int k = 0; k < 4; k++) v[k] = __ldg(cs + xe0 + k);
			}
			#pragma unroll
			for(int k = 0; k < 4; k++) cw[xe0 + k + COFF] = v[k];
		}
	}
	__syncthreads();

	const int x0 = tid * SPT;
	if(x0 >= W) return;

	mod_body<0, TY>(dp, dt, &la, cw + x0 + COFF - HALO, ntp, x0, (int) blockIdx.x, out, (int) blockIdx.x < acc_rows ? acc : NULL);
}

// ---------------------------------------------------------------------------
// Persistent modulator: one CTA per SM slot loops over scan lines; the next line's composite
// window (int32, written by k_raster) and its LineA2 descriptor are fetched by the TMA
// (cp.async.bulk global -> shared, mbarrier completion) into the other half of a double
// buffer while the current line is computed, so no thread spends instructions on staging
// and the load latency is hidden. Used whenever 4 | W (16-byte alignment of every window).
// ---------------------------------------------------------------------------

#define TOFF 28                       // window index = x + TOFF; the filter reads from x0 + (TOFF - 25 - 3)
#define TWIN(W) ((W) + 2 * TOFF + 4)  // ints per window (multiple of 4)

__device__ __forceinline__ unsigned smem_u32(const void *p) { return((unsigned) __cvta_generic_to_shared(p)); }

__device__ __forceinline__ void tma_load(void *dst_smem, const void *src_gmem, unsigned bytes, void *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
		:: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void mbar_wait(void *bar, unsigned parity)
{
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"WAIT_%=:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra DONE_%=;\n\t"
		"bra WAIT_%=;\n\t"
		"DONE_%=:\n\t}"
		:: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

template<int MAXT, int MINB, bool TY = false>
__global__ void __launch_bounds__(MAXT, MINB)
k_mod_tma(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineA2 *lap, const int *comp32, int nlines, int16_t *out,
	const int16_t *acc, int acc_rows)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int W = dp.W;
	const int NW = TWIN(W);
	// [buffer] composite windows, [buffer] descriptors, the NICAM pulse
	int *cw0 = reinterpret_cast<int *>(smem_raw);
	LineA2 *lab0 = reinterpret_cast<LineA2 *>(cw0 + 2 * NW);
	short *ntp = reinterpret_cast<short *>(lab0 + 2);
	__shared__ __align__(8) unsigned long long bar[2];
	const int tid = threadIdx.x;
	const unsigned bytes = (unsigned) (NW * sizeof(int) + sizeof(LineA2));

	if(dp.have_nicam)
	{
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	if(tid == 0)
	{
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bar[0])));
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bar[1])));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();

	int row = blockIdx.x;
	if(tid == 0 && row < nlines)
	{
		// the launch's composite stream starts one line early: line `row` begins at (row + 1) * W
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&bar[0])), "r"(bytes) : "memory");
		tma_load(cw0, comp32 + ((size_t) row + 1) * W - TOFF, NW * sizeof(int), &bar[0]);
		tma_load(lab0, lap + row, sizeof(LineA2), &bar[0]);
	}
	unsigned phase[2] = { 0, 0 };
	for(int it = 0; row < nlines; it++, row += gridDim.x)
	{
		const int cb = it & 1, nb = cb ^ 1;
		const int nrow = row + gridDim.x;
		if(tid == 0 && nrow < nlines)
		{
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&bar[nb])), "r"(bytes) : "memory");
			tma_load(cw0 + nb * NW, comp32 + ((size_t) nrow + 1) * W - TOFF, NW * sizeof(int), &bar[nb]);
			tma_load(lab0 + nb, lap + nrow, sizeof(LineA2), &bar[nb]);
		}
		mbar_wait(&bar[cb], phase[cb]);
		phase[cb] ^= 1;
		const int x0 = tid * SPT;
		if(x0 < W) mod_body<3, TY>(dp, dt, lab0 + cb, cw0 + cb * NW + x0, ntp, x0, row, out, row < acc_rows ? acc : NULL);
		__syncthreads();                                            // everyone is done with this half before it is refilled
	}
}


// ---------------------------------------------------------------------------
// Persistent modulator with the video filter on the tensor cores (htv_mma_fir.h): the 51-tap
// int16 FIR is an exact int8 contraction - the composite stream arrives as a high-byte and a
// low-byte plane (written by k_raster, fetched by the TMA) and is the B operand, loaded
// straight from the window with one 64-bit shared-memory load per fragment; the taps are the
// banded Toeplitz A operand, split the same way and laid out in fragment order on the host
// (dt.mma_atab). Four mma.sync.m16n8k32 (s8/u8 mixes) per k-step leave three int32 partial
// sums per output that recombine to the reference's int32 accumulator (ref fir.c:564-615).
// A warp owns one tile of 128 consecutive samples, I and Q; the results go through a
// shared-memory exchange buffer to the thread that owns four consecutive samples for the sound
// carriers and the store. Buffering: planes x2, exchange x2, descriptors x3 - one
// __syncthreads per line (between filter and sound phase), so a warp that is done with line i
// starts filtering line i + 1 while the others still add the sound carriers of line i.
// The scalar FIR this replaces was 51 half-rate IMAD + 50 IADD per sample (45 % of k_mod_tma).
// Used whenever 128 | W, a video filter is on, and the mode is not SECAM / FM video.
// ---------------------------------------------------------------------------

template<int MAXT, int MINB, bool TY = false>
__global__ void __launch_bounds__(MAXT, MINB)
k_mod_mma(const __grid_constant__ htv_dparams_t dp, const DevTables dt, const LineA2 *lap, const uint8_t *planes, size_t plane_stride,
	int pitch, int nlines, int16_t *out, const int16_t *acc, int acc_rows)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	const int W = dp.W;
	// pitch != 0: one self-contained row per line (any W); 0: the planes are the contiguous stream (128 | W)
	const int WB = pitch ? mf_row_bytes(W) : mf_window_bytes(W), PB = pitch ? WB : mf_plane_bytes(W);
	const int FW = mf_tiles(W) * 4 * MF_ROWW;                           // words of one exchange buffer
	// [buffer][plane] byte windows, the tap operand, two exchange buffers, three descriptors, the NICAM pulse
	unsigned char *pl0 = smem_raw;
	uint4 *atab = reinterpret_cast<uint4 *>(pl0 + 4 * PB);              // [k-step][I hi, I lo, Q hi, Q lo][lane]
	unsigned *fir0 = reinterpret_cast<unsigned *>(atab + MF_ATAB_WORDS / 4);
	LineA2 *lab0 = reinterpret_cast<LineA2 *>(fir0 + 2 * FW);
	short *ntp = reinterpret_cast<short *>(lab0 + 3);
	__shared__ __align__(8) unsigned long long bar[2];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
	const unsigned bytes = (unsigned) (2 * WB + sizeof(LineA2));
	const bool hasq = dp.vf_type == 3;

	if(dp.have_nicam)
	{
		const int4 *src = reinterpret_cast<const int4 *>(dt.nicam_tpad);
		int4 *dst = reinterpret_cast<int4 *>(ntp);
		for(int i = tid; i < (dp.nicam_tpad_len + 7) / 8; i += blockDim.x) dst[i] = __ldg(src + i);
	}
	for(int i = tid; i < MF_ATAB_WORDS / 4; i += blockDim.x) atab[i] = __ldg(reinterpret_cast<const uint4 *>(dt.mma_atab) + i);
	// the bytes behind the window are multiplied by zero taps only; the TMA never writes them
	// (contiguous layout; a pitched row arrives whole)
	for(int i = tid; i < 4 * (PB - WB) / 4; i += blockDim.x)
	{
		const int per = (PB - WB) / 4;
		reinterpret_cast<unsigned *>(pl0 + (i / per) * PB + WB)[i % per] = 0;
	}
	if(tid == 0)
	{
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bar[0])));
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bar[1])));
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();

	int row = blockIdx.x;
	if(tid == 0 && row < nlines)
	{
		// the launch's composite stream starts one line early: line `row` begins at (row + 1) * W
		const uint8_t *src = pitch ? planes + ((size_t) row + 1) * pitch : planes + ((size_t) row + 1) * W - MF_LEAD;
		asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&bar[0])), "r"(bytes) : "memory");
		tma_load(pl0, src, WB, &bar[0]);
		tma_load(pl0 + PB, src + plane_stride, WB, &bar[0]);
		tma_load(lab0, lap + row, sizeof(LineA2), &bar[0]);
	}
	unsigned phase[2] = { 0, 0 };
	int l3 = 0;                                                         // it % 3: descriptor buffer of this line
	for(int it = 0; row < nlines; it++, row += gridDim.x)
	{
		const int cb = it & 1, nb = cb ^ 1;
		const int n3 = l3 == 2 ? 0 : l3 + 1;
		const int nrow = row + gridDim.x;
		if(tid == 0 && nrow < nlines)
		{
			// plane buffer nb was last read by the filter phase of line it - 1 and descriptor n3 by the
			// sound phase of line it - 2: every thread was past both when it reached the barrier of
			// line it - 1, which this thread has left
			const uint8_t *src = pitch ? planes + ((size_t) nrow + 1) * pitch : planes + ((size_t) nrow + 1) * W - MF_LEAD;
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&bar[nb])), "r"(bytes) : "memory");
			tma_load(pl0 + (2 * nb) * PB, src, WB, &bar[nb]);
			tma_load(pl0 + (2 * nb + 1) * PB, src + plane_stride, WB, &bar[nb]);
			tma_load(lab0 + n3, lap + nrow, sizeof(LineA2), &bar[nb]);
		}
		mbar_wait(&bar[cb], phase[cb]);
		phase[cb] ^= 1;

		// ---- video filter: one tile of 128 samples per warp ---------------------
		const unsigned char *ph = pl0 + (2 * cb) * PB, *plo = ph + PB;
		unsigned *fir = fir0 + cb * FW;                                  // last read in the sound phase of line it - 2
		for(int nt = warp; nt < mf_tiles(W); nt += nwarps)
		{
			int ihh[4] = { 0, 0, 0, 0 }, imid[4] = { 0, 0, 0, 0 }, ill[4] = { 0, 0, 0, 0 };
			int qhh[4] = { 0, 0, 0, 0 }, qmid[4] = { 0, 0, 0, 0 }, qll[4] = { 0, 0, 0, 0 };
			const int o0 = mf_b_offset(nt, 0, lane);
			#pragma unroll
			for(int s = 0; s < MF_KSTEPS; s++)
			{
				const uint2 xh = *reinterpret_cast<const uint2 *>(ph + o0 + 32 * s);
				const uint2 xl = *reinterpret_cast<const uint2 *>(plo + o0 + 32 * s);
				const uint4 aih = atab[(s * 4 + 0) * 32 + lane], ail = atab[(s * 4 + 1) * 32 + lane];
				mma_ss(ihh, aih, xh);
				mma_su(imid, aih, xl);
				mma_us(imid, ail, xh);
				mma_uu(ill, ail, xl);
				if(hasq)
				{
					const uint4 aqh = atab[(s * 4 + 2) * 32 + lane], aql = atab[(s * 4 + 3) * 32 + lane];
					mma_ss(qhh, aqh, xh);
					mma_su(qmid, aqh, xl);
					mma_us(qmid, aql, xh);
					mma_uu(qll, aql, xl);
				}
			}
			#pragma unroll
			for(int ci = 0; ci < 4; ci++)
			{
				const int vi = sat16i(mf_combine(ihh[ci], imid[ci], ill[ci]) >> 15);
				const int vq = sat16i(mf_combine(qhh[ci], qmid[ci], qll[ci]) >> 15);    // 0 without Q taps
				fir[mf_fir_index(mf_out_x(nt, lane, ci))] = ((unsigned) vi & 0xFFFFu) | ((unsigned) vq << 16);
			}
		}
		__syncthreads();

		// ---- sound carriers, mixers, store: four consecutive samples per thread ----
		const int x0 = tid * SPT;
		if(x0 < W)
		{
			const uint4 v = *reinterpret_cast<const uint4 *>(fir + mf_fir_index(x0));
			int oi[SPT], oq[SPT];
			oi[0] = (int) (short) (v.x & 0xFFFF); oq[0] = (int) v.x >> 16;
			oi[1] = (int) (short) (v.y & 0xFFFF); oq[1] = (int) v.y >> 16;
			oi[2] = (int) (short) (v.z & 0xFFFF); oq[2] = (int) v.z >> 16;
			oi[3] = (int) (short) (v.w & 0xFFFF); oq[3] = (int) v.w >> 16;
			const LineA2 *la = lab0 + l3;
			kl_sound<-1, 1>(dp, dt, la, ntp, x0, oi, oq);
			mod_store<TY>(dp, dt, la, x0, row, oi, oq, out, row < acc_rows ? acc : NULL);
		}
		l3 = n3;
	}
}

// resident CTAs per SM of the persistent line kernels, by CTA size (256 / 320 / 384 threads <-> W <= 1024 / 1280 / 1536).
// tools/occ_ab.sh builds and times the alternatives. On an H100 SXM (700 W, 1980 MHz), ms per 64 frames: 3 CTAs of 256
// threads instead of 4 take 0.509 against 0.493 at W = 1024 and 0.422 against 0.347 at W = 858; 3 CTAs of 320 threads
// instead of 4 take 0.626 against 0.587 at W = 1280, although at 4 the compiler caps them at 48 registers and spills a little.
#ifndef KL_B256
#define KL_B256 4
#endif
#ifndef KL_B320
#define KL_B320 4
#endif
#ifndef KL_B384
#define KL_B384 2
#endif
#include "htv_line.cuh"
#include "htv_secam_raster.cuh"

// ---------------------------------------------------------------------------
// Kernel tables: every instantiation the host launches, with its entry point taken by address and its template arguments
// as data. Each table's macro passes the same literals to the template and to the entry, so that the selection
// (plan_kernels), the launch and the name htv_line_kernel reports all come from one entry.
// ---------------------------------------------------------------------------

// resident CTAs per SM of a persistent line kernel of MAXT threads
#define KL_MINB(T) ((T) <= 256 ? KL_B256 : (T) <= 320 ? KL_B320 : KL_B384)

typedef void (*KLineFn)(htv_dparams_t, DevTables, const LineR2 *, const LineA2 *, long long, int, int, int16_t *, const int16_t *, int,
	const int16_t *, const int16_t *);
// ps: the converted picture store and the subcarrier stage in k_line (encoders without a composite store); not part of
// the name htv_line_kernel reports
struct KLine { KLineFn fn; int vf, hq, full, csat, maxt, minb, src, snd, wc, st, ps; };
#define KL_ENTRY_PS(VF, HQ, FU, CS, T, SRC, SND, WC, ST, PS) \
	{ k_line<VF, HQ, FU, CS, T, KL_MINB(T), SRC, SND, WC, ST, PS>, VF, HQ, FU, CS, T, KL_MINB(T), SRC, SND, WC, ST, PS }
#define KL_ENTRY(VF, HQ, FU, CS, T, SRC, SND, WC, ST) KL_ENTRY_PS(VF, HQ, FU, CS, T, SRC, SND, WC, ST, false)
// at each CTA size, the int16 store and the store converting to dp.sample_type at run time
#define KL_MAXT(VF, HQ, FU, CS, SRC, PS) \
	KL_ENTRY_PS(VF, HQ, FU, CS, 256, SRC, -1, 0, HTV_TYPE_INT16, PS), KL_ENTRY_PS(VF, HQ, FU, CS, 256, SRC, -1, 0, -1, PS), \
	KL_ENTRY_PS(VF, HQ, FU, CS, 320, SRC, -1, 0, HTV_TYPE_INT16, PS), KL_ENTRY_PS(VF, HQ, FU, CS, 320, SRC, -1, 0, -1, PS), \
	KL_ENTRY_PS(VF, HQ, FU, CS, 384, SRC, -1, 0, HTV_TYPE_INT16, PS), KL_ENTRY_PS(VF, HQ, FU, CS, 384, SRC, -1, 0, -1, PS)
// no video filter, a real low-pass, VSB
#define KL_VF(FU, CS, SRC, PS) KL_MAXT(false, false, FU, CS, SRC, PS), KL_MAXT(true, false, FU, CS, SRC, PS), \
	KL_MAXT(true, true, FU, CS, SRC, PS)
static const KLine kl_tab[] = {
	KL_VF(true, false, false, false), KL_VF(false, false, false, false), KL_VF(false, true, false, false),   // 128 | W, a partial last tile, CSAT
	KL_VF(true, false, false, true), KL_VF(false, false, false, true), KL_VF(false, true, false, true),      // the same, PS
	KL_VF(true, false, true, false), KL_VF(false, false, true, false),                  // SECAM's SRC form: 128 | W, partial
	// PAL's VSB + FM + NICAM + complex output and W = 1024 (16 Msps) compiled in, storing int16 or int8 (the HackRF's format).
	// At 4 CTAs of 256 threads the int16 form's 62 registers (64 allocated) take the whole register file, so the next
	// call's sound pre-pass, records and raster descriptors run in the tail of k_line and between launches, not inside
	// it. That is on purpose: bounded to 48 registers, or at 56, the side kernels shared the SMs with k_line at
	// unpredictable points, and the step got slower and spread (DESIGN.md section 4).
	KL_ENTRY(true, true, true, false, 256, false, KL_SND_FM_NICAM, 1024, HTV_TYPE_INT16),
	KL_ENTRY(true, true, true, false, 256, false, KL_SND_FM_NICAM, 1024, HTV_TYPE_INT8),
};

// The k_line forms with the sound stages compiled in derive their sound state per lane (htv_line.cuh KlFeed, FED); every
// other modulator, the general k_line forms included, reads LineA2
static inline bool kl_fed(const DevPlan &p) { return((p.path == PATH_LINE || p.path == PATH_SEC_LINE) && p.kl && p.kl->snd >= 0); }

typedef void (*KSecFn)(htv_dparams_t, DevTables, const LineS2 *, int, int, int16_t *, SecScratch);
struct KSec { KSecFn fn; int full, maxt, minb; };
#define KS_ENTRY(FU, T) { k_sec_raster<FU, T, KL_MINB(T)>, FU, T, KL_MINB(T) }
static const KSec ks_tab[] = {
	KS_ENTRY(true, 256), KS_ENTRY(false, 256), KS_ENTRY(true, 320), KS_ENTRY(false, 320), KS_ENTRY(true, 384), KS_ENTRY(false, 384),
};

// the split modulators: k_mod (int16 stream), k_mod_tma (int32 stream, 4 | W), k_mod_mma (byte planes, video filter on);
// an entry has the entry point of its own kernel only
typedef void (*KModFn)(htv_dparams_t, DevTables, const LineA2 *, const int16_t *, int16_t *, const int16_t *, int);
typedef void (*KModTmaFn)(htv_dparams_t, DevTables, const LineA2 *, const int *, int, int16_t *, const int16_t *, int);
typedef void (*KModMmaFn)(htv_dparams_t, DevTables, const LineA2 *, const uint8_t *, size_t, int, int, int16_t *, const int16_t *, int);
struct KMod { const char *name; KModFn mod; KModTmaFn tma; KModMmaFn mma; int maxt, minb, ty; };
#define KM_ENTRY(T, B, TY) \
	{ "k_mod", k_mod<T, B, TY>, NULL, NULL, T, B, TY }, { "k_mod_tma", NULL, k_mod_tma<T, B, TY>, NULL, T, B, TY }, \
	{ "k_mod_mma", NULL, NULL, k_mod_mma<T, B, TY>, T, B, TY }
static const KMod km_tab[] = { KM_ENTRY(256, 4, false), KM_ENTRY(256, 4, true), KM_ENTRY(384, 2, false), KM_ENTRY(384, 2, true) };

typedef void (*KFmvBaseFn)(htv_dparams_t, DevTables, const LineA2 *, const int16_t *, int);
struct KFmvBase { KFmvBaseFn fn; int nt; };
#define KFB_ENTRY(NT) { k_fmv_base<NT>, NT }
static const KFmvBase kfb_tab[] = { KFB_ENTRY(0), KFB_ENTRY(67), KFB_ENTRY(71) };

typedef void (*KFmvModFn)(htv_dparams_t, DevTables, const LineA2 *, int16_t *, const int16_t *, int, int);
struct KFmvMod { KFmvModFn fn; int ty; };
#define KFM_ENTRY(TY) { k_fmv_mod<TY>, TY }
static const KFmvMod kfm_tab[] = { KFM_ENTRY(false), KFM_ENTRY(true) };

// the entry of tab that match accepts; none counts a miss
template<typename E, size_t N, typename F> static const E *kfind(const E (&tab)[N], int &miss, F match)
{
	for(const E &e : tab) if(match(e)) return(&e);
	miss++;
	return(NULL);
}

// The name of a k_line instantiation, every template argument spelled out (htv_line_kernel). The int16 forms keep their
// names; a store that converts appends its sample type: ",ST=int8" compiled in, ",ST=-1:float" converting at run time;
// the S-Video form (KL_SV at run time) appends ",SV".
static void kl_name(char *s, size_t n, const KLine &k, int type, bool sv)
{
	char ts[24] = "";
	if(k.st < 0) snprintf(ts, sizeof(ts), ",ST=-1:%s", htv_st_name(type));
	else if(k.st != HTV_TYPE_INT16) snprintf(ts, sizeof(ts), ",ST=%s", htv_st_name(k.st));
	snprintf(s, n, "k_line<VF=%d,HQ=%d,FULL=%d,CSAT=%d,MAXT=%d,SRC=%d,SND=%d,WC=%d%s%s>", k.vf, k.hq, k.full, k.csat, k.maxt, k.src, k.snd,
		k.wc, ts, sv ? ",SV" : "");
}

// ---------------------------------------------------------------------------
// Device layer (C linkage)
// ---------------------------------------------------------------------------

// A failed allocation sets alloc_failed, which fails htv_dev_create; a missing table (src NULL) is not a failure
static void *dev_copy(htv_dev_t *d, const void *src, size_t bytes)
{
	void *p = NULL;
	if(!src || !bytes) return(NULL);
	if(d->nalloc >= HTV_MAX_ALLOCS || cudaMalloc(&p, bytes) != cudaSuccess) { d->alloc_failed = 1; return(NULL); }
	if(cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) { cudaFree(p); d->alloc_failed = 1; return(NULL); }
	d->alloc[d->nalloc++] = p;
	return(p);
}

static void *dev_zero(htv_dev_t *d, size_t bytes)
{
	void *p = NULL;
	if(d->nalloc >= HTV_MAX_ALLOCS || cudaMalloc(&p, bytes) != cudaSuccess) { d->alloc_failed = 1; return(NULL); }
	if(cudaMemset(p, 0, bytes) != cudaSuccess) { cudaFree(p); d->alloc_failed = 1; return(NULL); }
	d->alloc[d->nalloc++] = p;
	return(p);
}

extern "C" int htv_dev_count(void)
{
	int n = 0;
	if(cudaGetDeviceCount(&n) != cudaSuccess) return(0);
	return(n);
}

extern "C" size_t htv_dev_audio_ring_pairs(void) { return(RA); }

// HTV_SEC: test and A/B switches of the SECAM chain (DESIGN §6), comma-separated key=value pairs read when an encoder is
// created. Unset, every value is the default below. An unknown key or a bad value fails the encoder: a typo must not
// quietly run the default path.
static bool sec_knobs(htv_dev_t *d, char *err, size_t errlen)
{
	d->sec_many = SEC_LIST_MANY; d->sec_pred = SEC_PRED; d->sec_repredict = 2; d->sec_repredict_min = 64;
	d->sec_sub = 0; d->sec_passes = 64;
	const char *env = getenv("HTV_SEC");
	if(!env) return(true);
	char buf[256];
	if(strlen(env) >= sizeof(buf)) { snprintf(err, errlen, "HTV_SEC is longer than %d characters", (int) sizeof(buf) - 1); return(false); }
	strcpy(buf, env);
	char *save = NULL;
	for(char *kv = strtok_r(buf, ",", &save); kv; kv = strtok_r(NULL, ",", &save))
	{
		char *v = strchr(kv, '=');
		if(!v) { snprintf(err, errlen, "HTV_SEC: '%s' is not key=value", kv); return(false); }
		*v++ = 0;
		if(!strcmp(kv, "list"))
		{
			// the list kernel: by length (auto), always one warp per line, always one thread per line
			if(!strcmp(v, "auto")) d->sec_many = SEC_LIST_MANY;
			else if(!strcmp(v, "warp")) d->sec_many = INT_MAX;
			else if(!strcmp(v, "thread")) d->sec_many = -1;
			else { snprintf(err, errlen, "HTV_SEC: list=%s is not auto, warp or thread", v); return(false); }
			continue;
		}
		const struct { const char *key; int *dst; long lo, hi; } num[] = {
			{ "pred", &d->sec_pred, 0, 64 },                       // predictor iterations
			{ "repredict", &d->sec_repredict, 0, 64 },             // re-predictions per launch
			{ "repredict_min", &d->sec_repredict_min, -1, INT_MAX },  // listed lines above which one fires (-1: any change)
			{ "sub", &d->sec_sub, 64, INT_MAX },                   // lines per chain launch (at most the default)
			{ "passes", &d->sec_passes, 1, 1024 },                 // refinement passes before HTV_ERROR
		};
		int k = 0;
		while(k < (int) (sizeof(num) / sizeof(num[0])) && strcmp(kv, num[k].key)) k++;
		if(k == (int) (sizeof(num) / sizeof(num[0]))) { snprintf(err, errlen, "HTV_SEC: unknown key '%s'", kv); return(false); }
		char *end = NULL;
		const long x = strtol(v, &end, 10);
		if(!*v || *end || x < num[k].lo || x > num[k].hi)
		{
			snprintf(err, errlen, "HTV_SEC: %s=%s is not an integer in [%ld, %ld]", kv, v, num[k].lo, num[k].hi);
			return(false);
		}
		*num[k].dst = (int) x;
	}
	return(true);
}

static DevSwitches dev_switches(void)
{
	const char *path = getenv("HTV_PATH"), *fir = getenv("HTV_FIR"), *kl = getenv("HTV_KL"), *ahead = getenv("HTV_AHEAD");
	DevSwitches s;
	s.split = path && !strcmp(path, "split");
	s.scalar = fir && !strcmp(fir, "scalar");
	s.kl_general = kl && !strcmp(kl, "general");
	s.no_ahead = ahead && !strcmp(ahead, "0");
	s.debug = getenv("HTV_DEBUG") != NULL;
	return(s);
}

// The kernels an encoder launches, from its tables, the switches and the output sample type alone - never from what the
// device could allocate: the path, the table entries it launches, their shared memory and the name htv_line_kernel
// reports. Host code without a CUDA call (htv_dev_plan_name runs it on a machine without a GPU).
static int plan_kernels(const struct htv_tables_t *t, const DevSwitches &sw, int type, DevPlan *p, char *err, size_t errlen)
{
	const htv_dparams_t &dp = t->dp;
	const int W = dp.W, W4 = (W + 3) & ~3, T = mf_tiles(W);
	const bool secam = dp.colour_mode == HTV_SECAM, typed = type != HTV_TYPE_INT16, full = W % MF_TILE == 0;
	const size_t ntp = sizeof(short) * ((dp.nicam_tpad_len + 7) & ~7);     // the padded NICAM pulse table in shared memory
	memset(p, 0, sizeof(*p));
	p->line_threads = ((W + 3) / 4 + 31) & ~31;
	if(p->line_threads < 64) p->line_threads = 64;
	p->kl_threads = 32 * T;
	// with --pixelrate the raster runs in a context of its own, at the pixel rate: its messages name that line
	const char *whose = t->raster_only ? "the pixel-rate raster's " : "";
	if(p->line_threads > 384) { snprintf(err, errlen, "%sline width %d exceeds the kernels' 1536-sample limit", whose, W); return(HTV_ERROR); }
	// The lower limit: k_line's rows carry 32 samples of each neighbouring line (KL_LEAD halos), and the split modulators
	// stage 32 samples of the line before (EXT), so a line shorter than that would take them from two lines back. FM
	// video's k_fmv_base stages FOFF = 40 samples of the line before from the composite stream, which starts one line
	// early: a shorter line would read in front of it.
	if(W < 32) { snprintf(err, errlen, "%sline width %d is below the kernels' 32-sample limit", whose, W); return(HTV_ERROR); }
	if(dp.have_fmv && W < FOFF)
	{
		snprintf(err, errlen, "line width %d is below FM video's %d-sample limit", W, FOFF);
		return(HTV_ERROR);
	}
	// kl_sound and the sound descriptors let at most one 32 kHz audio segment start in a 32-sample block
	if((dp.have_fm || dp.have_am) && t->rate < 32u * 32000u)
	{
		snprintf(err, errlen, "FM / AM sound at %u Hz is below the kernels' 1.024 MHz limit (one audio sample per 32-sample block)", t->rate);
		return(HTV_ERROR);
	}
	if(secam && t->rs_taps) { snprintf(err, errlen, "--pixelrate with SECAM is not on the accelerated path yet"); return(HTV_ERROR); }
	// The video filter's taps ahead of centre reach the next line's first 25 samples. The SECAM chain of a call runs
	// through the last line it emits, not the one after, so below about 5 Msps, where the burst window starts within
	// those 25 samples, a call's last line would miss the next line's subcarrier.
	if(secam && dp.vf_type && dp.burst_left < MF_NTAPS / 2)
	{
		snprintf(err, errlen, "SECAM with the video filter needs the burst window to start %d samples or more into the line "
			"(it starts at %d)", MF_NTAPS / 2, dp.burst_left);
		return(HTV_ERROR);
	}
	// The fused line kernel (htv_line.cuh) is the default wherever it applies: PAL / NTSC / mono rasters, AM or VSB
	// modulation (or baseband), a chroma low-pass the tensor-core form holds (11 .. 17 taps), no resampler in front of
	// this context. SECAM: its SRC form modulates what the raster and the chrominance chain wrote.
	const bool chroma_ok = dp.colour_mode == HTV_MONOCHROME ||
		((dp.colour_mode == HTV_PAL || dp.colour_mode == HTV_NTSC) && dp.chroma_ntaps >= 3 && dp.chroma_ntaps <= 17);
	// the video filter on the tensor cores (k_mod_mma, k_line), the default for every line width: multiples of 128
	// through the contiguous byte planes, the rest (NTSC 858, 864, ...) through the pitched plane layout (htv_mma_fir.h)
	const bool mma = !secam && dp.vf_type && !sw.scalar;
	if(t->raster_only) p->path = PATH_RASTER;
	else if(dp.have_fmv) p->path = PATH_FMV;
	else if(t->rs_taps) p->path = PATH_RS;
	else if(secam && !sw.split) p->path = PATH_SEC_LINE;
	else if(!secam && !sw.split && chroma_ok && (!dp.vf_type || mma)) p->path = PATH_LINE;
	else p->path = PATH_SPLIT;
	// S-Video has a form in the fused line kernels only (k_line KL_SV, k_sec_raster + k_sec_out's Q plane)
	if(dp.s_video && ((p->path != PATH_LINE && p->path != PATH_SEC_LINE) || (secam && sw.scalar)))
	{
		char why[96];
		if(sw.split) snprintf(why, sizeof(why), "HTV_PATH=split selects the split modulators");
		else if(sw.scalar) snprintf(why, sizeof(why), "HTV_FIR=scalar selects the scalar %s", secam ? "SECAM notch" : "video filter");
		else if(!chroma_ok) snprintf(why, sizeof(why), "a chroma low-pass of %d taps (k_line takes 3 .. 17) runs on the split modulators", dp.chroma_ntaps);
		else snprintf(why, sizeof(why), "path %d", p->path);
		snprintf(err, errlen, "S-Video runs on the fused line kernels only: %s", why);
		return(HTV_ERROR);
	}
	// The lines a call rasters around the ones it emits, for the raster descriptors, the raster stage and the row the
	// modulators read from: one on either side, which the video filter and the line kernels look into. SECAM's rows
	// reach one line further back. The pixel-rate raster reaches one line further on: emitted line t is resampled line
	// t + 1, which is made of raster lines t and t + 1.
	p->before = secam ? 2 : 1;
	p->after = p->path == PATH_RASTER ? 2 : 1;

	p->raster_smem = sizeof(int) * 2 * (W4 + 2 * UOFF);
	if(secam)
	{
		const size_t sm = sizeof(int) * ((((W4 + 2 * LOFF + 14) + 3) & ~3) + W4 + 32) + 2 * (size_t) mf_row_bytes(W) + 32;
		if(sm > p->raster_smem) p->raster_smem = sm;
	}
	const void *raster = secam ? (const void *) k_raster_secam : (const void *) k_raster;
	const int maxt = p->kl_threads <= 256 ? 256 : p->kl_threads <= 320 ? 320 : 384;
	const int vf = dp.vf_type != 0, hq = dp.vf_type == 3, kst = typed ? -1 : HTV_TYPE_INT16;
	const size_t rowb = (size_t) mf_row_bytes(W) + 16, uvb = (size_t) MF_TILE * T + 32;
	int miss = 0;                                    // instantiations the rule asks for and the tables lack
	switch(p->path)
	{
	case PATH_LINE:
	{
		// the chroma low-pass cannot leave the int16 range when the sum of |taps| is at most 32768. The Gaussian taps are
		// rounded one by one, so at about 1 % of sample rates they sum to 32769 .. 32771 (17.734475, 20.05 Msps: 32769),
		// and those rates run the CSAT form. The saturation itself is k_compose's now, so the CSAT forms run the code of
		// the partial-tile form; they, and the partial-tile form for CSAT rates where 128 divides W, stay only because the
		// instantiation names htv_line_kernel reports are pinned by the tests
		long long sum = 0;
		for(int i = 0; i < dp.chroma_ntaps; i++) sum += dp.chroma_taps[i] < 0 ? -dp.chroma_taps[i] : dp.chroma_taps[i];
		const int csat = sum > 32768;
		// the common case (128 | W, a chroma filter that cannot overflow) has its own instantiation, everything else the
		// general one; within it VSB + FM + NICAM + complex output at W = 1024 (PAL-I, B/G at 16 Msps) one with those
		// sound stages and the width compiled in, storing int16 or int8; other sample types run the general form
		// encoders whose subcarrier does not repeat within 4 frames have no composite store: the PS forms
		const int ps = t->comp_phases == 0;
		const bool fixed = !ps && hq && !csat && W == 1024 && kl_snd_mask(dp) == KL_SND_FM_NICAM && !sw.kl_general &&
			(type == HTV_TYPE_INT16 || type == HTV_TYPE_INT8);
		p->kl = kfind(kl_tab, miss, [&](const KLine &k) {
			return(k.vf == vf && k.hq == hq && k.full == (full && !csat) && k.csat == csat && k.maxt == maxt && !k.src &&
				k.snd == (fixed ? KL_SND_FM_NICAM : -1) && k.wc == (fixed ? W : 0) && k.st == (fixed ? type : kst) && k.ps == ps); });
		break;
	}
	case PATH_SEC_LINE:
		p->kl = kfind(kl_tab, miss, [&](const KLine &k) {
			return(k.vf == vf && k.hq == hq && k.full == full && !k.csat && k.maxt == maxt && k.src && k.snd == -1 && !k.wc && k.st == kst); });
		// the raster with the luma notch on the tensor cores (k_sec_raster); HTV_FIR=scalar: k_raster_secam
		if(!sw.scalar)
		{
			p->ks = kfind(ks_tab, miss, [&](const KSec &k) { return(k.full == full && k.maxt == maxt); });
			p->ks_smem = 2 * sizeof(LineS2) + 4 * rowb + 4 * uvb + sizeof(uint4) * (MF_KSTEPS * 2 * 32 + 64) + 64;
		}
		else p->raster = raster;
		break;
	case PATH_SPLIT:
	case PATH_RS:
	{
		// k_mod_mma where the video filter runs on the tensor cores, else k_mod_tma where 4 | W, else k_mod
		const bool tma = !mma && !secam && (W & 3) == 0;
		const char *name = mma ? "k_mod_mma" : tma ? "k_mod_tma" : "k_mod";
		const int mt = p->line_threads <= 256 ? 256 : 384;
		p->mod = kfind(km_tab, miss, [&](const KMod &k) { return(!strcmp(k.name, name) && k.maxt == mt && k.ty == typed); });
		if(mma)
		{
			p->plane_pitch = full ? 0 : mf_pitch(W);
			p->mod_smem = (size_t) 4 * (p->plane_pitch ? mf_row_bytes(W) : mf_plane_bytes(W)) + sizeof(uint32_t) * MF_ATAB_WORDS +
				sizeof(unsigned) * 2 * mf_tiles(W) * 4 * MF_ROWW + 3 * sizeof(LineA2) + ntp + 128;
		}
		else if(tma) p->mod_smem = sizeof(int) * 2 * TWIN(W) + 2 * sizeof(LineA2) + ntp + 128;
		else p->mod_smem = sizeof(int) * (W4 + 2 * EXT + 16) + ntp;
		// --pixelrate: the raster runs in the pixel-rate context (PATH_RASTER), k_resample brings it to this one
		if(p->path == PATH_SPLIT) p->raster = raster;
		break;
	}
	case PATH_FMV:
		p->raster = raster;
		p->fmv_base = kfind(kfb_tab, miss, [&](const KFmvBase &k) { return(k.nt == dp.fmv_ntaps); });
		p->fmv_mod = kfind(kfm_tab, miss, [&](const KFmvMod &k) { return(k.ty == typed); });
		p->fmv_smem = sizeof(int) * (W4 + 2 * FOFF) + ntp;
		if(!p->fmv_base) { snprintf(err, errlen, "unsupported FM pre-emphasis length %d", dp.fmv_ntaps); return(HTV_ERROR); }
		break;
	case PATH_RASTER:
		p->raster = (const void *) k_raster;
		break;
	}
	if(miss) { snprintf(err, errlen, "no kernel instantiation for path %d at W = %d", p->path, W); return(HTV_ERROR); }

	// the name: a split modulator whose store converts appends its TY with the type (k_line spells its own)
	const char *rname = p->ks ? "k_sec_raster" : p->path == PATH_RS ? "k_raster + k_resample" : secam ? "k_raster_secam" : "k_raster";
	char kl[128] = "", tail[24] = "";
	snprintf(tail, sizeof(tail), typed ? " ST=-1:%s" : "", htv_st_name(type));
	if(p->kl)
	{
		kl_name(kl, sizeof(kl), *p->kl, type, dp.s_video);
		// the composite ring and the tap operand where k_line filters: the PS and SRC forms (htv_line.cuh)
		const bool ring = vf && (p->kl->ps || p->kl->src);
		p->kl_smem = (p->kl->snd >= 0 ? 0 : 2 * sizeof(LineA2)) + 2 * sizeof(LineR2) + (ring ? 8 * rowb + sizeof(uint32_t) * MF_ATAB_WORDS : 0) + ntp + 128;
		// PS forms with S-Video: two rows of chroma, four int16 per thread (htv_line.cuh)
		if(dp.s_video && p->kl->ps) p->kl_smem += sizeof(short) * 2 * 4 * p->kl_threads;
	}
	if(p->path == PATH_LINE) snprintf(p->kname, sizeof(p->kname), "%s", kl);
	else if(p->ks) snprintf(p->kname, sizeof(p->kname), "%s<FULL=%d,MAXT=%d> + %s", rname, p->ks->full, p->ks->maxt, kl);
	else if(p->kl) snprintf(p->kname, sizeof(p->kname), "%s + %s", rname, kl);
	else if(p->mod) snprintf(p->kname, sizeof(p->kname), "%s + %s<%d,%d>%s", rname, p->mod->name, p->mod->maxt, p->mod->minb, tail);
	else if(p->fmv_base) snprintf(p->kname, sizeof(p->kname), "%s + k_fmv_base<%d> + k_fmv_scan + k_fmv_mod%s", rname, p->fmv_base->nt, tail);
	return(HTV_OK);
}

// Gives each kernel of the plan the dynamic shared memory it launches with. The limit belongs to the function, which every
// encoder in the process shares, and encoders of one instantiation ask for different amounts (the NICAM pulse table,
// S-Video's chroma rows): it is only ever raised, so that an encoder created later cannot lower it under an earlier one.
static bool plan_attributes(const DevPlan &p, char *err, size_t errlen)
{
	const KMod *m = p.mod;
	const struct { const void *fn; size_t smem; } k[] = {
		{ p.raster, p.raster_smem },
		{ p.kl ? (const void *) p.kl->fn : NULL, p.kl_smem },
		{ p.ks ? (const void *) p.ks->fn : NULL, p.ks_smem },
		{ !m ? NULL : m->mma ? (const void *) m->mma : m->tma ? (const void *) m->tma : (const void *) m->mod, p.mod_smem },
		{ p.fmv_base ? (const void *) p.fmv_base->fn : NULL, p.fmv_smem },
	};
	for(const auto &e : k)
	{
		if(!e.fn) continue;
		cudaFuncAttributes fa;
		cudaError_t r = cudaFuncGetAttributes(&fa, e.fn);
		if(r == cudaSuccess && (size_t) fa.maxDynamicSharedSizeBytes < e.smem)
			r = cudaFuncSetAttribute(e.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) e.smem);
		if(r != cudaSuccess) { snprintf(err, errlen, "%s: %zu bytes of shared memory refused (%s)", p.kname, e.smem, cudaGetErrorString(r)); return(false); }
	}
	return(true);
}

extern "C" int htv_dev_plan_name(const struct htv_tables_t *t, int sample_type, char *name, size_t len)
{
	DevPlan p;
	if(plan_kernels(t, dev_switches(), sample_type, &p, name, len) != HTV_OK) return(HTV_ERROR);
	snprintf(name, len, "%s", p.kname);
	return(HTV_OK);
}

// k_vf_rows over the store rows of the composite-store entries cv.e and, after them, nexc CTAs for the lines
// k_line_desc_r listed (vf_exception) among the raster descriptors from line `first`
static void launch_vf_rows(htv_dev_t *d, const VfConv &cv, int64_t first, int nexc, cudaStream_t st)
{
	const htv_dparams_t &dp = d->dp;
	const unsigned grid = (unsigned) (cv.n * (dp.lines - 2) + nexc);
	const size_t smem = 2 * ((size_t) mf_row_bytes(dp.W) + 16);
	if(dp.vf_type == 3) k_vf_rows<true><<<grid, d->plan.kl_threads, smem, st>>>(dp, d->dt, cv, first);
	else k_vf_rows<false><<<grid, d->plan.kl_threads, smem, st>>>(dp, d->dt, cv, first);
}

// An encoder's side streams and events, in the one list htv_dev_create creates and htv_dev_destroy destroys. ev0 and
// ev1 time the last modulator launch (htv_dev_last_line_ms); every other event only orders work, without timing.
struct DevSync { cudaStream_t *stream[5]; cudaEvent_t *timed[2]; cudaEvent_t *event[11]; };
static DevSync dev_sync(htv_dev_t *d)
{
	return(DevSync{ { &d->side, &d->side2, &d->side3, &d->up, &d->pic }, { &d->ev0, &d->ev1 },
		{ &d->ev_nic, &d->ev_up, &d->ev_chunk[0], &d->ev_chunk[1], &d->ev_in, &d->ev_kl[0], &d->ev_kl[1], &d->ev_r2, &d->ev_audio,
		  &d->ev_pic, &d->ev_call } });
}

// htv_dev_create's way out: the message, and everything allocated so far freed
static htv_dev_t *create_fail(htv_dev_t *d, char *err, size_t errlen, const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(err, errlen, fmt, ap);
	va_end(ap);
	htv_dev_destroy(d);
	return(NULL);
}

extern "C" htv_dev_t *htv_dev_create(const struct htv_tables_t *t, int max_frame_slots, int device, char *err, size_t errlen)
{
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if(e != cudaSuccess || n < 1)
	{
		snprintf(err, errlen, "no CUDA device available (%s)", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
		return(NULL);
	}
	if(device >= n)
	{
		snprintf(err, errlen, "CUDA device %d requested, %d present", device, n);
		return(NULL);
	}
	if(device < 0 && cudaGetDevice(&device) != cudaSuccess) device = 0;    // the calling thread's current device
	DevGuard guard(device);
	htv_dev_t *d = (htv_dev_t *) calloc(1, sizeof(htv_dev_t));
	if(!d) { snprintf(err, errlen, "out of memory"); return(NULL); }
	d->device = device;
	d->tab = t;
	d->dp = t->dp;
	d->sw = dev_switches();
	if(!sec_knobs(d, err, errlen) || plan_kernels(t, d->sw, d->dp.sample_type, &d->plan, err, errlen) != HTV_OK) { free(d); return(NULL); }
	const htv_dparams_t &dp = d->dp;
	const DevPlan &p = d->plan;
	DevTables &dt = d->dt;

	dt.codes = (const uint16_t *) dev_copy(d, t->codes, sizeof(uint16_t) * t->ncodes);
	dt.tmpl_out = (const int16_t *) dev_copy(d, t->tmpl_out, sizeof(int16_t) * (size_t) t->tmpl_rows * t->dp.W);
	dt.tmpl_keep = (const int16_t *) dev_copy(d, t->tmpl_keep, sizeof(int16_t) * (size_t) t->tmpl_rows * t->dp.W);
	dt.tmpl_keep_any = (const uint8_t *) dev_copy(d, t->tmpl_keep_any, t->tmpl_rows);
	dt.glut = (const double *) dev_copy(d, t->glut, sizeof(t->glut));
	dt.clut = (const htv_c16_t *) dev_copy(d, t->clut, sizeof(htv_c16_t) * t->clut_len);
	dt.burst_win = (const int16_t *) dev_copy(d, t->burst_win, sizeof(int16_t) * (t->burst_width + 1));
	dt.fm_ang = (const uint64_t *) dev_copy(d, t->fm_ang, t->fm_ang ? sizeof(uint64_t) * 65536 : 0);
	dt.fm_rot8 = (const float2 *) dev_copy(d, t->fm_rot8, t->fm_rot8 ? sizeof(float) * 2 * 65536 : 0);
	dt.fmv_ang = (const uint64_t *) dev_copy(d, t->fmv_ang, t->fmv_ang ? sizeof(uint64_t) * 65536 : 0);
	dt.afir_v = (const int32_t *) dev_copy(d, t->afir_v, sizeof(t->afir_v));
	dt.afir_f = (const int32_t *) dev_copy(d, t->afir_f, sizeof(t->afir_f));
	dt.lim_shape = (const int16_t *) dev_copy(d, t->lim_shape, sizeof(t->lim_shape));
	dt.nicam_taps = (const int16_t *) dev_copy(d, t->nicam_taps, sizeof(int16_t) * t->nicam_ntaps);
	dt.nicam_lut = (const int16_t *) dev_copy(d, t->nicam_lut, t->nicam_lut ? sizeof(int16_t) * (t->nicam_lut_len + HTV_NICAM_LUT_PAD) : 0);
	dt.nicam_tpad = (const int16_t *) dev_copy(d, t->nicam_tpad, t->nicam_tpad ? sizeof(int16_t) * ((t->dp.nicam_tpad_len + 7) & ~7) : 0);
	dt.nicam_cc = (const htv_c16_t *) dev_copy(d, t->nicam_cc, t->nicam_cc ? sizeof(htv_c16_t) * (t->nicam_cc_len + t->dp.W + 64) : 0);
	dt.nicam_prn = (const uint8_t *) dev_copy(d, t->nicam_prn, sizeof(t->nicam_prn));
	dt.offset_start = (const uint8_t *) dev_copy(d, t->offset_start, t->offset_start ? 32768 : 0);
	dt.secam_fm_lut = (const htv_c32_t *) dev_copy(d, t->secam_fm_lut, t->secam_fm_lut ? sizeof(htv_c32_t) * 65536 : 0);
	dt.secam_bell = (const htv_c16_t *) dev_copy(d, t->secam_bell, t->secam_bell ? sizeof(htv_c16_t) * 65536 : 0);

	{
		short4 *lut = NULL;
		if(!dt.glut || cudaMalloc((void **) &lut, sizeof(short4) << 24) != cudaSuccess)
			return(create_fail(d, err, errlen, "device allocation failed (RGB -> YUV table, 134 MB)"));
		d->alloc[d->nalloc++] = lut;
		if(dp.colour_mode == HTV_SECAM) k_yuv_lut<true><<<65536, 256>>>(dp, dt.glut, lut);
		else k_yuv_lut<false><<<65536, 256>>>(dp, dt.glut, lut);
		dt.yuv_lut = lut;
	}

	d->frame_pixels = (size_t) dp.active_width * dp.active_lines;
	d->max_slots = max_frame_slots < 1 ? 1 : max_frame_slots;
	d->d_frames = (uint32_t *) dev_zero(d, d->frame_pixels * 4 * d->max_slots);
	d->frame_map_cap = 4096;
	d->d_frame_map = (int32_t *) dev_zero(d, sizeof(int32_t) * d->frame_map_cap * 2);      // two halves: see htv_dev_set_frame_map
	if(cudaMallocHost((void **) &d->h_map, sizeof(int32_t) * d->frame_map_cap * MAPBUFS) != cudaSuccess) d->h_map = NULL;
	for(int i = 0; i < MAPBUFS; i++) cudaEventCreateWithFlags(&d->ev_map[i], cudaEventDisableTiming);
	d->d_pcm = (int16_t *) dev_zero(d, sizeof(int16_t) * 2 * RA);
	dt.frames = d->d_frames;
	dt.frame_map = d->d_frame_map;
	if(p.path == PATH_LINE)
	{
		d->ev_slot = (cudaEvent_t *) calloc((size_t) d->max_slots, sizeof(cudaEvent_t));
		if(!d->ev_slot) return(create_fail(d, err, errlen, "out of memory"));
		for(int i = 0; i < d->max_slots; i++)
			if(cudaEventCreateWithFlags(&d->ev_slot[i], cudaEventDisableTiming) != cudaSuccess) return(create_fail(d, err, errlen, "event creation failed"));
	}
	if(p.path == PATH_LINE && !t->comp_phases)
	{
		// the converted picture store (k_picture) of the PS forms: a row per source row of every slot and of the black
		// slot, which also holds the lines with a picture area and no source row; (max_slots + 1) x pic_nrows x W x 6 bytes
		dt.pic_rows = (const int4 *) dev_copy(d, t->pic_rows, sizeof(int32_t) * 4 * t->pic_nrows);
		dt.line_row = (const int32_t *) dev_copy(d, t->line_row, sizeof(int32_t) * (dp.lines + 1));
		dt.pic_nrows = t->pic_nrows;
		dt.pic_black = d->max_slots;
		const size_t n = (size_t) (d->max_slots + 1) * t->pic_nrows * dp.W;
		dt.pic_val = (int16_t *) dev_zero(d, sizeof(int16_t) * n);
		if(dp.colour_mode != HTV_MONOCHROME) dt.pic_cuv = (uint32_t *) dev_zero(d, sizeof(uint32_t) * n);
	}
	if(p.path == PATH_LINE && t->comp_phases)
	{
		// the composite store (k_compose): every line of every slot and of the black slot at each colour-frame phase, and
		// the two stream-start rows; ((max_slots + 1) x comp_phases x lines + 2) x W x 2 bytes, twice with S-Video (87 MB
		// for PAL at 16 Msps). Stream line 0 shares its row with every encoder start: it must have no picture area.
		if(t->codes[1] & (HTV_LC_LEFT_ACTIVE | HTV_LC_RIGHT_ACTIVE))
			return(create_fail(d, err, errlen, "line 1 of the frame has a picture area: not on the fused line kernel"));
		dt.comp_phases = t->comp_phases;
		dt.comp_black = d->max_slots;
		dt.comp_start = (int64_t) (d->max_slots + 1) * dt.comp_phases * dp.lines;
		const size_t n = (size_t) (dt.comp_start + 2) * dp.W;
		if(n >= (size_t) INT32_MAX) return(create_fail(d, err, errlen, "composite store of %zu samples: more than k_line addresses", n));
		d->comp_valid = (uint8_t *) calloc((size_t) d->max_slots, 1);
		if(!d->comp_valid) return(create_fail(d, err, errlen, "out of memory"));
		dt.comp = (int16_t *) dev_zero(d, sizeof(int16_t) * n);
		if(dp.s_video) dt.comp_q = (int16_t *) dev_zero(d, sizeof(int16_t) * n);
		if(p.kl->vf)
		{
			// the filtered store (k_vf_rows): a row for every composite-store row but the stream-start rows, 4 bytes a
			// sample (174 MB for PAL at 16 Msps). One k_vf_rows launch per call takes every pending conversion.
			if(d->max_slots * dt.comp_phases > VF_CONV)
				return(create_fail(d, err, errlen, "%d picture slots x %d phases: more conversions than k_vf_rows takes (%d)",
					d->max_slots, dt.comp_phases, VF_CONV));
			d->vf_conv = (int *) calloc((size_t) d->max_slots * dt.comp_phases, sizeof(int));
			if(!d->vf_conv) return(create_fail(d, err, errlen, "out of memory"));
			dt.filt = (uint32_t *) dev_zero(d, sizeof(uint32_t) * (size_t) dt.comp_start * dp.W);
		}
	}
	dt.pcm = d->d_pcm;
	if(dp.have_fm)
	{
		dt.lim_var = (int32_t *) dev_zero(d, sizeof(int32_t) * RA);
		dt.lim_fix = (int32_t *) dev_zero(d, sizeof(int32_t) * RA);
		dt.fm_p = (int16_t *) dev_zero(d, sizeof(int16_t) * RA);
		dt.fm_B = (uint64_t *) dev_zero(d, sizeof(uint64_t) * RA);
		dt.fm_inc = (uint64_t *) dev_zero(d, sizeof(uint64_t) * RA);
		dt.scan_carry = (unsigned long long *) dev_zero(d, sizeof(unsigned long long) * 8);
		dt.scan_tot = (unsigned long long *) dev_zero(d, sizeof(unsigned long long) * (RA / SCAN_BLK + 8));
	}
	if(dp.have_nicam)
	{
		dt.nic_local = (uint8_t *) dev_zero(d, RS);
		dt.nic_ftot = (uint8_t *) dev_zero(d, RF);
		dt.nic_fstart = (uint8_t *) dev_zero(d, RF);
	}
	if(kl_fed(p))
	{
		// k_line's sound feed: its records, and what one line adds to each quotient and remainder of its state
		if(dp.have_fm) dt.seg_rec = (SegRec *) dev_zero(d, sizeof(SegRec) * RA);
		if(dp.have_nicam) dt.nic_rec = (uint32_t *) dev_zero(d, sizeof(uint32_t) * RS);
		htv_dparams_t &dw = d->dp;
		dw.kl_w_kk = dw.W % 32767;
		dw.kl_w_aq = (uint32_t) (((uint64_t) dw.W * HTV_AUDIO_RATE) / (uint64_t) dw.rate);
		dw.kl_w_ar = (uint32_t) (((uint64_t) dw.W * HTV_AUDIO_RATE) % (uint64_t) dw.rate);
		if(dw.have_nicam)
		{
			dw.kl_w_cc = dw.W % dw.nicam_cc_len;
			dw.kl_w_sq = (uint32_t) (((uint64_t) dw.W * (uint64_t) dw.nicam_D) / (uint64_t) dw.nicam_F);
			dw.kl_w_sr = (uint32_t) (((uint64_t) dw.W * (uint64_t) dw.nicam_D) % (uint64_t) dw.nicam_F);
		}
	}
	if(!dt.codes || !d->h_map || d->alloc_failed || cudaGetLastError() != cudaSuccess) return(create_fail(d, err, errlen, "device allocation failed"));
	d->fm_jc = -1;
	d->nic_kc = 0;
	d->fm_jr = -2;
	d->nic_kr = -1;

	const int W = dp.W;
	const bool secam = dp.colour_mode == HTV_SECAM;
	int nsm = 132;
	cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, d->device);
	// sub-batches keep the int16 composite scratch (2 B/sample) resident in the 50 MB L2
	// SECAM: the cross-line chain is latency bound per launch, so one launch should cover the whole call
	d->sub_lines = ((secam ? 160 : 16) * 1024 * 1024) / (W * 2);
	if(d->sub_lines < 64) d->sub_lines = 64;
	if(secam && d->sec_sub)
	{
		// HTV_SEC=sub=...: shorter chain launches, so that a call crosses launch boundaries (tests)
		if(d->sec_sub > d->sub_lines)
			return(create_fail(d, err, errlen, "HTV_SEC: sub=%d is more than the %d lines of one launch", d->sec_sub, d->sub_lines));
		d->sub_lines = d->sec_sub;
	}
	const size_t rows = (size_t) d->sub_lines + 3;       // every path's before + after is at most 3 (plan_kernels)
	if(p.path != PATH_LINE && cudaMalloc((void **) &d->d_comp, sizeof(int16_t) * rows * W + 256) != cudaSuccess)
		return(create_fail(d, err, errlen, "device allocation failed"));
	if(secam && dp.s_video && cudaMalloc((void **) &d->d_compq, sizeof(int16_t) * rows * W + 256) != cudaSuccess)
		return(create_fail(d, err, errlen, "device allocation failed"));
	if(p.path == PATH_FMV)
	{
		dt.fmv_base = (int16_t *) dev_zero(d, sizeof(int16_t) * (rows + 1) * W + 256);
		dt.fmv_tot = (unsigned long long *) dev_zero(d, sizeof(unsigned long long) * (rows + 1));
		dt.fmv_rowbase = (unsigned long long *) dev_zero(d, sizeof(unsigned long long) * (rows + 1));
		dt.fmv_carry = (unsigned long long *) dev_zero(d, sizeof(unsigned long long));
		if(!dt.fmv_ang) return(create_fail(d, err, errlen, "FM video without its modulator table"));
	}
	if(p.mod && p.mod->tma)
	{
		const size_t bytes = sizeof(int) * (rows * W + 256);
		if(cudaMalloc((void **) &d->d_comp32, bytes) != cudaSuccess) return(create_fail(d, err, errlen, "device allocation failed"));
		cudaMemset(d->d_comp32, 0, bytes);
	}
	if(p.mod && p.mod->mma)
	{
		d->plane_stride = rows * (p.plane_pitch ? p.plane_pitch : W) + 256;
		if(cudaMalloc((void **) &d->d_planes, 2 * d->plane_stride) != cudaSuccess) return(create_fail(d, err, errlen, "device allocation failed"));
		cudaMemset(d->d_planes, 0, 2 * d->plane_stride);
	}
	if(p.mod) d->mod_grid = nsm * p.mod->minb;
	if(p.kl) d->kl_ctas = nsm * p.kl->minb;
	if(p.path == PATH_RS)
	{
		d->rs_I = t->rs_I; d->rs_D = t->rs_D; d->rs_ataps = t->rs_ataps; d->rs_wp = t->rs_wp;
		d->d_rs_taps = (int16_t *) dev_copy(d, t->rs_taps, sizeof(int16_t) * t->rs_I * t->rs_ataps);
	}
	// the tap operands of the tensor-core filters the plan's kernels read
	if((p.kl && p.kl->vf) || (p.mod && p.mod->mma))
	{
		uint32_t atab[MF_ATAB_WORDS];
		mf_build_atab(dp.vf_i, dp.vf_q, atab);
		dt.mma_atab = (const uint32_t *) dev_copy(d, atab, sizeof(atab));
	}
	if(secam && !d->sw.scalar)
	{
		uint32_t nt[MF_KSTEPS * 2 * 32 * 4];
		for(int s3 = 0; s3 < MF_KSTEPS; s3++) for(int lo = 0; lo < 2; lo++) for(int lane = 0; lane < 32; lane++) for(int reg = 0; reg < 4; reg++)
			nt[((s3 * 2 + lo) * 32 + lane) * 4 + reg] = mf_a_word(dp.secam_notch, s3, lane, reg, lo);
		dt.notch_atab = (const uint32_t *) dev_copy(d, nt, sizeof(nt));
	}
	auto lp_atab = [d](const int32_t *taps, int ntaps) {                 // a low-pass of one k-step: SECAM's baseband
		uint32_t ctab[256];
		for(int lo = 0; lo < 2; lo++) for(int lane = 0; lane < 32; lane++) for(int reg = 0; reg < 4; reg++)
			ctab[(lo * 32 + lane) * 4 + reg] = kl_chroma_a_word(taps, ntaps, lane, reg, lo);
		return((const uint32_t *) dev_copy(d, ctab, sizeof(ctab)));
	};
	if(p.ks) dt.sec_lpf_atab = lp_atab(dp.secam_lpf, 15);
	if(secam)
	{
		const size_t groups = (size_t) (W + 2 + 7) / 8 + 1;
		d->sec.rows = (int) rows;
		{
			// the subcarrier's window indexed by line sample, so that k_sec_out loads 8 entries at a time
			const int W8 = (W + 7) & ~7;
			int16_t *w = (int16_t *) calloc((size_t) W8, sizeof(int16_t));
			if(w && t->burst_win)
			{
				for(int x = dp.burst_left; x < W && x - dp.burst_left < t->burst_width; x++) w[x] = t->burst_win[x - dp.burst_left];
				dt.sec_win = (const int16_t *) dev_copy(d, w, sizeof(int16_t) * W8);
			}
			free(w);
		}
		d->sec.cbT = (int16_t *) dev_zero(d, sizeof(int16_t) * groups * rows * 8);
		d->sec.tail = (int *) dev_zero(d, sizeof(int) * rows * SEC_TAIL);
		d->sec.st[0] = (SecState *) dev_zero(d, sizeof(SecState) * rows);
		d->sec.st[1] = (SecState *) dev_zero(d, sizeof(SecState) * rows);
		d->sec.used = (SecState *) dev_zero(d, sizeof(SecState) * rows);
		d->sec.outc = (SecState *) dev_zero(d, sizeof(SecState) * rows);
		d->sec.carry = (SecState *) dev_zero(d, sizeof(SecState));
		d->sec.flags = (int *) dev_zero(d, sizeof(int) * 4);
		d->sec.yT = (int16_t *) dev_zero(d, sizeof(int16_t) * groups * rows * 8);
		d->sec.phT = (int *) dev_zero(d, sizeof(int) * groups * rows * 8);
		d->sec.iyc = (double *) dev_zero(d, sizeof(double) * ((size_t) W / SEC_IYC + 2) * rows);
		d->sec.chk = (SecChk *) dev_zero(d, sizeof(SecChk) * rows);
		d->sec.list = (int *) dev_zero(d, sizeof(int) * rows);
	}
	if(d->alloc_failed) return(create_fail(d, err, errlen, "device allocation failed"));
	if(!plan_attributes(p, err, errlen)) { htv_dev_destroy(d); return(NULL); }
	// the black slot (at every phase) and the stream-start rows, once, behind the RGB -> YUV table on the default stream
	if(dt.pic_val) k_picture<<<dim3(dt.pic_nrows, 1), p.line_threads, p.raster_smem>>>(dp, dt, dt.pic_black);
	if(dt.comp)
	{
		for(int ph = 0; ph < t->comp_phases; ph++) k_compose<<<dp.lines, p.line_threads, p.raster_smem>>>(dp, dt, dt.comp_black, ph, 0);
		k_compose<<<2, p.line_threads, p.raster_smem>>>(dp, dt, dt.comp_black, 0, 1);
		if(dt.filt)
		{
			VfConv cv;
			cv.n = t->comp_phases;
			for(int ph = 0; ph < cv.n; ph++) cv.e[ph] = dt.comp_black * cv.n + ph;
			launch_vf_rows(d, cv, 0, 0, 0);
		}
	}
	const DevSync sy = dev_sync(d);
	bool made = true;
	for(cudaStream_t *s : sy.stream) made &= cudaStreamCreateWithFlags(s, cudaStreamNonBlocking) == cudaSuccess;
	for(cudaEvent_t *e : sy.timed) made &= cudaEventCreate(e) == cudaSuccess;
	for(cudaEvent_t *e : sy.event) made &= cudaEventCreateWithFlags(e, cudaEventDisableTiming) == cudaSuccess;
	if(!made) return(create_fail(d, err, errlen, "stream or event creation failed"));
	d->ahead = p.path == PATH_LINE && !d->sw.no_ahead;
	// the table build and the memsets above ran on the default stream, which the (non-blocking)
	// streams the encoder works on do not wait for
	if(cudaDeviceSynchronize() != cudaSuccess)
		return(create_fail(d, err, errlen, "device initialisation failed (%s)", cudaGetErrorString(cudaGetLastError())));
	return(d);
}

extern "C" void htv_dev_destroy(htv_dev_t *d)
{
	if(!d) return;
	DevGuard guard(d->device);
	// the side streams may still be ahead of the caller's; nothing of this encoder is freed under running work
	cudaDeviceSynchronize();
	for(int i = 0; i < d->nalloc; i++) cudaFree(d->alloc[i]);
	cudaFree(d->d_desc_r); cudaFree(d->d_desc_a2); cudaFree(d->d_vfx); cudaFree(d->d_vfl); cudaFree(d->d_comp); cudaFree(d->d_compq); cudaFree(d->d_comp32); cudaFree(d->d_planes);
	if(d->h_map) cudaFreeHost(d->h_map);
	if(d->h_ov_line) { cudaFreeHost(d->h_ov_line); cudaFreeHost(d->h_ov_meta); cudaFreeHost(d->h_ov_add); }
	cudaFree(d->d_ov_line); cudaFree(d->d_ov_meta); cudaFree(d->d_ov_add);
	if(d->ev_ov) cudaEventDestroy(d->ev_ov);
	for(int i = 0; i < MAPBUFS; i++) if(d->ev_map[i]) cudaEventDestroy(d->ev_map[i]);
	const DevSync sy = dev_sync(d);
	for(cudaStream_t *s : sy.stream) if(*s) cudaStreamDestroy(*s);
	for(cudaEvent_t *e : sy.timed) if(*e) cudaEventDestroy(*e);
	for(cudaEvent_t *e : sy.event) if(*e) cudaEventDestroy(*e);
	free(d->comp_valid);
	free(d->vf_conv);
	if(d->ev_slot) for(int i = 0; i < d->max_slots; i++) if(d->ev_slot[i]) cudaEventDestroy(d->ev_slot[i]);
	free(d->ev_slot);
	free(d);
}

// Uploads of chunk c overwrite picture slots last read by chunk c-2 (see htv_host.c): wait for that
// chunk's kernels, then run beside chunk c-1's. The compute stream joins at htv_dev_uploads_end.
extern "C" void *htv_dev_uploads_begin(htv_dev_t *d)
{
	DevGuard guard(d->device);
	cudaStreamWaitEvent(d->up, d->ev_chunk[d->chunk_i & 1], 0);
	return((void *) d->up);
}

extern "C" int htv_dev_uploads_end(htv_dev_t *d, void *stream)
{
	DevGuard guard(d->device);
	CK(cudaEventRecord(d->ev_up, d->up));
	CK(cudaStreamWaitEvent((cudaStream_t) stream, d->ev_up, 0));
	return(HTV_OK);
}

extern "C" int htv_dev_overlay_capacity(void) { return(HTV_OV_CAP); }

// Overlay table of the next launch sequence: n entries sorted by global line index; add rows are
// copied out of the caller's buffers here (pinned staging), so they may change after the call.
extern "C" int htv_dev_set_overlays(htv_dev_t *d, int n, const long long *line, const int *from, const int *to,
	const int *value, const int16_t *const *add)
{
	DevGuard guard(d->device);
	const int W = d->dp.W;
	if(n > HTV_OV_CAP) return(HTV_ERROR);
	if(n > 0 && !d->h_ov_line)
	{
		CK(cudaMallocHost((void **) &d->h_ov_line, sizeof(long long) * HTV_OV_CAP));
		CK(cudaMallocHost((void **) &d->h_ov_meta, sizeof(int4) * HTV_OV_CAP));
		CK(cudaMallocHost((void **) &d->h_ov_add, sizeof(int16_t) * (size_t) HTV_OV_CAP * W));
		CK(cudaMalloc((void **) &d->d_ov_line, sizeof(long long) * HTV_OV_CAP));
		CK(cudaMalloc((void **) &d->d_ov_meta, sizeof(int4) * HTV_OV_CAP));
		CK(cudaMalloc((void **) &d->d_ov_add, sizeof(int16_t) * (size_t) HTV_OV_CAP * W));
		CK(cudaEventCreateWithFlags(&d->ev_ov, cudaEventDisableTiming));
		d->dt.ov_line = d->d_ov_line; d->dt.ov_meta = d->d_ov_meta; d->dt.ov_add = d->d_ov_add;
	}
	d->dt.ov_n = n;
	if(n == 0) return(HTV_OK);
	CK(cudaEventSynchronize(d->ev_ov));                            // the previous table has left the staging buffers
	int rows = 0;
	for(int i = 0; i < n; i++)
	{
		d->h_ov_line[i] = line[i];
		int row = -1;
		if(add[i]) { row = rows++; memcpy(d->h_ov_add + (size_t) row * W, add[i], sizeof(int16_t) * W); }
		d->h_ov_meta[i] = make_int4(from[i], to[i], value[i], row);
	}
	// on the upload stream: the table of the previous sequence may still be read by its kernels, but
	// uploads_begin made this stream wait for the sequence two back only - so order behind the
	// previous sequence explicitly
	CK(cudaStreamWaitEvent(d->up, d->ev_chunk[(d->chunk_i + 1) & 1], 0));
	CK(cudaMemcpyAsync(d->d_ov_line, d->h_ov_line, sizeof(long long) * n, cudaMemcpyHostToDevice, d->up));
	CK(cudaMemcpyAsync(d->d_ov_meta, d->h_ov_meta, sizeof(int4) * n, cudaMemcpyHostToDevice, d->up));
	if(rows) CK(cudaMemcpyAsync(d->d_ov_add, d->h_ov_add, sizeof(int16_t) * (size_t) rows * W, cudaMemcpyHostToDevice, d->up));
	CK(cudaEventRecord(d->ev_ov, d->up));
	return(HTV_OK);
}

// A new picture in slots slot .. slot + count - 1, copied on `st`. The conversions run on the pic stream, each behind its
// slot's copy, so that the next copies on the upload stream go on beside them; the caller's stream waits for them
// (ev_pic) only when there were any. The converted picture store (PS forms) converts the picture here, the composite
// store marks all phases of the slot stale for htv_dev_set_frame_map. Their slots are under the RGB slots' protection:
// the host cycles 16 slots and brings at most 7 new pictures per call (htv_host.c), and the uploads of call c wait for
// call c - 2's kernels (htv_dev_uploads_begin), which waited for their conversions.
static int slots_uploaded(htv_dev_t *d, int slot, int count, cudaStream_t st)
{
	if(!d->ev_slot) return(HTV_OK);
	for(int i = slot; i < slot + count; i++) CK(cudaEventRecord(d->ev_slot[i], st));
	if(d->comp_valid) memset(d->comp_valid + slot, 0, (size_t) count);
	if(d->dt.pic_val)
	{
		CK(cudaStreamWaitEvent(d->pic, d->ev_slot[slot], 0));
		k_picture<<<dim3(d->dp.active_lines, count), d->plan.line_threads, d->plan.raster_smem, d->pic>>>(d->dp, d->dt, slot);
		d->launches++;
		CK(cudaGetLastError());
		d->pic_pending = 1;
	}
	return(HTV_OK);
}

extern "C" int htv_dev_upload_frame(htv_dev_t *d, int slot, const uint32_t *rgb, void *stream)
{
	DevGuard guard(d->device);
	if(slot < 0 || slot >= d->max_slots) return(HTV_ERROR);
	CK(cudaMemcpyAsync(d->d_frames + (size_t) slot * d->frame_pixels, rgb, d->frame_pixels * 4,
		cudaMemcpyHostToDevice, (cudaStream_t) stream));
	return(slots_uploaded(d, slot, 1, (cudaStream_t) stream));
}

// `count` pictures, contiguous in host memory, into `count` consecutive slots
extern "C" int htv_dev_upload_frames(htv_dev_t *d, int slot, int count, const uint32_t *rgb, void *stream)
{
	DevGuard guard(d->device);
	if(slot < 0 || count < 1 || slot + count > d->max_slots) return(HTV_ERROR);
	// with a store, the last picture goes up in a copy of its own: the others can be converted while it is copied, so
	// that one picture's conversion, not the run's, stands between the copies and the line kernel
	const int head = d->ev_slot && count > 1 ? count - 1 : count;
	for(int at = 0, n = head; at < count; at += n, n = count - at)
	{
		CK(cudaMemcpyAsync(d->d_frames + (size_t) (slot + at) * d->frame_pixels, rgb + (size_t) at * d->frame_pixels,
			d->frame_pixels * 4 * (size_t) n, cudaMemcpyHostToDevice, (cudaStream_t) stream));
		const int r = slots_uploaded(d, slot + at, n, (cudaStream_t) stream);
		if(r != HTV_OK) return(r);
	}
	return(HTV_OK);
}

// The pictures of one k_ingest launch, by value: the kernel parameter holds them, nothing goes up before the launch
struct IngestList { htv_device_frame_t f[HTV_INGEST_MAX]; };

// A picture from device memory into a slot (htv_set_video_device_source): three strided uint8 channels to the slot's
// R << 16 | G << 8 | B words, which every raster path reads as it reads an uploaded picture. One CTA per row blockIdx.x
// of picture blockIdx.y, into slot slot0 + blockIdx.y; the stores are coalesced, the loads are as the strides make them
__global__ void __launch_bounds__(256)
k_ingest(uint32_t *frames, int width, int lines, int slot0, const __grid_constant__ IngestList list)
{
	const htv_device_frame_t &f = list.f[blockIdx.y];
	const uint8_t *row = (const uint8_t *) f.data + (int64_t) blockIdx.x * f.stride_y;
	uint32_t *out = frames + ((size_t) (slot0 + blockIdx.y) * lines + blockIdx.x) * width;
	for(int x = threadIdx.x; x < width; x += blockDim.x)
	{
		const uint8_t *p = row + (int64_t) x * f.stride_x;
		out[x] = (uint32_t) p[0] << 16 | (uint32_t) p[f.stride_c] << 8 | (uint32_t) p[2 * f.stride_c];
	}
}

extern "C" int htv_dev_mark_call(htv_dev_t *d, void *stream)
{
	DevGuard guard(d->device);
	CK(cudaEventRecord(d->ev_call, (cudaStream_t) stream));
	return(HTV_OK);
}

// `count` pictures in device memory into `count` consecutive slots, on `stream` behind the caller's stream at the start
// of the render call (htv_dev_mark_call). Split as htv_dev_upload_frames splits its copy: with a store, the last picture
// is a launch of its own, so that the earlier ones are converted while it is ingested.
extern "C" int htv_dev_ingest_frames(htv_dev_t *d, int slot, int count, const htv_device_frame_t *frames, void *stream)
{
	DevGuard guard(d->device);
	if(slot < 0 || count < 1 || count > HTV_INGEST_MAX || slot + count > d->max_slots) return(HTV_ERROR);
	for(int i = 0; i < count; i++)
	{
		cudaPointerAttributes pa;
		if(cudaPointerGetAttributes(&pa, frames[i].data) != cudaSuccess) { cudaGetLastError(); pa.type = cudaMemoryTypeUnregistered; }
		if((pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged) || pa.device != d->device)
		{
			fprintf(stderr, "hacktv_b200: a device source picture must be device or managed memory on CUDA device %d\n", d->device);
			return(HTV_ERROR);
		}
	}
	const cudaStream_t st = (cudaStream_t) stream;
	CK(cudaStreamWaitEvent(st, d->ev_call, 0));
	const int head = d->ev_slot && count > 1 ? count - 1 : count;
	for(int at = 0, n = head; at < count; at += n, n = count - at)
	{
		IngestList list;
		memset(&list, 0, sizeof(list));
		memcpy(list.f, frames + at, sizeof(htv_device_frame_t) * n);
		k_ingest<<<dim3(d->dp.active_lines, n), 256, 0, st>>>(d->d_frames, d->dp.active_width, d->dp.active_lines, slot + at, list);
		d->launches++;
		CK(cudaGetLastError());
		const int r = slots_uploaded(d, slot + at, n, st);
		if(r != HTV_OK) return(r);
	}
	return(HTV_OK);
}

// The composite rows the frames of this call show and no conversion has filled since their slot's picture came up:
// (slot, frame mod comp_phases) for each frame with a picture (the black slot's are converted at htv_dev_create). A
// (slot, phase) entry is written only when its slot has just been uploaded, or when no line has read that phase since,
// so no line kernel reads it meanwhile. Then the caller's stream waits for this call's conversions, if there were any.
static int convert_frames(htv_dev_t *d, const int32_t *slot_of_frame, int n, int64_t first_frame, cudaStream_t stream)
{
	const int P = d->dt.comp_phases;
	for(int i = 0; d->comp_valid && i < n; i++)
	{
		const int s = slot_of_frame[i], ph = (int) ((first_frame + i) % P);
		if(s < 0 || s >= d->max_slots || (d->comp_valid[s] >> ph & 1)) continue;
		CK(cudaStreamWaitEvent(d->pic, d->ev_slot[s], 0));
		k_compose<<<d->dp.lines, d->plan.line_threads, d->plan.raster_smem, d->pic>>>(d->dp, d->dt, s, ph, 0);
		d->launches++;
		CK(cudaGetLastError());
		d->comp_valid[s] |= (uint8_t) (1u << ph);
		if(d->dt.filt)
		{
			int k = 0;
			while(k < d->vf_nconv && d->vf_conv[k] != s * P + ph) k++;
			if(k == d->vf_nconv) d->vf_conv[d->vf_nconv++] = s * P + ph;
		}
		d->pic_pending = 1;
	}
	if(d->pic_pending)
	{
		CK(cudaEventRecord(d->ev_pic, d->pic));
		CK(cudaStreamWaitEvent(stream, d->ev_pic, 0));
		d->pic_pending = 0;
	}
	return(HTV_OK);
}

extern "C" int htv_dev_set_frame_map(htv_dev_t *d, const int32_t *slot_of_frame, int n, int64_t first_frame, void *stream)
{
	DevGuard guard(d->device);
	if(n > d->frame_map_cap) return(HTV_ERROR);
	const int b = d->map_i;
	d->map_i = (b + 1) % MAPBUFS;
	int32_t *hm = d->h_map + (size_t) b * d->frame_map_cap;
	CK(cudaEventSynchronize(d->ev_map[b]));                        // its previous use (MAPBUFS calls ago) has been consumed
	memcpy(hm, slot_of_frame, sizeof(int32_t) * n);
	if(d->ahead)
	{
		// fused line kernel: the map of the coming call goes into the half its raster descriptors will read, on the
		// stream they run on - beside the previous call's line kernel, once the call before that has let go of the half
		int32_t *dm = d->d_frame_map + (size_t) d->kl_buf * d->frame_map_cap;
		CK(cudaStreamWaitEvent(d->side3, d->ev_kl[d->kl_buf], 0));
		CK(cudaStreamWaitEvent(d->side3, d->ev_up, 0));               // the overlay table, which the raster descriptors read, came up on the upload stream
		CK(cudaMemcpyAsync(dm, hm, sizeof(int32_t) * n, cudaMemcpyHostToDevice, d->side3));
		CK(cudaEventRecord(d->ev_map[b], d->side3));
		d->dt.frame_map = dm;
		d->r2_armed = 1;
	}
	else
	{
		CK(cudaMemcpyAsync(d->d_frame_map, hm, sizeof(int32_t) * n, cudaMemcpyHostToDevice, (cudaStream_t) stream));
		CK(cudaEventRecord(d->ev_map[b], (cudaStream_t) stream));
	}
	d->dt.frame_map_first = first_frame;
	d->dt.frame_map_len = n;
	return(convert_frames(d, slot_of_frame, n, first_frame, (cudaStream_t) stream));
}

extern "C" int htv_dev_upload_audio(htv_dev_t *d, int64_t j0, const int16_t *pcm, size_t npairs, void *stream)
{
	DevGuard guard(d->device);
	while(npairs)
	{
		size_t at = (size_t) (j0 & (RA - 1)), n = npairs;
		if(at + n > RA) n = RA - at;
		CK(cudaMemcpyAsync(d->d_pcm + at * 2, pcm, n * 4, cudaMemcpyHostToDevice, (cudaStream_t) stream));
		pcm += n * 2; j0 += n; npairs -= n;
	}
	return(HTV_OK);
}

// One sample of a device PCM block as the int16 the ring holds (the header's rule for HTV_PCM_FLOAT32: the product
// in float32, rounded to nearest even, clamped; NaN is 0)
__device__ __forceinline__ short pcm_sample(const char *p, int format)
{
	if(format == HTV_PCM_INT16) return(*(const short *) p);
	const float x = __fmul_rn(*(const float *) p, 32767.0f);
	if(x != x) return(0);
	return((short) fminf(fmaxf(rintf(x), -32768.0f), 32767.0f));
}

// A block of stereo PCM from device memory into the sound ring (htv_set_audio_device_source): pair i of the block to
// ring pair (j0 + i) & (RA - 1), wrapping, as the int16 pair the host path copies up. One thread per pair: the stores
// are coalesced 32-bit words, the loads are as the strides make them
__global__ void __launch_bounds__(256)
k_pcm_ingest(short2 *ring, int64_t j0, const __grid_constant__ htv_device_audio_t b)
{
	const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= (int64_t) b.npairs) return;
	const char *p = (const char *) b.data + i * b.stride_pair;
	ring[(j0 + i) & (RA - 1)] = make_short2(pcm_sample(p, b.format), pcm_sample(p + b.stride_ch, b.format));
}

// A device PCM block into ring pairs [j0, j0 + npairs), queued where htv_dev_upload_audio queues its copy: on the
// upload stream, between htv_dev_uploads_begin and htv_dev_uploads_end. The events that order it:
//  - ev_call (waited for here): the block is read after all the work the caller queued on its stream before the render
//    call, so a block written there needs no synchronise;
//  - ev_chunk (htv_dev_uploads_begin): the upload stream runs behind the kernels of the launch sequence before last.
//    The pairs written here lie past everything the previous sequence's pre-pass and line kernel still read (the ring
//    holds about 32 s, a sequence at most 4 s and a piece 8 s), as with the copy;
//  - ev_up (recorded behind the ingest at htv_dev_uploads_end): the pre-pass chains on the side streams (which run
//    ahead, beside the previous call's line kernel) and the caller's stream wait for it, so nothing reads the new
//    pairs before they are written.
extern "C" int htv_dev_ingest_audio(htv_dev_t *d, int64_t j0, const htv_device_audio_t *b, void *stream)
{
	DevGuard guard(d->device);
	const int64_t size = b->format == HTV_PCM_INT16 ? 2 : b->format == HTV_PCM_FLOAT32 ? 4 : 0;
	if(!size)
	{
		fprintf(stderr, "hacktv_b200: unknown device PCM format %d (HTV_PCM_INT16, HTV_PCM_FLOAT32)\n", (int) b->format);
		return(HTV_ERROR);
	}
	if(b->npairs == 0) return(HTV_OK);
	if(b->npairs > RA) return(HTV_ERROR);
	if(((int64_t) (uintptr_t) b->data | b->stride_pair | b->stride_ch) & (size - 1))
	{
		fprintf(stderr, "hacktv_b200: a device PCM block's address and strides must be multiples of its %d-byte samples\n", (int) size);
		return(HTV_ERROR);
	}
	cudaPointerAttributes pa;
	if(cudaPointerGetAttributes(&pa, b->data) != cudaSuccess) { cudaGetLastError(); pa.type = cudaMemoryTypeUnregistered; }
	if((pa.type != cudaMemoryTypeDevice && pa.type != cudaMemoryTypeManaged) || pa.device != d->device)
	{
		fprintf(stderr, "hacktv_b200: a device source PCM block must be device or managed memory on CUDA device %d\n", d->device);
		return(HTV_ERROR);
	}
	const cudaStream_t st = (cudaStream_t) stream;
	CK(cudaStreamWaitEvent(st, d->ev_call, 0));
	k_pcm_ingest<<<(unsigned) ((b->npairs + 255) / 256), 256, 0, st>>>((short2 *) d->d_pcm, j0, *b);
	d->launches++;
	CK(cudaGetLastError());
	return(HTV_OK);
}

extern "C" int htv_dev_audio_prepass(htv_dev_t *d, int64_t m0, int64_t m1, void *stream)
{
	DevGuard guard(d->device);
	const htv_dparams_t &dp = d->dp;
	if(m1 <= m0) return(HTV_OK);
	// everything the caller queued so far (PCM uploads) precedes the pre-pass, which runs on the
	// side stream so that it overlaps the raster kernels of the same call
	// Fused line kernel: the pre-pass chains and their records touch nothing the caller's stream produces - the PCM comes
	// up on the upload stream (ev_up), the rings hold two calls - so they do not wait for the previous call's line kernel
	// but run beside its tail (HTV_AHEAD=0: in the caller's stream order, for A/B)
	if(d->ahead) CK(cudaStreamWaitEvent(d->side, d->ev_up, 0));
	else
	{
		CK(cudaEventRecord(d->ev_in, (cudaStream_t) stream));
		CK(cudaStreamWaitEvent(d->side, d->ev_in, 0));
	}
	d->side_armed = 1;
	cudaStream_t st = d->side;
	// the records of k_line's sound feed, where the plan's k_line reads them (a sample type set after htv_dev_create can
	// choose a general form, which reads LineA2)
	const bool fed = kl_fed(d->plan);
	DevTables dtr = d->dt;
	if(!fed) { dtr.seg_rec = NULL; dtr.nic_rec = NULL; }
	if(dp.have_fm)
	{
		const int64_t jA = d->fm_jc;                               // restart from the last valid prefix entry
		const int64_t jB = fetches_by(m1 - 1, dp.rate) - 1;
		if(jB - jA + 64 + HTV_LIM_W + HTV_AFIR_N >= RA / 2) return(HTV_ERROR);
		if(jB >= jA)
		{
			if(dp.have_lim)
			{
				const int64_t u0 = jA - 2 * HTV_LIM_W, n = jB - u0 + 1;
				k_fm_fir<<<(unsigned) ((n + 127) / 128), 128, 0, st>>>(dp, d->dt, u0, jB);   // 128 = the kernel's tile
				d->launches++;
			}
			const int64_t n = jB - jA + 1;
			k_fm_limit<<<(unsigned) ((n + 127) / 128), 128, 0, st>>>(dp, d->dt, jA, jB);
			const unsigned nb = (unsigned) ((n + SCAN_BLK - 1) / SCAN_BLK);
			k_fm_scan_local<<<nb, SCAN_T, 0, st>>>(d->dt, jA, jB);
			k_fm_scan_fix<<<nb, SCAN_T, 0, st>>>(dtr, jA, jB, d->fm_jr);
			d->launches += 3;
			d->fm_jc = jB;
			if(dtr.seg_rec) d->fm_jr = jB;
		}
	}
	if(dp.have_nicam)
	{
		// its own stream beside the FM chain: the NICAM half of the sound descriptors follows it there
		CK(cudaStreamWaitEvent(d->side2, d->ahead ? d->ev_up : d->ev_in, 0));
		st = d->side2;
		const int64_t s_lo = (int64_t) (((unsigned long long) (m0 > dp.nicam_ntaps ? m0 - dp.nicam_ntaps : 0) * dp.nicam_D) / dp.nicam_F);
		const int64_t s_hi = (int64_t) (((unsigned long long) (m1 - 1) * dp.nicam_D) / dp.nicam_F);
		int64_t k_lo = s_lo / 364, k_hi = s_hi / 364;
		if(k_lo > d->nic_kc) k_lo = d->nic_kc;                     // keep the frame-start chain contiguous
		if(k_hi - k_lo + 2 >= RF / 2 || (k_hi - k_lo + 2) * 364 >= RS / 2) return(HTV_ERROR);
		k_nicam_frames<<<(unsigned) (k_hi - k_lo + 1), 64, 0, st>>>(dp, d->dt, k_lo);
		k_nicam_rec<<<(unsigned) (k_hi - k_lo + 1), NR_T, 0, st>>>(dp, dtr, k_lo, k_hi, d->nic_kr + 1);
		d->launches += 2;
		d->nic_kc = k_hi;                                          // fstart[k_hi] is valid; recompute from there next time
		if(dtr.nic_rec && k_hi > d->nic_kr) d->nic_kr = k_hi;
	}
	if(fed)
	{
		// k_line reads the records (and, for AM, the PCM): its wait for the sound is a wait for the two chains
		CK(cudaEventRecord(d->ev_audio, d->side));
		if(dp.have_nicam) CK(cudaEventRecord(d->ev_nic, d->side2));
	}
	CK(cudaGetLastError());
	return(HTV_OK);
}

// The sound descriptors of lines line0 .. line0 + n - 1 (every modulator but the k_line forms kl_fed feeds), each half on the side stream of the pre-pass chain it depends
// on; ev_audio and ev_nic mark the two halves done. The fused line kernel's buffers are two, so that the next call's
// descriptors may be written while this call's line kernel runs: with HTV_AHEAD they wait for the line kernel that last
// read their buffer, not for the caller's stream. Every other path's wait for this call's place in the caller's stream.
static int launch_desc_a2(htv_dev_t *d, int64_t line0, int n, cudaStream_t st, LineA2 **la)
{
	*la = (LineA2 *) d->d_desc_a2 + (size_t) d->kl_buf * ((size_t) d->desc_cap + 1);
	if(d->ahead && d->side_armed)
	{
		CK(cudaStreamWaitEvent(d->side, d->ev_kl[d->kl_buf], 0));
		CK(cudaStreamWaitEvent(d->side2, d->ev_kl[d->kl_buf], 0));
	}
	else
	{
		if(!d->side_armed)
		{
			CK(cudaEventRecord(d->ev_in, st));
			CK(cudaStreamWaitEvent(d->side, d->ev_in, 0));
		}
		CK(cudaStreamWaitEvent(d->side2, d->ev_in, 0));             // ev_in: this call's place in the caller's stream (pre-pass or above)
	}
	const int dgrid = (n + KD_LINES * KD_WARPS - 1) / (KD_LINES * KD_WARPS);
	k_line_desc_a2<1><<<dgrid, 32 * KD_WARPS, 0, d->side>>>(d->dp, d->dt, *la, line0, n);
	k_line_desc_a2<2><<<dgrid, 32 * KD_WARPS, 0, d->side2>>>(d->dp, d->dt, *la, line0, n);
	CK(cudaEventRecord(d->ev_audio, d->side));
	CK(cudaEventRecord(d->ev_nic, d->side2));
	d->side_armed = 0;
	d->launches += 2;
	return(HTV_OK);
}

// The descriptor buffers of calls of up to n lines: raster descriptors where the context rasters, sound descriptors
// where it modulates, two of each for the fused line kernel. Growing them first waits for every stream that may still
// read the old ones.
static int desc_reserve(htv_dev_t *d, int n, cudaStream_t st)
{
	if(n <= d->desc_cap) return(HTV_OK);
	const DevPlan &p = d->plan;
	const size_t bufs = p.path == PATH_LINE ? 2 : 1;
	cudaStreamSynchronize(st);
	cudaStreamSynchronize(d->side);
	cudaStreamSynchronize(d->side2);
	cudaStreamSynchronize(d->side3);
	cudaFree(d->d_desc_r); cudaFree(d->d_desc_a2); cudaFree(d->d_vfx); cudaFree(d->d_vfl);
	d->d_desc_r = d->d_desc_a2 = NULL;
	d->d_vfx = NULL; d->d_vfl = NULL;
	d->desc_cap = 0;
	static_assert(sizeof(LineS2) == sizeof(LineR2), "one raster descriptor buffer holds either");
	if(p.path != PATH_RS) CK(cudaMalloc(&d->d_desc_r, bufs * sizeof(LineR2) * ((size_t) n + p.before + p.after)));
	// + 1: FM video's fill line (fm_skip)
	if(p.path != PATH_RASTER && !kl_fed(p)) CK(cudaMalloc(&d->d_desc_a2, bufs * sizeof(LineA2) * ((size_t) n + 1)));
	if(d->dt.filt)
	{
		d->vf_cap = vf_list_bound(n + p.before + p.after, p.before, d->dp.lines, HTV_OV_CAP);
		CK(cudaMalloc(&d->d_vfx, bufs * sizeof(uint32_t) * d->vf_cap * d->dp.W));
		CK(cudaMalloc(&d->d_vfl, bufs * sizeof(int) * (1 + d->vf_cap)));
	}
	d->desc_cap = n;
	return(HTV_OK);
}

// The raster descriptors of a call of n lines from line0, entry i <-> line line0 - before + i, by the context c that
// rasters them (d, or its pixel-rate raster context); d counts the launch. Behind the frame map on side3 where
// htv_dev_set_frame_map put it there (the overlays were staged by the host before this call), else on the caller's stream.
static int launch_desc_r(htv_dev_t *d, htv_dev_t *c, int64_t line0, int n, cudaStream_t st, void **lr)
{
	const DevPlan &p = c->plan;
	const int rows = n + p.before + p.after;
	const bool side = c->ahead && c->r2_armed;
	*lr = (char *) c->d_desc_r + (size_t) c->kl_buf * sizeof(LineR2) * ((size_t) c->desc_cap + p.before + p.after);
	const cudaStream_t s = side ? c->side3 : st;
	if(c->dt.filt)
	{
		// the lines of this call that vf_exception lists, and their filtered rows, in the descriptor buffers' half
		c->dt.vf_list = c->d_vfl + (size_t) c->kl_buf * (1 + c->vf_cap);
		c->dt.vfx = c->d_vfx + (size_t) c->kl_buf * c->vf_cap * c->dp.W;
		CK(cudaMemsetAsync(c->dt.vf_list, 0, sizeof(int), s));
	}
	k_line_desc_r<<<(rows + 63) / 64, 64, 0, s>>>(c->dp, c->dt, *lr, line0 - p.before, rows);
	d->launches++;
	if(c->dt.filt)
	{
		// the video filter of those lines and of the store rows of this call's conversions, in one launch per call (the
		// pending conversions are distinct entries, at most max_slots x comp_phases <= VF_CONV: htv_dev_create). The
		// conversions ran on the pic stream: the caller's stream has waited for them (convert_frames), side3 waits here
		if(side && c->vf_nconv) CK(cudaStreamWaitEvent(s, c->ev_pic, 0));
		VfConv cv;
		cv.n = c->vf_nconv;
		for(int k = 0; k < cv.n; k++) cv.e[k] = c->vf_conv[k];
		launch_vf_rows(c, cv, line0 - p.before, vf_list_bound(rows, p.before, c->dp.lines, c->dt.ov_n), s);
		d->launches++;
		c->vf_nconv = 0;
	}
	if(side)
	{
		CK(cudaEventRecord(c->ev_r2, c->side3));
		CK(cudaStreamWaitEvent(st, c->ev_r2, 0));
		c->r2_armed = 0;
	}
	return(HTV_OK);
}

// The persistent grid of k_line and k_sec_raster over n rows: every CTA walks its own run of consecutive rows, at least
// 4 (a run of k_line rasters or stages two lines more than it emits)
static int persistent_grid(int n, int ctas, int *run)
{
	*run = (n + ctas - 1) / ctas;
	if(*run < 4) *run = 4;
	return((n + *run - 1) / *run);
}

// The plan's split modulator over n lines: descriptors la, the composite stream as k_raster / k_resample left it for
// this modulator (byte planes, int32, or the int16 `comp`), output o
static void launch_mod(const htv_dev_t *d, int n, const LineA2 *la, const int16_t *comp, int16_t *o, const int16_t *acc,
	int acc_rows, cudaStream_t st)
{
	const DevPlan &p = d->plan;
	const KMod &m = *p.mod;
	const int grid = n < d->mod_grid ? n : d->mod_grid;                // the persistent forms
	if(m.mma) m.mma<<<grid, p.line_threads, p.mod_smem, st>>>(d->dp, d->dt, la, d->d_planes, d->plane_stride, p.plane_pitch, n, o, acc, acc_rows);
	else if(m.tma) m.tma<<<grid, p.line_threads, p.mod_smem, st>>>(d->dp, d->dt, la, d->d_comp32, n, o, acc, acc_rows);
	else m.mod<<<n, p.line_threads, p.mod_smem, st>>>(d->dp, d->dt, la, comp, o, acc, acc_rows);
}

// The SECAM chrominance chain (htv_secam.cuh) over a sub-batch of n lines, whose raster rows start at ls (rows 0 .. n + 2
// <-> lines first - 2 .. first + n): pass 0 over every line, the predictor, then refinement passes until no line's
// outgoing state changes - at that fixed point every line was computed from its true predecessor state = the
// sequential result. The loop needs the change count on the host, so SECAM launches synchronise.
static int sec_chain(htv_dev_t *d, const LineS2 *ls, int n, cudaStream_t st)
{
	const int nch = n + 2, nb = (nch + 31) / 32;     // the chain's rows: 0 .. n + 1, lines first - 2 .. first + n - 1
	cudaEvent_t dbg0 = NULL, dbg1 = NULL;
	const bool dbg = d->sw.debug;
	if(dbg) { cudaEventCreate(&dbg0); cudaEventCreate(&dbg1); cudaEventRecord(dbg0, st); }
	int pass = 0, changed = 1, repredict = d->sec_repredict;
	htv_secam_chain_t &cs = d->sec_stats;
	cs.launches++;
	for(; pass <= d->sec_passes && changed; pass++)
	{
		int fl[4];
		cudaMemsetAsync(d->sec.flags, 0, sizeof(int) * 4, st);
		if(pass == 0)
		{
			k_sec_pass0<<<nb, 32, 0, st>>>(d->dp, d->dt, ls, d->sec, nch);
			// propose the states pass 1 starts from (see k_sec_predict); st[0] takes them over
			k_sec_predict<<<(nch + SEC_PRED_T - SEC_PRED_HALO - 1) / (SEC_PRED_T - SEC_PRED_HALO), SEC_PRED_T, 0, st>>>(d->dp, d->dt, ls, d->sec, nch, d->sec_pred);
			cudaMemcpyAsync(d->sec.st[0], d->sec.st[1], sizeof(SecState) * nch, cudaMemcpyDeviceToDevice, st);
			d->launches += 2;
			continue;
		}
		k_sec_refine<<<nb, 32, 0, st>>>(d->dp, d->dt, ls, d->sec, nch, pass);
		k_sec_fm_list<<<512, 32 * SEC_LIST_WARPS, 0, st>>>(d->dp, d->dt, ls, d->sec, pass, d->sec_many);
		k_sec_fm_list_t<<<nb, 32, 0, st>>>(d->dp, d->dt, ls, d->sec, pass, d->sec_many);
		d->launches += 3;
		CK(cudaMemcpyAsync(fl, d->sec.flags, sizeof(fl), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		changed = fl[0];
		// what the chain did, from the counts this pass copies back anyway
		cs.passes++;
		cs.recomputed += fl[2];
		if(fl[3] > d->sec_many) cs.listed_thread += fl[3]; else cs.listed_warp += fl[3];
		if(fl[3] > cs.list_max) cs.list_max = fl[3];
		if(dbg)
		{
			float ms = 0;
			cudaEventRecord(dbg1, st); cudaEventSynchronize(dbg1); cudaEventElapsedTime(&ms, dbg0, dbg1);
			fprintf(stderr, "secam pass %d: recomputed %d (FM in full: %d), output changed %d, cumulative %.3f ms\n", pass, fl[2], fl[3], fl[0], ms);
		}
		if(changed && fl[3] > d->sec_repredict_min && repredict > 0)
		{
			// many lines had their FM recurrence re-run: their A, B moved, and plain iteration would carry that down
			// the lines at 3x per pass - propose again from the new checkpoints (the pass's outputs go to st[0] first)
			repredict--;
			if(pass & 1) cs.repredict_odd++; else cs.repredict_even++;
			if(pass & 1) cudaMemcpyAsync(d->sec.st[0], d->sec.st[1], sizeof(SecState) * nch, cudaMemcpyDeviceToDevice, st);
			k_sec_predict<<<(nch + SEC_PRED_T - SEC_PRED_HALO - 1) / (SEC_PRED_T - SEC_PRED_HALO), SEC_PRED_T, 0, st>>>(d->dp, d->dt, ls, d->sec, nch, d->sec_pred);
			if(!(pass & 1)) cudaMemcpyAsync(d->sec.st[0], d->sec.st[1], sizeof(SecState) * nch, cudaMemcpyDeviceToDevice, st);
			d->launches++;
		}
	}
	if(pass - 1 > cs.passes_max) cs.passes_max = pass - 1;
	if(changed)
	{
		fprintf(stderr, "hacktv_b200: SECAM cross-line state did not converge in %d passes\n", d->sec_passes);
		return(HTV_ERROR);
	}
	if((pass - 1) & 1) cs.final_odd++; else cs.final_even++;
	k_sec_carry<<<1, 32, 0, st>>>(ls, d->sec, n - 1, pass - 1);
	k_sec_out<<<dim3((d->dp.W + 63) / 64, (nch + 31) / 32), 256, 0, st>>>(d->dp, d->dt, ls, d->sec, d->d_comp, nch, d->d_compq);
	d->launches += 2;
	return(HTV_OK);
}

// ---------------------------------------------------------------------------
// --pixelrate (SURVEY.md section 8f rank 4): the raster is built at the pixel rate by a second
// device context and the reference's polyphase resampler (ref _init_vresampler video.c:3627-3651,
// fir_int16_resampler_init fir.c:393-428, fir_int16_process fir.c:304-355) brings it to the sample
// rate in front of the video filter. Closed form of the output index (oracle resample_line, pinned
// to the reference): output k of resampled line R uses the rs_ataps inputs ending at
// R * Wp + floor(k D / I) with the taps of phase (k D) mod I (a whole line is a whole number of
// periods because Ws D = Wp I). Row b of `comp` is raster line first - 1 + b of the launch; row b
// of the output is resampled line first + b, which reaches back into comp rows b and b + 1.
// Output goes wherever the modulator of this context reads, in k_raster's store (store_line4): byte planes, pitched
// or contiguous, int32 or int16 stream.
// Parity: tests/test_gpu_zz_pixelrate.py against the oracle (itself pinned to the reference's --pixelrate).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(384)
k_resample(const int16_t *comp, int Wp, int Ws, int I, int D, int A, const int16_t *taps,
	uint8_t *planes, size_t plane_stride, int plane_pitch, int *comp32, int16_t *comp16)
{
	const int b = blockIdx.x;
	const int x0 = threadIdx.x * SPT;
	if(x0 >= Ws) return;
	const int16_t *in = comp + (size_t) (b + 1) * Wp;                   // input 0 of resampled line first + b
	int v[SPT];
	#pragma unroll
	for(int k = 0; k < SPT; k++) v[k] = x0 + k < Ws ? rs_output(in, x0 + k, I, D, A, taps) : 0;
	store_line4(v, x0, Ws, comp16, comp32, planes, plane_stride, plane_pitch);
}

// Lines line0 .. line0 + nlines - 1 into d_out. d is the encoder; r is NULL, or with --pixelrate the raster context built
// from tables at the pixel rate (pictures, frame map and VBI overlays are uploaded to it), whose lines k_resample brings
// to d's rate. The raster and sound descriptors of the whole call come first, then each sub-batch runs a raster stage
// into the composite scratch and a modulator stage from it. The fused line kernel rasters its own lines in one
// persistent launch over the whole call: its one sub-batch has no raster stage.
extern "C" int htv_dev_render_lines(htv_dev_t *d, htv_dev_t *r, int64_t line0, int nlines, int16_t *d_out,
	const int16_t *d_acc, int acc_lines, void *stream)
{
	DevGuard guard(d->device);
	cudaStream_t st = (cudaStream_t) stream;
	const DevPlan &p = d->plan;
	const htv_dparams_t &dp = d->dp;
	if(nlines <= 0) return(HTV_OK);
	if((p.path == PATH_RS) != (r != NULL) || (r && r->plan.path != PATH_RASTER)) return(HTV_ERROR);
	const bool secam = dp.colour_mode == HTV_SECAM;
	// FM video with a pre-emphasis filter: the modulator also integrates the pipeline's fill line
	const int fm_skip = dp.have_fmv && dp.fmv_ntaps > 0 && line0 == 0 ? 1 : 0;
	if(desc_reserve(d, nlines, st) != HTV_OK || (r && desc_reserve(r, nlines, st) != HTV_OK)) return(HTV_ERROR);
	void *desc_r;                                   // entry i <-> line line0 - before + i
	LineA2 *la2 = NULL;                             // la2[i] <-> line line0 - fm_skip + i
	if(launch_desc_r(d, r ? r : d, line0, nlines, st, &desc_r) != HTV_OK ||
		(!kl_fed(p) && launch_desc_a2(d, line0 - fm_skip, nlines + fm_skip, st, &la2) != HTV_OK)) return(HTV_ERROR);
	int sub = p.path == PATH_LINE ? nlines : d->sub_lines;
	if(r && r->sub_lines < sub) sub = r->sub_lines;
	// where the split and FM-video modulators read the composite scratch: line b of the sub-batch at row b + 1
	const int16_t *comp = d->d_comp + (size_t) (p.before - 1) * dp.W;
	int n = 0;
	for(int done = 0; done < nlines; done += n)
	{
		n = nlines - done < sub ? nlines - done : sub;
		const int rows = n + p.before + p.after;
		int16_t *o = (int16_t *) ((char *) d_out + (size_t) done * dp.W * htv_st_bytes(dp.sample_type, dp.complex_out));
		// the stream to sum into (channel combiner): its first acc_lines lines, laid out like d_out
		const int16_t *acc = d_acc && acc_lines > done ? d_acc + (size_t) done * dp.W * (dp.complex_out ? 2 : 1) : NULL;
		const int acc_rows = acc ? acc_lines - done : 0;
		// raster stage
		if(r)
		{
			// the raster at the pixel rate into r's int16 stream, then the rows this context's modulator reads
			k_raster<<<n + r->plan.before + r->plan.after, r->plan.line_threads, r->plan.raster_smem, st>>>(r->dp, r->dt,
				(const LineR2 *) desc_r + done, r->d_comp, NULL, NULL, 0, 0);
			k_resample<<<rows, p.line_threads, 0, st>>>(r->d_comp, r->dp.W, dp.W, d->rs_I, d->rs_D, d->rs_ataps, d->d_rs_taps,
				d->d_planes, d->plane_stride, p.plane_pitch, d->d_comp32, d->d_comp);
			d->launches += 2;
		}
		else if(secam)
		{
			const LineS2 *ls = (const LineS2 *) desc_r + done;
			if(p.ks)
			{
				int run;
				const int grid = persistent_grid(rows, d->kl_ctas, &run);
				p.ks->fn<<<grid, p.kl_threads, p.ks_smem, st>>>(dp, d->dt, ls, rows, run, d->d_comp, d->sec);
				d->launches++;
			}
			else k_raster_secam<<<rows, p.line_threads, p.raster_smem, st>>>(dp, d->dt, ls, d->d_comp, d->sec);
			if(sec_chain(d, ls, n, st) != HTV_OK) return(HTV_ERROR);
			if(d->dt.ov_n > 0)
			{
				k_overlay_secam<<<rows, 256, 0, st>>>(dp, d->dt, line0 + done - p.before, d->d_comp);
				d->launches++;
			}
		}
		else if(p.path != PATH_LINE)
		{
			k_raster<<<rows, p.line_threads, p.raster_smem, st>>>(dp, d->dt, (const LineR2 *) desc_r + done, d->d_comp, d->d_comp32,
				d->d_planes, d->plane_stride, p.plane_pitch);
			d->launches++;
		}
		if(done == 0)
		{
			CK(cudaStreamWaitEvent(st, d->ev_audio, 0));
			CK(cudaStreamWaitEvent(st, d->ev_nic, 0));
		}
		// modulator stage
		if(d->timing && done + n >= nlines) cudaEventRecord(d->ev0, st);
		if(p.kl)
		{
			// k_line from its own raster, or k_line<SRC> from the SECAM raster stage's rows
			int run;
			const int grid = persistent_grid(n, d->kl_ctas, &run);
			const bool line = p.path == PATH_LINE;
			p.kl->fn<<<grid, p.kl_threads, p.kl_smem, st>>>(dp, d->dt, line ? (const LineR2 *) desc_r : NULL, la2 ? la2 + done : NULL,
				(line0 + done) * (long long) dp.W + dp.shift, n, run, o, acc, acc_rows, line ? NULL : d->d_comp, line ? NULL : d->d_compq);
			if(line)
			{
				// this call's descriptor buffers are free again once ev_kl has passed; the next call takes the other two
				CK(cudaEventRecord(d->ev_kl[d->kl_buf], st));
				d->kl_buf ^= 1;
			}
		}
		else if(p.path == PATH_FMV)
		{
			const int pre = fm_skip && done == 0 ? 1 : 0, frows = n + pre;
			const LineA2 *lap = la2 + done + fm_skip - pre;
			p.fmv_base->fn<<<frows, p.line_threads, p.fmv_smem, st>>>(dp, d->dt, lap, comp, pre);
			k_fmv_scan<<<1, 1024, 0, st>>>(d->dt, frows);
			p.fmv_mod->fn<<<frows, p.line_threads, 0, st>>>(dp, d->dt, lap, o, acc, acc_rows, -pre);
			d->launches += 2;
		}
		else launch_mod(d, n, la2 + done, comp, o, acc, acc_rows, st);
		d->launches++;
	}
	if(d->timing) { cudaEventRecord(d->ev1, st); d->ev_pending = 1; }
	d->last_mod_lines = n;
	strcpy(d->kname, p.kname);
	htv_dev_t *const ctx[] = { d, r };
	for(htv_dev_t *c : ctx) if(c)
	{
		CK(cudaEventRecord(c->ev_chunk[c->chunk_i & 1], st));
		c->chunk_i++;
	}
	CK(cudaGetLastError());
	return(HTV_OK);
}

// Standalone channel combiner: acc[i] += in[i] with int16 wrap (ref video.c:3536-3539). Pure
// streaming: 2 B read + 2 B read + 2 B written per value, HBM-bound. `in` may be peer memory.
__global__ void __launch_bounds__(256) k_mix_add(int16_t *acc, const int16_t *in, size_t nvalues)
{
	const size_t n8 = nvalues / 8;
	const size_t stride = (size_t) gridDim.x * blockDim.x;
	for(size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride)
	{
		int4 a = __ldcs(reinterpret_cast<const int4 *>(acc) + i);
		const int4 b = __ldcs(reinterpret_cast<const int4 *>(in) + i);
		a.x = __vadd2(a.x, b.x); a.y = __vadd2(a.y, b.y); a.z = __vadd2(a.z, b.z); a.w = __vadd2(a.w, b.w);
		__stcs(reinterpret_cast<int4 *>(acc) + i, a);
	}
	if(blockIdx.x == 0 && threadIdx.x < (nvalues & 7))
	{
		const size_t i = n8 * 8 + threadIdx.x;
		acc[i] = (int16_t) (acc[i] + in[i]);
	}
}

extern "C" int htv_dev_mix_add(int16_t *d_acc, const int16_t *d_in, size_t nvalues, void *stream)
{
	if(!nvalues) return(HTV_OK);
	if((((uintptr_t) d_acc) | ((uintptr_t) d_in)) & 15) return(HTV_ERROR);
	int dev = 0, nsm = 132;
	cudaGetDevice(&dev);
	{
		// run where the accumulator lives (d_in may be peer memory)
		cudaPointerAttributes pa;
		if(cudaPointerGetAttributes(&pa, d_acc) == cudaSuccess && pa.type == cudaMemoryTypeDevice) dev = pa.device;
	}
	DevGuard guard(dev);
	cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
	size_t blocks = (nvalues / 8 + 255) / 256;
	if(blocks > (size_t) nsm * 8) blocks = (size_t) nsm * 8;
	if(blocks < 1) blocks = 1;
	k_mix_add<<<(unsigned) blocks, 256, 0, (cudaStream_t) stream>>>(d_acc, d_in, nvalues);
	CK(cudaGetLastError());
	return(HTV_OK);
}

// The sample type the stores convert to (htv_set_sample_type, before the first rendered line): the plan again, for the
// instantiations whose store converts
extern "C" int htv_dev_set_sample_type(htv_dev_t *d, int type)
{
	DevGuard guard(d->device);
	DevPlan p;
	char err[256];
	const bool ok = plan_kernels(d->tab, d->sw, type, &p, err, sizeof(err)) == HTV_OK && plan_attributes(p, err, sizeof(err));
	if(!ok) { fprintf(stderr, "hacktv_b200: %s\n", err); return(HTV_ERROR); }
	d->plan = p;
	d->dp.sample_type = type;
	return(HTV_OK);
}

// The alignment htv_render and htv_render_add need of d_out: the widest access the plan's store and channel combiner make
// there. mod_store moves four int16 samples at a time where 4 | W (16 bytes complex, 8 real); every other store - k_line's
// (kl_post_store), mod_store's per-sample branch and the typed stores - moves one sample, I and Q together
extern "C" int htv_dev_out_align(const htv_dev_t *d)
{
	const htv_dparams_t &dp = d->dp;
	if(d->plan.kl || dp.sample_type != HTV_TYPE_INT16 || (dp.W & 3)) return(htv_st_bytes(dp.sample_type, dp.complex_out));
	return(dp.complex_out ? 16 : 8);
}

// htv_convert: dst[i] = the `type` form of src[i] (htv_sample_type.h), eight values per thread and step: one 16-byte
// load, one store of 8, 16 or 32 bytes
template<int T>
__global__ void __launch_bounds__(256) k_convert(void *dst, const int16_t *src, size_t nvalues)
{
	constexpr int S = T == HTV_TYPE_INT8 || T == HTV_TYPE_UINT8 ? 1 : (T == HTV_TYPE_INT32 || T == HTV_TYPE_FLOAT ? 4 : 2);
	const size_t n8 = nvalues / 8;
	const size_t stride = (size_t) gridDim.x * blockDim.x;
	for(size_t i = (size_t) blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += stride)
	{
		const int4 a = __ldcs(reinterpret_cast<const int4 *>(src) + i);
		const int v[8] = { (short) a.x, a.x >> 16, (short) a.y, a.y >> 16, (short) a.z, a.z >> 16, (short) a.w, a.w >> 16 };
		if(S == 1)
		{
			uint2 o;
			o.x = htv_st_bits(T, v[0]) | (htv_st_bits(T, v[1]) << 8) | (htv_st_bits(T, v[2]) << 16) | (htv_st_bits(T, v[3]) << 24);
			o.y = htv_st_bits(T, v[4]) | (htv_st_bits(T, v[5]) << 8) | (htv_st_bits(T, v[6]) << 16) | (htv_st_bits(T, v[7]) << 24);
			__stcs(reinterpret_cast<uint2 *>(dst) + i, o);
		}
		else if(S == 2)
		{
			const uint4 o = make_uint4(htv_st_bits(T, v[0]) | (htv_st_bits(T, v[1]) << 16), htv_st_bits(T, v[2]) | (htv_st_bits(T, v[3]) << 16),
				htv_st_bits(T, v[4]) | (htv_st_bits(T, v[5]) << 16), htv_st_bits(T, v[6]) | (htv_st_bits(T, v[7]) << 16));
			__stcs(reinterpret_cast<uint4 *>(dst) + i, o);
		}
		else
		{
			__stcs(reinterpret_cast<uint4 *>(dst) + 2 * i, make_uint4(htv_st_bits(T, v[0]), htv_st_bits(T, v[1]), htv_st_bits(T, v[2]), htv_st_bits(T, v[3])));
			__stcs(reinterpret_cast<uint4 *>(dst) + 2 * i + 1, make_uint4(htv_st_bits(T, v[4]), htv_st_bits(T, v[5]), htv_st_bits(T, v[6]), htv_st_bits(T, v[7])));
		}
	}
	if(blockIdx.x == 0 && threadIdx.x < (nvalues & 7))
	{
		const size_t i = n8 * 8 + threadIdx.x;
		htv_st_put(dst, i, T, src[i]);
	}
}

extern "C" int htv_dev_convert(void *d_dst, int type, const int16_t *d_src, size_t nvalues, void *stream)
{
	if(!htv_st_size(type) || (((uintptr_t) d_dst) | ((uintptr_t) d_src)) & 15) return(HTV_ERROR);
	if(!nvalues) return(HTV_OK);
	int dev = 0, nsm = 132;
	cudaGetDevice(&dev);
	{
		// run where the destination lives
		cudaPointerAttributes pa;
		if(cudaPointerGetAttributes(&pa, d_dst) == cudaSuccess && pa.type == cudaMemoryTypeDevice) dev = pa.device;
	}
	DevGuard guard(dev);
	cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
	size_t blocks = (nvalues / 8 + 255) / 256;
	if(blocks > (size_t) nsm * 8) blocks = (size_t) nsm * 8;
	if(blocks < 1) blocks = 1;
	cudaStream_t st = (cudaStream_t) stream;
	switch(type)
	{
	case HTV_TYPE_UINT8: k_convert<HTV_TYPE_UINT8><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	case HTV_TYPE_INT8: k_convert<HTV_TYPE_INT8><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	case HTV_TYPE_UINT16: k_convert<HTV_TYPE_UINT16><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	case HTV_TYPE_INT16: k_convert<HTV_TYPE_INT16><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	case HTV_TYPE_INT32: k_convert<HTV_TYPE_INT32><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	case HTV_TYPE_FLOAT: k_convert<HTV_TYPE_FLOAT><<<(unsigned) blocks, 256, 0, st>>>(d_dst, d_src, nvalues); break;
	}
	CK(cudaGetLastError());
	return(HTV_OK);
}

extern "C" int htv_dev_sync(htv_dev_t *d, void *stream)
{
	DevGuard guard(d->device);
	CK(cudaStreamSynchronize((cudaStream_t) stream));
	return(HTV_OK);
}

extern "C" int htv_dev_memcpy_d2h(htv_dev_t *d, void *dst, const void *src, size_t bytes, void *stream)
{
	DevGuard guard(d->device);
	CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t) stream));
	return(HTV_OK);
}

extern "C" int htv_dev_memcpy_h2d(htv_dev_t *d, void *dst, const void *src, size_t bytes, void *stream)
{
	DevGuard guard(d->device);
	CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t) stream));
	return(HTV_OK);
}

// thin stream / event wrappers for the host layer's copy-compute pipeline
extern "C" void *htv_dev_stream_new(htv_dev_t *d) { DevGuard guard(d->device); cudaStream_t s = NULL; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); return((void *) s); }
extern "C" void htv_dev_stream_free(void *s) { if(s) cudaStreamDestroy((cudaStream_t) s); }
extern "C" void *htv_dev_event_new(htv_dev_t *d) { DevGuard guard(d->device); cudaEvent_t e = NULL; cudaEventCreateWithFlags(&e, cudaEventDisableTiming); return((void *) e); }
extern "C" void *htv_dev_event_new_timed(htv_dev_t *d) { DevGuard guard(d->device); cudaEvent_t e = NULL; cudaEventCreate(&e); return((void *) e); }
extern "C" float htv_dev_event_elapsed(void *e0, void *e1) { float ms = -1; cudaEventSynchronize((cudaEvent_t) e1); cudaEventElapsedTime(&ms, (cudaEvent_t) e0, (cudaEvent_t) e1); return(ms); }
extern "C" void htv_dev_event_free(void *e) { if(e) cudaEventDestroy((cudaEvent_t) e); }
extern "C" int htv_dev_event_record(void *e, void *stream) { CK(cudaEventRecord((cudaEvent_t) e, (cudaStream_t) stream)); return(HTV_OK); }
extern "C" int htv_dev_event_wait(void *e) { CK(cudaEventSynchronize((cudaEvent_t) e)); return(HTV_OK); }
extern "C" int htv_dev_stream_wait(void *stream, void *e) { CK(cudaStreamWaitEvent((cudaStream_t) stream, (cudaEvent_t) e, 0)); return(HTV_OK); }

extern "C" int htv_dev_device(const htv_dev_t *d) { return(d->device); }

extern "C" void *htv_dev_alloc(htv_dev_t *d, size_t bytes)
{
	DevGuard guard(d->device);
	void *p = NULL;
	if(cudaMalloc(&p, bytes) != cudaSuccess) return(NULL);
	return(p);
}

extern "C" void htv_dev_free(htv_dev_t *d, void *p) { DevGuard guard(d->device); if(p) cudaFree(p); }

extern "C" void *htv_dev_alloc_pinned(size_t bytes)
{
	void *p = NULL;
	if(cudaMallocHost(&p, bytes) != cudaSuccess) return(NULL);
	return(p);
}

extern "C" void htv_dev_free_pinned(void *p) { if(p) cudaFreeHost(p); }

extern "C" uint64_t htv_dev_launches(const htv_dev_t *d) { return(d->launches); }
extern "C" const char *htv_dev_line_kernel(const htv_dev_t *d) { return(d->kname); }
extern "C" void htv_dev_secam_chain(const htv_dev_t *d, htv_secam_chain_t *out) { *out = d->sec_stats; }
extern "C" void htv_dev_set_timing(htv_dev_t *d, int on) { d->timing = on; }

extern "C" int htv_dev_last_line_count(const htv_dev_t *d) { return(d->last_mod_lines); }

extern "C" float htv_dev_last_line_ms(htv_dev_t *d)
{
	DevGuard guard(d->device);
	float ms = 0;
	if(!d->ev_pending) return(0);
	if(cudaEventSynchronize(d->ev1) != cudaSuccess) return(0);
	cudaEventElapsedTime(&ms, d->ev0, d->ev1);
	return(ms);
}
