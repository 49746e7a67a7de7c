/* nrsc5_b200 — C ABI of the H100-native NRSC-5 FM physical-layer receive
 * engine (libnrsc5_b200.so).  Plain pointers and sizes only.
 *
 * What each entry point replaces in the reference (theori-io/nrsc5 @ a5c0972):
 *
 *   nrsc5b_create / nrsc5b_destroy / nrsc5b_reset
 *       input_init / input_free / input_reset      reference src/input.h:37-40,
 *                                                   src/input.c:126-170
 *   nrsc5b_push_cu8 (+ nrsc5b_push_cu8_device, nrsc5b_push_cu8_all)
 *       input_push_cu8(input_t*, const uint8_t*, uint32_t)
 *                                                   reference src/input.h:42, src/input.c:96-117
 *   nrsc5b_push_cs16
 *       input_push_cs16(input_t*, const int16_t*, uint32_t)   (FM: samples already at 744 187.5 S/s)
 *                                                   reference src/input.h:43, src/input.c:119-124
 *       The reference handles one stream per call; the engine takes a stream
 *       index so that many independent channels share one GPU (BASELINE
 *       configs 3-5).  `nbytes` counts uint8 values, as in the reference.
 *   nrsc5b_process
 *       the synchronous work input_push() triggers: acquire_process ->
 *       sync_push -> decode_push_pm -> nrsc5_conv_decode_* -> descramble
 *                                                   reference src/input.c:41-50,
 *                                                   src/acquire.c:98-263, src/sync.c:339-610,
 *                                                   src/decode.c:378-471, src/conv_dec.c:429-463
 *       All service modes the reference tells apart are decoded: FM MP1, MP2, MP3, MP5, MP6, MP11
 *       (src/sync.c:30-35,343-357,537-595); AM MA1 and MA3 (src/sync.c:612-767).
 *   nrsc5b_drain
 *       the downstream calls of the path, as records in call order:
 *         REC_FRAME      frame_push(frame_t*, bits, len, lc)   reference src/frame.h:53
 *         REC_PIDS       pids_frame_push(pids_t*, bits)        reference src/pids.h:98
 *         REC_SYNC       nrsc5_report_sync                     reference src/private.h:51
 *         REC_LOST_SYNC  nrsc5_report_lost_sync                reference src/private.h:52
 *         REC_MER        nrsc5_report_mer                      reference src/private.h:53
 *         REC_BER        nrsc5_report_ber                      reference src/private.h:54
 *         REC_BLOCK      output_advance (one per 32-symbol block, before that
 *                        block's PDUs)                          reference src/acquire.c:108
 *   nrsc5b_set_sync_state
 *       input_set_sync_state(input_t*, SYNC_STATE_NONE) — the L2->L3 feedback
 *                                                   reference src/input.h:41, src/frame.c:538-539
 *       The engine evaluates the same predicate on the GPU (RS(255,247) header
 *       check, reference src/frame.c:158-179 + src/rs_decode.c) so batch use
 *       needs no host round trip; a host L2 may still force the state.
 *   nrsc5b_enable_l2 / nrsc5b_l2_frames
 *       frame_push / frame_process / frame_reset (L2 framing: PCI, audio PDU headers, packet locations, HEF, CRC-8,
 *       PSD over HDLC, fixed data)                  reference src/frame.h:53-54, src/frame.c:516-742
 *   nrsc5b_rs_decode
 *       decode_rs_char(rs, data, NULL, 0) for the (255,247) code set up at
 *                                                   reference src/frame.c:747, src/rs_decode.c:16
 *
 * Record stream format (identical to the test oracle's): u32 type, u32
 * payload_len, payload padded to 4 bytes.  Frame bits are packed MSB-first.
 *
 * All functions return 0 on success, a negative NRSC5B_E* code otherwise.
 * The engine never falls back to a CPU path: without a CUDA device
 * nrsc5b_create() fails with NRSC5B_ENODEV.
 */
#ifndef NRSC5_B200_H
#define NRSC5_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NRSC5B_MODE_FM 0
#define NRSC5B_MODE_AM 1      /* MA1 / MA3; cs16 at 46 511.72 S/s (input_cs16 = 1) or cu8 at 1 488 375 S/s (input_cs16 = 0,
                               * decimated by 32 on the device); first, unoptimised path */

enum {
    NRSC5B_OK = 0,
    NRSC5B_ENODEV = -1,   /* no CUDA device / CUDA error at creation */
    NRSC5B_EINVAL = -2,
    NRSC5B_ENOMEM = -3,
    NRSC5B_ECUDA = -4,
    NRSC5B_EFULL = -5,    /* input buffer of that stream cannot take the push */
    NRSC5B_EOVERFLOW = -6, /* nrsc5b_drain_all: delivered, but at least one stream's log had overflowed (see nrsc5b_take_overflow) */
};

enum {
    NRSC5B_REC_FRAME = 1,     /* u32 lc (0 = P1, 1 = P3, 2 = P4: logical_channel_t, reference src/frame.h), u32 nbits
                               * (FM: 146176 P1; 4608 P3/P4, 2304 P3 in MP2.  AM: 3750 P1; 24000 / 30000 P3), packed bits */
    NRSC5B_REC_PIDS = 2,      /* 10 bytes (80 bits, MSB first) + u8: 1 if the frame passes the CRC-12 of pids.c:52-86 */
    NRSC5B_REC_SYNC = 3,      /* f32 freq_offset, i32 psmi [AM: + i32 pli, hppi, aabi, rdbi; FM: those stay -1] */
    NRSC5B_REC_LOST_SYNC = 4,
    NRSC5B_REC_MER = 5,       /* f32 lower, f32 upper                      */
    NRSC5B_REC_BER = 6,       /* f32 cber                                  */
    NRSC5B_REC_SOFT_PM = 8,   /* u32 bc, 23040 int8 (only when enabled)    */
    NRSC5B_REC_BLOCK = 9,     /* i32 state_in, i32 samperr, f32 angle, f32 ph_re, f32 ph_im, i32 cfo, i64 start */
    NRSC5B_REC_L2 = 20,       /* what frame_process() made of one frame (nrsc5b_enable_l2): u32 frame_off (log offset of the
                               * frame's packed bits in this drain; nrsc5b_l2_frames: index of the frame), u32 lc, u32 nbits,
                               * u32 pci, u32 flags (1: the sync-loss predicate of frame.c:535-540 fired, 2: event staging
                               * overflowed), u32 pdu_len, u32 ev_len, u32 frame ordinal; then ev_len bytes of events, then
                               * the PDU bytes (PCI removed, headers corrected; padded to 4).  Events, in the order of the
                               * reference's L2 -> L3 calls, each {u32 type, u32 len, payload padded to 4}:
                               *   16 nrsc5_report_audio_service (frame.c:590): i32 program, access, type, codec_mode,
                               *      blend_control, digital_audio_gain, common_delay, latency
                               *   17 output_align (frame.c:606): u32 program, stream_id, offset
                               *   18 output_aas_push (frame.c:365): the bytes (protocol and FCS removed)
                               *   19 output_push (frame.c:635): u32 program, stream_id, seq, shape, flags, size, and the
                               *      packet's offset in the PDU bytes */
};

typedef struct nrsc5b_engine nrsc5b_engine_t;

typedef struct {
    int device;                 /* CUDA device ordinal                                  */
    int nstreams;               /* independent channels on this GPU                     */
    int mode;                   /* NRSC5B_MODE_FM or NRSC5B_MODE_AM                     */
    size_t input_capacity;      /* bytes of cu8 each stream can hold on the device      */
    size_t log_capacity;        /* bytes of output records per stream between drains    */
    int emit_soft;              /* also emit REC_SOFT_PM (debug / parity taps)          */
    int input_cs16;             /* 0: cu8 I/Q at 1 488 375 S/s (nrsc5b_push_cu8); 1: cs16 at 744 187.5 S/s,
                                   i.e. already decimated (nrsc5b_push_cs16), as input_push_cs16 takes it */
} nrsc5b_config_t;

int nrsc5b_create(nrsc5b_engine_t **out, const nrsc5b_config_t *cfg);
void nrsc5b_destroy(nrsc5b_engine_t *e);
int nrsc5b_reset(nrsc5b_engine_t *e, int stream);          /* stream < 0: all */
/* Restart every stream (FM or AM; receiver and L2 state start over) from sample 0 of the input it already holds
 * (benchmark loops). */
int nrsc5b_rewind(nrsc5b_engine_t *e);

/* Use this CUDA stream (a cudaStream_t cast to void*) for all engine work; NULL = legacy default. */
int nrsc5b_set_cuda_stream(nrsc5b_engine_t *e, void *cuda_stream);

/* Append cu8 I/Q (host memory; staged through pinned memory, asynchronous H2D). nbytes % 4 == 0. */
int nrsc5b_push_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes);
/* Append cs16 I/Q (engines created with input_cs16 = 1): nvalues counts int16 values, as in the reference
 * (input_push_cs16, reference src/input.c:119-124; nvalues % 2 == 0). */
int nrsc5b_push_cs16(nrsc5b_engine_t *e, int stream, const int16_t *buf, size_t nvalues);
/* Append `nbytes` to EVERY stream from one page-locked host slab (stream s at host + s*host_stride) with a single
 * strided copy; the streams must hold equally many samples (batch ingest of equally paced channels). */
int nrsc5b_push_cu8_all(nrsc5b_engine_t *e, const uint8_t *host, size_t host_stride, size_t nbytes);
/* Append cu8 I/Q that already lives in device memory (device-to-device copy). */
int nrsc5b_push_cu8_device(nrsc5b_engine_t *e, int stream, const void *dev_buf, size_t nbytes);
/* Point every stream at an existing device buffer [nstreams][stride] holding nbytes valid bytes each (no copy). */
int nrsc5b_attach_device_input(nrsc5b_engine_t *e, const void *dev_buf, size_t stride, size_t nbytes);

/* Write the output records into a caller-owned device buffer [nstreams][stride] (stride % 16 == 0), e.g. one
 * that an NCCL gather can ship to another rank; nrsc5b_drain keeps working on it. */
int nrsc5b_attach_device_log(nrsc5b_engine_t *e, void *dev_buf, size_t stride);

/* Run every 32-symbol block for which a stream's buffered samples suffice; returns when no stream can advance. */
int nrsc5b_process(nrsc5b_engine_t *e);
/* Same, but does not wait for input copies still in flight (pushes are asynchronous): lets the next
 * nrsc5b_push_cu8 overlap with this call's compute.  A later nrsc5b_process() picks up the rest. */
int nrsc5b_process_available(nrsc5b_engine_t *e);
/* Overlapping transfer and compute: nrsc5b_push_fence() marks "everything pushed so far" and returns a token;
 * nrsc5b_process_fence(token) processes exactly that as soon as it has landed, while later pushes keep copying. */
int nrsc5b_push_fence(nrsc5b_engine_t *e);
int nrsc5b_process_fence(nrsc5b_engine_t *e, int token);
/* ---- asynchronous use: nothing below waits for the GPU unless asked to ----
 * nrsc5b_stage_cu8 / _cs16: input_push_cu8 / input_push_cs16 (reference src/input.c:96-124) without a CUDA call - the
 *     samples are copied into page-locked staging memory and travel to the device, one copy per stream, with the next
 *     batch (or when the 4 MiB staging area is full, or at nrsc5b_process).  NRSC5B_EFULL: the device buffer is full of
 *     samples the receiver has not used yet; the engine keeps the rest of the call's samples - wait for the batch in
 *     flight (nrsc5b_poll), submit the next, and call again with (NULL, 0) until it returns 0.
 * nrsc5b_submit: enqueue the passes the buffered samples can need (sized on the host from the sample counts and the
 *     streams' last known window positions: a caller that pushes less than a block at a time launches nothing on most
 *     calls) followed by the export of all records to page-locked host memory.  1 = enqueued, 0 = nothing to do or a
 *     batch is still in flight.  flush != 0 also sends staged input that completes no block yet.
 * nrsc5b_poll: 1 = the batch has finished (wait != 0: block until it has), its records can be read with
 *     nrsc5b_batch_records until the next submit; 0 = none in flight / still running.
 * One batch is in flight at a time; nrsc5b_process / nrsc5b_drain must not be mixed in while one is.  This is what the
 * drop-in libnrsc5.so runs on: pushes return at once, callbacks are made - in the reference's order - from a later
 * push (or from nrsc5_close) as batches complete. */
int nrsc5b_prepare_async(nrsc5b_engine_t *e);      /* optional: allocate the page-locked staging / export buffers now */
int nrsc5b_stage_cu8(nrsc5b_engine_t *e, int stream, const uint8_t *buf, size_t nbytes);
int nrsc5b_stage_cs16(nrsc5b_engine_t *e, int stream, const int16_t *buf, size_t nvalues);
int nrsc5b_submit(nrsc5b_engine_t *e, int flush);
int nrsc5b_poll(nrsc5b_engine_t *e, int wait);
const uint8_t *nrsc5b_batch_records(nrsc5b_engine_t *e, int stream, size_t *nbytes);

/* Wait for the GPU and copy the records of `stream` produced since the last drain.
 * Returns the number of bytes written (>= 0) or a negative error; *needed gets the full size. */
long nrsc5b_drain(nrsc5b_engine_t *e, int stream, uint8_t *out, size_t cap, size_t *needed);
/* nrsc5b_drain for every stream in one call: stream s's records land at out + s*out_stride, sizes[s] bytes.
 * Returns NRSC5B_EFULL (and drains nothing) if a stream's records exceed out_stride. */
int nrsc5b_drain_all(nrsc5b_engine_t *e, uint8_t *out, size_t out_stride, size_t *sizes);
/* 1 if a drain of `stream` since the last call found its log truncated (log_capacity too small for what the stream
 * produced between two drains: the records handed out are a prefix), else 0.  Reading clears it.  Draining rewinds
 * the log and clears the device-side flag, so every truncated drain is reported exactly once. */
int nrsc5b_take_overflow(nrsc5b_engine_t *e, int stream);
/* Wait for the GPU without draining. */
int nrsc5b_synchronize(nrsc5b_engine_t *e);

int nrsc5b_set_sync_state(nrsc5b_engine_t *e, int stream, int state);   /* 0 none, 1 coarse, 2 fine */

typedef struct {
    uint64_t blocks;          /* 32-symbol blocks processed (all streams)       */
    uint64_t samples;         /* cu8 complex samples consumed (all streams)     */
    uint64_t p1_frames;       /* P1 frames decoded                              */
    uint64_t kernel_launches; /* kernels launched by the engine                 */
    uint64_t p1_fallbacks;    /* P1 frames the fast Viterbi handed to the exact fallback kernels */
    uint64_t log_overflows;   /* drains that found a stream's record log truncated */
} nrsc5b_stats_t;
int nrsc5b_get_stats(nrsc5b_engine_t *e, nrsc5b_stats_t *st);

/* Per-kernel device time from CUDA events around every launch (a separate, slower pass):
 * ms4/n4: slot 1 = the front-end kernel (k_stream), slot 3 = the P1 decode group, slot 2 = the L2 kernel (k_l2,
 * when enabled); slot 0 unused. */
int nrsc5b_set_profiling(nrsc5b_engine_t *e, int on);
int nrsc5b_get_kernel_times(nrsc5b_engine_t *e, double *ms4, unsigned long long *n4);

/* SM cycles spent by the stream-resident front-end kernel per phase, summed over streams since the last reset /
 * rewind: cyc12/n12 = {pids flush, prep with coarse acquisition, prep in fine sync, demod (32 symbols),
 * sync+demap of a block that started in fine sync, sync of any other block (vote / CFO search)} followed
 * by six sub-phases of the fine-sync slot {reference gather, Costas loops, tables + feedback, staging,
 * equalise + error sums, demap + bookkeeping}. */
int nrsc5b_get_phase_cycles(nrsc5b_engine_t *e, unsigned long long *cyc12, unsigned long long *n12);

/* AM engines: SM cycles of k_am per phase summed over streams since the last reset / rewind, twelve values: {window + coarse
 * acquisition, first demodulation pass, second pass, sync + slicing, PIDS, P1 + P3 + interleaver, of which P3's post-processing,
 * of which interleaver; across all decodes: K=9 recursion, traceback; window load of the blocks in fine sync; spare}. */
int nrsc5b_get_am_phase_cycles(nrsc5b_engine_t *e, unsigned long long *cyc12);

/* Experiment switches for kernel tuning (bit 0: do not overlap carrier staging with the Costas loops; bit 1: library
 * sincosf / atan2f on the Costas loops' dependent chain instead of the short-chain versions; bit 3: nrsc5b_viterbi_k9 prints its
 * cycle counts per frame); 0 = default.  Also read
 * from the environment (NRSC5_B200_DBG) when an engine is created. */
int nrsc5b_debug_set(int flags);

/* L2 framing on the device (SURVEY 8 f1) for every frame the engine (FM or AM) decodes from now on: after each REC_FRAME's pass
 * the log also holds a REC_L2 record with what frame_push / frame_process (reference src/frame.c:516-714) would have
 * handed on: audio service changes, elastic-buffer alignment, PSD / AAS messages and the HDC packets with their CRC
 * verdicts.  The per-stream L2 state (service table, PSD and fixed-data assembly) lives on the GPU. */
int nrsc5b_enable_l2(nrsc5b_engine_t *e, int on);

/* ---- single-stage entry points (kernel-level parity tests, host buffers) ---- */
/* cu8 -> Q15 -> halfband /2 from zero history: out[2*npairs] int16 (reference src/firdecim_q15.c:137-165) */
int nrsc5b_halfband_fm(int device, const uint8_t *cu8, size_t npairs, int16_t *out_ri);
/* batch of tail-biting K=7 rate-1/3 Viterbi decodes: in[nframes][3*len] int8 -> out[nframes][len] bits (one per byte) */
int nrsc5b_viterbi_k7(int device, const int8_t *in, uint8_t *out, int len, int nframes);
/* same; *fallbacks = frames the register-resident fast path handed to the exact fallback kernels */
int nrsc5b_viterbi_k7_ex(int device, const int8_t *in, uint8_t *out, int len, int nframes, int *fallbacks);
/* batch RS(255,247) decode in place; rc[n] = corrections or -1 (reference src/rs_decode.c:16) */
int nrsc5b_rs_decode(int device, uint8_t *blocks255, int *rc, int nblocks);
/* The AM chain's K=9 rate-1/3 tail-biting Viterbi decoder (reference src/conv_dec.c + src/conv_gen.h with K = 9 as
 * src/decode.c:487,515-539 call it): njobs frames of len bits; in = 3 * len hard symbols per frame (-1, 0 = punctured, +1:
 * the AM chain slices hard, other values are rejected), out = len bits per frame.  warmup / chunk_warmup <= 0 select the
 * production warm-up of the segmented traceback / of the recursion's chunks; rounds (optional, [njobs]) receives the repair
 * rounds the traceback needed (low 16 bits) and the chunks of the recursion that had to be run again (high 16 bits). */
int nrsc5b_viterbi_k9(int device, const int8_t *in, uint8_t *out, int len, int njobs, unsigned g0, unsigned g1, unsigned g2,
                      int warmup, int chunk_warmup, int *rounds);
/* L2 alone on one stream: frames = {u32 lc, u32 nbits, packed bits padded to 4 bytes} back to back, nbits == 0 standing
 * for frame_reset (frame.c:716); all six frame lengths of frame.c:651-690.  Writes one REC_L2 record per frame
 * (frame_off = the frame's index in the list) and returns the bytes written, or NRSC5B_EFULL. */
long nrsc5b_l2_frames(int device, const uint8_t *frames, size_t nbytes, uint8_t *out, size_t cap, size_t *needed);
/* 2048-point forward complex FFT of nffts rows (float2 interleaved), natural order, for numerics tests */
int nrsc5b_fft2048(int device, const float *in, float *out, int nffts);

/* ---- wideband channeliser (SURVEY 8 f3; the reference has no counterpart: its ingest is one narrowband device per
 * handle, reference src/nrsc5.c:130-207) ----
 * One cu8 capture at 32 x 744 187.5 = 23 814 000 S/s -> `nch` FM channels at 744 187.5 S/s cs16, the format
 * input_push_cs16 (reference src/input.c:119-124) / nrsc5b_push_cs16 take.  Channel k is centred `offsets_100khz[k]` x
 * 100 kHz from the capture's centre.  Integer-exact definition (csrc/channelizer.cu header; restated in numpy by
 * tests/test_channelizer.py):
 *     acc = sum_{u<256} W_k[u] * (x[32 n + u] - (127 + 127j));   v = (acc + 2^12) >> 13;
 *     y[k][n] = saturate16((v * conj(P[(1600 m_k n) mod 11907]) + 2^14) >> 15)
 * with the 16-bit taps W_k and the phasor table P as returned by nrsc5b_chan_tables.  Runs on the tensor cores
 * (wgmma u8 x s8, TMA-fed, accumulators in registers). */
typedef struct nrsc5b_channelizer nrsc5b_channelizer_t;
int nrsc5b_chan_create(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch);
void nrsc5b_chan_destroy(nrsc5b_channelizer_t *c);
/* taps[nch][256][2] (real, imaginary part of W_k[u]) and phasor[11907][2]; either may be NULL */
int nrsc5b_chan_tables(nrsc5b_channelizer_t *c, int16_t *taps, int16_t *phasor);
/* the same tables computed on the host without a device (the definition's inputs, for the numpy restatement) */
int nrsc5b_chan_make_tables(const int *offsets_100khz, int nch, int16_t *taps, int16_t *phasor);
/* output samples per channel for a capture of nbytes (a multiple of 64): nbytes / 64 - 7 */
long long nrsc5b_chan_outputs(size_t nbytes);
/* device capture (64-byte aligned, nbytes % 64 == 0) -> device out[nch][out_stride] (int16 values, I/Q interleaved;
 * out_stride >= 2 * outputs, even), asynchronous on cuda_stream (a cudaStream_t cast to void*, NULL = default) */
int nrsc5b_chan_run_device(nrsc5b_channelizer_t *c, const void *d_cu8, size_t nbytes, void *d_out, size_t out_stride, void *cuda_stream);
/* host capture -> host out[nch][2 * outputs]; synchronous (tests) */
int nrsc5b_chan_run(nrsc5b_channelizer_t *c, const uint8_t *cu8, size_t nbytes, int16_t *out);

const char *nrsc5b_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NRSC5_B200_H */
