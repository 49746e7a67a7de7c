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
    NRSC5B_REC_PAD = 12,      /* no payload, stands for no call: readers skip it.  FM keeps one after the P1 frame of a
                               * block that also ends a P3 / P4 frame; if the P1 frame's header check fails, it becomes
                               * REC_LOST_SYNC, so that the sync loss comes before those frames, as in the reference
                               * (frame_push in decode_push_pm reports it before decode_push_px1 / _px2 run) */
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
/* the register-resident fast path alone with chunks of ch steps (len, ch multiples of 32): dec[nframes][len+64][2] its
 * decision words (bit 8*(n>>4) + (n&7) of word (n>>3)&1 set = new state n's survivor comes from the odd predecessor),
 * retry[nframes] != 0 where it would hand the frame to the exact fallback */
int nrsc5b_viterbi_k7_fast(int device, const int8_t *in, int len, int nframes, int ch, uint32_t *dec, int *retry);
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
 * (wgmma u8 x s8, TMA-fed, accumulators in registers).
 *
 * Streaming (nrsc5b_chan_push, nrsc5b_chan_feed): a live capture arrives in pieces, so a handle keeps two values,
 *     T, the complex samples pushed since create / nrsc5b_chan_reset, and the carry, the last < 256 samples it has not
 *     consumed yet.
 * With N(T) = T >= 256 ? (T - 256) / 32 + 1 : 0, a push that takes T to T' emits exactly outputs N(T) .. N(T') - 1 of
 * every channel, n in the mixer's phasor index being that absolute output index; the carry kept afterwards is the
 * samples from 32 N(T') on (at most 255 samples, 510 bytes).  So pushing a capture in pieces of any even byte count
 * (shorter than the filter, not a multiple of 64, empty) gives, concatenated, the outputs of nrsc5b_chan_run on the
 * whole capture, bit for bit.  The one-shot entry points (nrsc5b_chan_run*) neither use nor change T and the carry. */
typedef struct nrsc5b_channelizer nrsc5b_channelizer_t;
int nrsc5b_chan_create(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch);
void nrsc5b_chan_destroy(nrsc5b_channelizer_t *c);
/* taps[nch][256][2] (real, imaginary part of W_k[u]; an AM-plan handle: [nch][512][2]) and phasor[11907][2]; either
 * may be NULL */
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
/* Start the stream over: T = 0, the carry is dropped. */
int nrsc5b_chan_reset(nrsc5b_channelizer_t *c);
/* Push the next nbytes (even; otherwise NRSC5B_EINVAL) of the capture and write the outputs they complete to the
 * device buffer d_out[nch][out_stride] (int16 values, I/Q interleaved; row k = channel k, this push's first output at
 * column 0; out_stride even and >= 2 * *nout, d_out 4-byte aligned).  cu8 may be pageable or page-locked host memory or
 * device memory.  Asynchronous on cuda_stream (a cudaStream_t cast to void*, NULL = default); page-locked and device
 * input must stay valid until the stream has run the copy.  *nout (may be NULL) = outputs written per channel,
 * N(T') - N(T).  Internally the channeliser stages up to 4 MiB at a time, so a push of any size works. */
int nrsc5b_chan_push(nrsc5b_channelizer_t *c, const uint8_t *cu8, size_t nbytes, void *d_out, size_t out_stride, void *cuda_stream,
                     long long *nout);
/* The same push, but channel k is appended straight to the input of stream streams[k] of the cs16 engine `e` (streams
 * NULL: stream k), as nrsc5b_push_cs16 would append it.  `e` must be an FM engine created with input_cs16 = 1 on the
 * channeliser's device that reads its own input buffers (not nrsc5b_attach_device_input); the stream indices must be
 * distinct and < nstreams.  Otherwise, and for odd nbytes: NRSC5B_EINVAL, nothing changed.
 * Runs on the engine's CUDA stream and publishes each stream's new sample count after the kernel; it does not wait for
 * the GPU, except for the synchronous trim a full stream gets (as in nrsc5b_push_cs16).  All or nothing: if a target
 * stream has no room for the push's outputs even after trimming, it returns NRSC5B_EFULL and neither the channeliser
 * nor the engine has taken any of it - run nrsc5b_process and push the same bytes again.  Like nrsc5b_process, it must
 * not be mixed with an asynchronous batch in flight (nrsc5b_submit .. nrsc5b_poll). */
int nrsc5b_chan_feed(nrsc5b_channelizer_t *c, nrsc5b_engine_t *e, const int *streams, const uint8_t *cu8, size_t nbytes);

/* cs16 wideband input: complex int16, I/Q interleaved (the nrsc5b_push_cs16 layout), at 23 814 000 S/s; 16 bits hold
 * the 40-60 dB between a band's stations that 8 bits cannot.  The same taps W_k, phasor table P, N(T), carry rule and
 * mixer index as cu8, no offset and unit gain (1 output LSB per input LSB):
 *     acc = sum_{u<256} W_k[u] * x[32 n + u]   (exact, |acc| < 2^36);   v = sat16((acc + 2^18) >> 19);
 *     y[k][n] = sat16((v * conj(P[(1600 m_k n) mod 11907]) + 2^14) >> 15)
 * For x16 = 64 (x8 - 127) the output equals the cu8 output on x8 bit for bit ((64 a + 2^18) >> 19 == (a + 2^12) >> 13,
 * and on cu8 input |v| < 2^15).  On cs16 input near full scale |v| can reach about 2^16; sat16 clamps it there.
 * The format is fixed at create: a cu8 entry point called on a cs16 handle, or a cs16 one on a cu8 handle, returns
 * NRSC5B_EINVAL and changes nothing.  nrsc5b_chan_destroy / _reset / _tables / _outputs are shared: the outputs of a
 * capture of nvalues int16 values are nrsc5b_chan_outputs(nvalues) (nvalues / 2 samples, as nbytes / 2 for cu8).
 * nvalues must be even (whole complex samples).  A cs16 handle owns 32 MiB + 2 KiB of device scratch, whatever the
 * capture size: a staging buffer of 2^22 + 256 samples and the two byte planes (x = 256 x_hi + x_lo) the tensor cores
 * read, made from it or from the caller's capture by a split pass. */
int nrsc5b_chan_create_cs16(nrsc5b_channelizer_t **out, int device, const int *offsets_100khz, int nch);
/* host capture of nvalues int16 values -> host out[nch][2 * outputs]; synchronous (tests) */
int nrsc5b_chan_run_cs16(nrsc5b_channelizer_t *c, const int16_t *cs16, size_t nvalues, int16_t *out);
/* device capture (16-byte aligned) -> device out[nch][out_stride] as nrsc5b_chan_run_device writes it; asynchronous
 * on cuda_stream.  The capture is only read (split into the handle's planes 2^17 outputs at a time). */
int nrsc5b_chan_run_device_cs16(nrsc5b_channelizer_t *c, const void *d_cs16, size_t nvalues, void *d_out, size_t out_stride,
                                void *cuda_stream);
/* nrsc5b_chan_push / nrsc5b_chan_feed for cs16: the same rules, nvalues int16 values (any alignment, host or device) */
int nrsc5b_chan_push_cs16(nrsc5b_channelizer_t *c, const int16_t *cs16, size_t nvalues, void *d_out, size_t out_stride,
                          void *cuda_stream, long long *nout);
int nrsc5b_chan_feed_cs16(nrsc5b_channelizer_t *c, nrsc5b_engine_t *e, const int *streams, const int16_t *cs16, size_t nvalues);

/* AM band plan: one cu8 or cs16 capture at 32 x 46 511.71875 = 1 488 375 S/s - the rate the reference asks of an AM
 * device; it spans +-744 kHz, the whole medium-wave band - -> `nch` AM channels at 46 511.71875 S/s cs16, the format an
 * NRSC5B_MODE_AM engine created with input_cs16 = 1 takes.  Channel k is centred `offsets_10khz[k]` x 10 kHz from the
 * capture's centre; offsets beyond +-74 are outside the capture: NRSC5B_EINVAL.  10 kHz / 1 488 375 Hz = 80 / 11907, so
 * the phasor table P is the FM plan's; the filter has 512 taps (h_am: Kaiser-windowed sinc, -6 dB at 23 kHz, beta 8.8,
 * unit DC gain; the integer taps of channel 0 are within +-0.001 dB up to 15 kHz and 87.1 dB down from 31.5 kHz on,
 * where the stations that alias onto a channel after the decimation by 32 begin).  Integer-exact definition:
 *     W_k[u]  = round(2^19 h_am[511-u] conj(P[(80 m_k u) mod 11907]) / 32767)
 *     cu8:   acc = sum_{u<512} W_k[u] (x[32 n + u] - (127+127j));  v = (acc + 2^12) >> 13
 *     cs16:  acc = sum_{u<512} W_k[u]  x[32 n + u];                v = sat16((acc + 2^18) >> 19)
 *     y[k][n] = sat16((v conj(P[(2560 m_k n) mod 11907]) + 2^14) >> 15)
 *     N_am(T) = T >= 512 ? (T - 512) / 32 + 1 : 0;   carry = the samples from 32 N_am(T) on (at most 511 samples:
 *     1022 bytes of cu8, 2044 of cs16)
 * The cu8 gain is 64 output LSB per input LSB, as in the FM plan (the reference's own AM cu8 path has 128; the AM
 * receiver normalises on its carrier and training symbols).  For x16 = 64 (x8 - 127) the cs16 output equals the cu8
 * output bit for bit.
 * The plan is fixed at create, like the sample format.  Every other entry point (nrsc5b_chan_run*, _push*, _feed*,
 * _tables, _reset, _destroy) is shared and behaves as documented above with 512 taps and N_am(T): nrsc5b_chan_tables
 * returns taps[nch][512][2], and nrsc5b_chan_feed* takes exactly an NRSC5B_MODE_AM engine with input_cs16 = 1 that reads
 * its own buffers (an FM handle on an AM engine, an AM handle on an FM engine, an AM engine created for cu8 input:
 * NRSC5B_EINVAL, nothing changed).
 * A stream fed from a channel that holds exact zeros (a digitally silent channel of a synthetic capture) behaves as
 * the reference does on such input: its carrier regression divides by the previous symbol's centre bin (reference
 * src/acquire.c:199-201) and stays NaN from then on; nrsc5b_reset(e, stream) recovers it.  A real capture's noise
 * floor keeps clear of that. */
int nrsc5b_chan_create_am(nrsc5b_channelizer_t **out, int device, const int *offsets_10khz, int nch);
int nrsc5b_chan_create_am_cs16(nrsc5b_channelizer_t **out, int device, const int *offsets_10khz, int nch);
/* the AM plan's tables without a device: taps[nch][512][2], phasor[11907][2] (the FM table); either may be NULL */
int nrsc5b_chan_make_tables_am(const int *offsets_10khz, int nch, int16_t *taps, int16_t *phasor);
/* output samples per channel of an AM-plan capture of nbytes (cu8; cs16: int16 values): nbytes / 64 - 15 for
 * nbytes % 64 == 0 */
long long nrsc5b_chan_outputs_am(size_t nbytes);

/* FM plans for narrower captures: one cu8 or cs16 capture at fs = D x 744 187.5 S/s, D = decim in {8, 16, 32}
 * (5 953 500, 11 907 000 or 23 814 000 S/s) -> `nch` FM channels at 744 187.5 S/s cs16, the same output as the FM plan
 * above.  Channel k is centred offsets_100khz[k] x 100 kHz from the capture's centre.  Integer-exact definition (m_k
 * the offset, h_D the plan's 256-tap prototype, unit DC gain):
 *     W_k[u] = round(2^14 D h_D[255-u] conj(P[((1600 / D) m_k u) mod 11907]) / 32767)         u < 256
 *     cu8:   acc = sum_u W_k[u] (x[D n + u] - (127+127j));   v = (acc + 2^(s-1)) >> s,          s = 13 - log2(32 / D)
 *     cs16:  acc = sum_u W_k[u]  x[D n + u];                 v = sat16((acc + 2^(t-1)) >> t),   t = 19 - log2(32 / D)
 *     y[k][n] = sat16((v conj(P[(1600 m_k n) mod 11907]) + 2^14) >> 15)
 *     N_D(T) = T >= 256 ? (T - 256) / D + 1 : 0;   carry = the samples from D N_D(T) on (at most 255)
 * D = 32 is exactly the FM plan: nrsc5b_chan_create_fm(out, device, 32, ...) is nrsc5b_chan_create(out, device, ...).
 * The tap scale 2^14 D keeps the largest tap near 16 380 for every D (the prototype's -6 dB point stays at 372 kHz, so
 * its peak doubles each time D halves); the shifts keep the gain at 64 output LSB per cu8 LSB and 1 per cs16 LSB, and
 * for x16 = 64 (x8 - 127) the cs16 output equals the cu8 output bit for bit.  h_D is a Kaiser-windowed sinc, -6 dB at
 * 372 kHz, beta 9 for D = 16 and 8; its integer taps for channel 0 are within 0.001 dB over +-200 kHz and 85.4 dB
 * (D = 16) and 80.2 dB (D = 8) down from 544 kHz on.  Offsets must lie inside the capture: |m_k| <= 59 for D = 16,
 * <= 29 for D = 8; otherwise, and for a decim not in {8, 16, 32}: NRSC5B_EINVAL.  Every other entry point
 * (nrsc5b_chan_run*, _push*, _feed*, _tables, _reset, _destroy) is shared and behaves as documented above with D in
 * place of 32: nrsc5b_chan_feed* takes an FM cs16 engine. */
int nrsc5b_chan_create_fm(nrsc5b_channelizer_t **out, int device, int decim, const int *offsets_100khz, int nch);
int nrsc5b_chan_create_fm_cs16(nrsc5b_channelizer_t **out, int device, int decim, const int *offsets_100khz, int nch);
/* the plan's tables without a device: taps[nch][256][2], phasor[11907][2]; either may be NULL */
int nrsc5b_chan_make_tables_fm(int decim, const int *offsets_100khz, int nch, int16_t *taps, int16_t *phasor);
/* output samples per channel of a capture of nbytes (cu8; cs16: int16 values) at D = decim: nbytes / 64 - 7 (D = 32),
 * nbytes / 32 - 15 (D = 16), nbytes / 16 - 31 (D = 8) for nbytes % 64 == 0; NRSC5B_EINVAL for any other decim */
long long nrsc5b_chan_outputs_fm(int decim, size_t nbytes);

/* A capture at the radio's own rate: fs = rate_hz (integer Hz) -> the plan's capture rate R = D x 744 187.5 S/s (mode
 * NRSC5B_MODE_FM, D = decim in {8, 16, 32}) or 1 488 375 S/s (NRSC5B_MODE_AM, decim = 32) through an exact polyphase
 * resampler, then the plan's cs16 definition above, unchanged, on the result.  With R / fs = L / M in lowest terms:
 *     b_n = floor(n M / L),  p_n = n M mod L
 *     y[n] = sat16((sum_{j<64} G[p_n][j] x[b_n + j] + 2^13) >> 14)       (cu8 input: x = 64 (x8 - 127))
 *     K(T) = T >= 64 ? ((T - 63) L - 1) / M + 1 : 0;   outputs of T input samples: N_plan(K(T))
 * G[L][64] (nrsc5b_chan_resampler_tables): a Kaiser-windowed sinc (beta 8.41) designed at L fs, -6 dB at min(fs, R) / 2,
 * split into L phases of 64 taps, each rounded to sum exactly 2^14 (unit DC gain) with sum |G[p]| < 2^16 (so the int32
 * accumulation is exact).  The largest per-phase gain is about 2.8: full-scale cs16 input saturates y, as sat16 says.
 * A cu8 handle equals a cs16 handle fed 64 (x8 - 127), bit for bit.
 * Accepted: R / 32 <= fs <= 4 R and L <= 11 907 (every multiple of 2 kHz at D = 32, 1 kHz at D = 16, 500 Hz at D = 8,
 * 125 Hz for AM).  The usable band is |f| <= f_p = (min(fs, R) - 11 fs / 128) / 2; a channel must lie inside it,
 * |m| x 100 kHz + 200 kHz (FM) or |m| x 10 kHz + 15 kHz (AM) <= f_p, as well as inside the plan's own range.  Largest
 * |offset| (nrsc5b_chan_resampler_tables), FM at every D it takes unless noted: 2.048 MS/s: 7; 2.4 MS/s: 8; 2.5 MS/s:
 * 9; 3 MS/s: 11; 6 MS/s: 25; 8 MS/s: 24 (D = 8), 34; 10 MS/s: 23 (D = 8), 43; 20 MS/s: 19 (D = 8), 48 (D = 16),
 * 89 (D = 32); 30.72 MS/s: 44 (D = 16), 103 (D = 32); 61.44 MS/s: 90 (D = 32).  AM: 768 kS/s: 33; 912 kS/s: 40;
 * 2.4 MS/s: 62.
 * Anything else: NRSC5B_EINVAL.  fs == R returns the plan's own handle (no stage), as nrsc5b_chan_create_fm does.
 * Every other entry point (nrsc5b_chan_run*, _push*, _feed*, _tables, _reset, _destroy) is shared and keeps its rules,
 * T counting input samples at fs; pushing a capture in pieces of any even size gives the one-shot output bit for bit.
 * The one-shot entry points use every complex sample in both formats (no whole 64-byte rows), and one-shot device
 * input needs 16-byte alignment only.  nrsc5b_chan_feed* takes the plan's engine (FM or AM, cs16, own buffers).
 * Device scratch of a handle with a stage, whatever the capture size: 32 MiB + 2 KiB of staging and planes (as a cs16
 * handle), 2 KiB for the streamed resampled carry (kept apart from the planes, so that a one-shot call between pushes
 * leaves the stream as it was) and the table, L x 128 bytes (at most 1.5 MB). */
int nrsc5b_chan_create_rate(nrsc5b_channelizer_t **out, int device, int mode, int decim, uint32_t rate_hz, const int *offsets, int nch);
int nrsc5b_chan_create_rate_cs16(nrsc5b_channelizer_t **out, int device, int mode, int decim, uint32_t rate_hz, const int *offsets,
                                 int nch);
/* L, M, the largest usable |offset| and G[L][64] (may be NULL; any pointer may be NULL); no device needed.  fs == R:
 * L = M = 1, the plan's own offset limit (0: none) and G the identity row. */
int nrsc5b_chan_resampler_tables(int mode, int decim, uint32_t rate_hz, int *L, int *M, int *max_offset, int16_t *G);
/* N_plan(K(T)) for T = samples input samples at fs; NRSC5B_EINVAL for a rate the library does not take */
long long nrsc5b_chan_outputs_rate(int mode, int decim, uint32_t rate_hz, long long samples);
/* The rate stage alone (kernel-level parity): host capture of nvalues cu8 bytes (cs16 = 0) or int16 values (cs16 = 1)
 * -> host out[2 K(T)], y[0 .. K(T) - 1] I/Q interleaved; synchronous.  fs == R: NRSC5B_EINVAL (no stage). */
int nrsc5b_resample(int device, int mode, int decim, uint32_t rate_hz, int cs16, const void *in, size_t nvalues, int16_t *out);
/* The rate stage of a rate handle's one-shot device path alone (to time it apart from the channel bank): the k_resample
 * launches nrsc5b_chan_run_device* makes for this capture (nvalues cu8 bytes or cs16 values, the handle's format,
 * 16-byte aligned), into the handle's own scratch; no channel output.  NRSC5B_EINVAL on a handle without a stage. */
int nrsc5b_chan_resample_device(nrsc5b_channelizer_t *c, const void *d_in, size_t nvalues, void *cuda_stream);

/* ---- band scan: which channels carry an NRSC-5 signal (the reference has no counterpart; the nearest thing is the
 * coarse acquisition of one stream, reference src/acquire.c:120-158: band-pass, fold the cyclic-prefix correlation
 * over 32 symbols, take the arg-max) ----
 * Input: channel output y[n], complex int16, what nrsc5b_chan_* writes: FM channels at 744 187.5 S/s, AM channels at
 * 46 511.71875 S/s.  Per mode, lag F (the FFT length), CP length P, symbol S = F + P, subsampling q and the sidebands:
 *     FM: F = 2048, P = 112, S = 2160, q = 4; carriers -478..-356 / +356..+478 (129.4 - 173.7 kHz), in the primary
 *         main partitions every FM service mode has.  Not the whole partition (up to carrier 546, 198.4 kHz): a station
 *         400 kHz away has its own sideband from 202 kHz on, and 64 taps need about 28 kHz for 40 dB, so the band stops
 *         short of it as it stops short of the channel's own analogue host (100 kHz)
 *     AM: F = 256,  P = 14,  S = 270,  q = 2; carriers -81..-33 / +33..+81 (6.0 - 14.7 kHz).  The inner carriers
 *         2..32 lie under a hybrid (MA1) station's analogue audio, far stronger than they are, and in an all-digital
 *         (MA3) station their lag-F correlation comes out with the wrong sign (measured -0.50 per unit energy over
 *         0.36 - 5 kHz against +0.58 and +0.66 over 5 - 10 and 10 - 15 kHz), which would put the CFO half a
 *         subcarrier off
 * With g_U[u], u < 64, the upper sideband's Q15 taps (nrsc5b_scan_make_tables) and g_L = conj(g_U), for s in {L, U}:
 *     z_s[n]    = sat16((sum_u g_s[u] y[n - 63 + u] + 2^14) >> 15)      per component, n = 0 (mod q), n >= 63
 *     p_s[n]    = z_s[n] conj(z_s[n + F]),   e_s[n] = |z_s[n]|^2 + |z_s[n + F]|^2          exact in int64
 *     Fold_s[j] = sum_m p_s[q j + m S],      En_s[j] likewise                                j < J = S / q
 *     C_s[j]    = sum_{i < P/q} Fold_s[(j + i) mod J],   E_s[j] likewise over En_s
 * n counts from the first sample the scan was given; a product counts once both its samples have been (n + F < T, T
 * the samples pushed since create / reset).  |Re p|, |Im p| <= 2^31 and e <= 2^32, so Fold and En fit int64 up to 2^24
 * symbols: a push that takes T / S beyond 2^24 returns NRSC5B_EINVAL and changes nothing.
 * Taps: a Kaiser-windowed sinc low-pass moved to the sideband, unit passband gain (Q15: 32768), sum |Re g| and
 * sum |Im g| below 2^16.  FM: centred on 151 kHz, -6 dB 37 kHz either side, >= 40 dB down at |f| <= 100 kHz (the
 * channel's own analogue host) and at f >= 202 kHz (the sideband of a station 400 kHz away; measured 41.3 dB both),
 * within 0.5 dB over carriers 356..478 (measured 0.13 dB).  AM: centred on
 * 10.4 kHz, -6 dB 5 kHz either side, with the window subtracted in proportion so that sum g = 0 exactly: an exact null
 * at DC (the analogue carrier), flat within 0.5 dB over 6.5 - 14 kHz (measured 0.11 dB; 64 taps at 46.5 kS/s cannot
 * resolve a sharper edge) and 15.6 dB down at 5 kHz.
 * Metrics (nrsc5b_scan_result; in double, ties to the smallest j; phi = q j):
 *     C = C_L + C_U, mean C' = sum_j C[j] / J, j* = argmax_j |C[j] - C'|: the mean removes every stationary component
 *         in expectation (tones, spurs, an analogue host, a neighbour's host inside the sideband); a CP-periodic (OFDM)
 *         signal survives
 *     score     = |C[j*] - C'| / (1/2 (E_L + E_U)[j*])
 *     symbols   M = N_p q / S, N_p the products counted per sideband
 *     score_s   = |C_s[j*] - C'_s| / (1/2 E_s[j*]), each sideband at the timing found
 *     threshold tau(M) = c / sqrt(M P / q),  threshold_sideband tau_1(M) = c1 / sqrt(M P / q)
 *     detected  = M >= 32 and score >= tau(M) and score_L >= tau_1(M) and score_U >= tau_1(M) and
 *               Re(D_L conj(D_U)) >= cos(45 deg) |D_L| |D_U|, D_s = C_s[j*] - C'_s
 *               Both sidebands must carry the CP correlation: a station's one sideband also falls into the filter
 *               of the channel 300 kHz (FM; AM: 20 kHz) beside it - its upper sideband, +129..+198 kHz, is the lower
 *               passband, -174..-129 kHz, of the channel 300 kHz above - where the combined score alone reaches
 *               almost the station's own; there the other sideband holds no correlation at that timing.  And both
 *               must agree in phase: the two sidebands of one station share its carrier, so their correlations share
 *               its CFO, while an AM channel 10 kHz beside a station takes the station's inner carriers into one
 *               filter and its spectrum beyond 15 kHz into the other (measured 53 - 63 degrees apart on synthetic MA1
 *               and MA3 stations 60 dB over the noise, against at most 11 degrees in the stations' own channels).
 *               What still holds: (1) a channel whose two sidebands take one sideband each of two stations with the
 *               same symbol timing (to within the window) and CFO would pass; independent stations share neither on
 *               purpose, so this needs two transmitters locked to each other 600 kHz (AM: 40 kHz) apart.  (2) The
 *               stopbands are about 40 dB: a station some 45 dB or more over the noise leaks into both filters of the
 *               channels 100 kHz (AM: 10 - 20 kHz) beside it, with its own timing and phase, and can be detected
 *               there too; its score there stays far below the station's own.
 *     timing    = (q j* - 32) mod S: the first CP sample of a symbol in the channel's own sample index (the taps' group
 *               delay of 31.5 samples removed)
 *     cfo_hz    = -arg(C[j*] - C') fs / (2 pi F): the CFO within +-1/2 subcarrier, in the channel's own spectrum
 *     rho_s     = |C_s[j*] - C'_s| / (1/2 mean_j E_s[j]);  snr_db_s = 10 log10(rho_s / (kappa - rho_s)), -inf / +inf
 *               outside (0, kappa).  The energy averaged over all timings, not E_s[j*]: the pulse shape (reference
 *               src/acquire.c:320-342) halves the signal's energy at the CP while the noise stays uniform.
 *     power_dbfs = 10 log10(mean |y|^2 / 2^30) over the samples given; power_dbfs_lower / _upper likewise of z_s over
 *               the products' samples (sum_j En_s[j] / 2 N_p)
 * c: under noise alone, z_s is complex Gaussian and C - C' a sum of N = M P / q products, so score = R sqrt(gamma / 2N)
 * with R^2 ~ Exp(1) and gamma = sum_k |r(k q)|^2 the products' correlation (r: the normalised autocorrelation of g_U;
 * 2.542 FM, 2.342 AM).  Treating the J positions as independent (neighbours are correlated, so this errs on the safe
 * side), P(max R > r) = J e^(-r^2) = 1e-6 per channel gives r^2 = ln(1e6 J) and c = sqrt(gamma ln(1e6 J) / 2).
 * c1: for one sideband at a given timing (not a maximum over J), score_s = R sqrt(gamma / N), and P(R > r) = e^(-r^2)
 * = 1e-3 gives c1 = sqrt(gamma ln(1e3)): with the 1e-6 of tau(M) in front of it, a sideband that holds only noise
 * passes tau_1 once in a thousand, while a station at -3 dB per sideband passes it in half a second.
 * kappa: the mean of rho_L and rho_U for a noise-free synthetic station (the pulse shape's 1/pi, less the filter's
 * spread), measured with the numpy restatement (tests/scan_oracle.py) on one MP1 frame (1.49 s, decimated from the
 * generator's 1 488 375 S/s; FM: 0.3163 and 0.3042) and four MA3 frames (AM: 0.3145 and 0.3107). */
#define NRSC5B_SCAN_C_FM 5.055
#define NRSC5B_SCAN_C_AM 4.682
#define NRSC5B_SCAN_C1_FM 4.190
#define NRSC5B_SCAN_C1_AM 4.022
#define NRSC5B_SCAN_KAPPA_FM 0.310
#define NRSC5B_SCAN_KAPPA_AM 0.313
/* raw int64 values per channel of nrsc5b_scan_result: Fold_L re, im, En_L, Fold_U re, im, En_U, then C_L re, im, E_L,
 * C_U re, im, E_U, each [J]; then sum |y|^2 as two uint64 words (low, high).  J = 540 (FM), 135 (AM). */
#define NRSC5B_SCAN_RAW(J) (12 * (J) + 2)
typedef struct {
    double score, threshold, symbols, cfo_hz;
    double score_lower, score_upper, threshold_sideband;
    double snr_db_lower, snr_db_upper;
    double power_dbfs, power_dbfs_lower, power_dbfs_upper;
    int32_t detected;
    int32_t timing;
} nrsc5b_scan_t;
typedef struct nrsc5b_scanner nrsc5b_scanner_t;
/* A scanner of `nch` channels of mode NRSC5B_MODE_FM or NRSC5B_MODE_AM; NRSC5B_ENODEV without a device. */
int nrsc5b_scan_create(nrsc5b_scanner_t **out, int device, int mode, int nch);
void nrsc5b_scan_destroy(nrsc5b_scanner_t *s);
/* Start over: T = 0, every accumulator 0. */
int nrsc5b_scan_reset(nrsc5b_scanner_t *s);
/* The next nsamples of every channel: device memory [nch][stride] int16 values (4-byte aligned, stride even and
 * >= 2 nsamples), asynchronous on cuda_stream (a cudaStream_t cast to void*, NULL = default).  The handle keeps the
 * last F + 63 samples of every channel, so a capture pushed in pieces of any size gives every accumulator of the
 * one-shot scan bit for bit. */
int nrsc5b_scan_push_device(nrsc5b_scanner_t *s, const void *d_ch, size_t stride, size_t nsamples, void *cuda_stream);
/* The same from host memory [nch][2 nsamples]; synchronous (tests). */
int nrsc5b_scan_push(nrsc5b_scanner_t *s, const int16_t *cs16, size_t nsamples);
/* The metrics of every channel so far (out[nch]); raw (optional): [nch][NRSC5B_SCAN_RAW(J)] the exact sums.  Waits for
 * the pushes; the scan goes on from where it is. */
int nrsc5b_scan_result(nrsc5b_scanner_t *s, nrsc5b_scan_t *out, int64_t *raw);
/* Channelise and scan: the capture (nvalues cu8 bytes or cs16 values, the handle's format, host or device memory) goes
 * through the channeliser's streaming push (nrsc5b_chan_push*: every plan, decim and rate handle) into the scanner's
 * own device buffer and from there into the scan, piece by piece, on the default CUDA stream; no channel output comes
 * back to the host.  The scanner must have the plan's mode, device and channel count (channel k = the plan's channel
 * k); otherwise, for odd nvalues, or if the scan would pass 2^24 symbols: NRSC5B_EINVAL, neither handle changed.  The
 * scanner's buffer is 2^18 bytes per channel, allocated at the first call. */
int nrsc5b_chan_scan(nrsc5b_channelizer_t *c, nrsc5b_scanner_t *s, const void *capture, size_t nvalues);
/* The upper sideband's taps[64][2] (Re, Im of g_U; g_L = conj(g_U)) and kappa for the mode, without a device. */
int nrsc5b_scan_make_tables(int mode, int16_t *taps, double *kappa);

/* ---- band receiver: every HD Radio station of a live wideband capture decoded, engines attached and detached as the
 * scan finds and loses stations (the reference has no counterpart: it takes one narrowband device per handle,
 * reference src/nrsc5.c:130-207) ----
 * One handle owns a channeliser of the plan (nrsc5b_chan_create_fm / _am / _rate, cu8 or cs16), a scanner of its
 * channels and one cs16 engine of the plan's mode with max_stations streams (nrsc5b_enable_l2 if l2 != 0).
 * Pipeline, per push of any size:
 *   1. Every channel is channelised once (nrsc5b_chan_push*) into a device window buffer of W = window_symbols x S
 *      samples per channel (S = 2160 FM, 270 AM).  The capture is split so that windows fill exactly (a rate stage's
 *      one input sample can emit several outputs; those past W open the next window).  Channel sample n counts the
 *      plan's outputs from the first sample pushed; window w holds n in [wW, (w+1)W).
 *   2. A full window gets a verdict: nrsc5b_scan_push_device of its W samples, nrsc5b_scan_result, nrsc5b_scan_reset.
 *      Window w's rows are exactly the one-shot scan of channel samples [wW, (w+1)W); the scan's 2^24-symbol bound
 *      never applies (a window is at most 512 symbols).
 *   3. The policy, on the host, once per window, in this order:
 *      Suppression.  A detected channel k is leakage if some other detected channel j has |m_j - m_k| <= r (r = 1 FM,
 *        2 AM, in grid steps), a higher score (equal scores: the smaller m wins) and a timing within P / 2 samples
 *        mod S (56 FM, 7 AM; P the cyclic prefix).  A station some 45 dB or more over the noise is detected in the
 *        channels beside it too, with its own timing (case (2) of the scan's "What still holds"); this takes those out.
 *        The timing found there wanders with the leaked content: on synthetic FM stations 60 dB over the noise it came
 *        out more than the scan's 2q (8 samples) off the station's own, and a tolerance of 2q opened a second session
 *        on the neighbour.  P / 2 is the top half of the CP window sum's triangle around the station's timing.
 *        Present = detected and not leakage.  Not covered: an AM channel 10 kHz beside an MA1 station scores above the station itself (about 1.2
 *        against 0.6 on a synthetic MA1 station) and is normally refused by the scan's phase rule; in a
 *        window where it passes, this rule keeps the neighbour and flags the station as leakage.
 *      Detach.  A session whose channel has not been present in hold_windows consecutive windows closes: n1 = the end
 *        of its last routed window (wW in window w), the engine runs, its records are drained into the session, the
 *        stream is reset (nrsc5b_reset) and freed.  A channel present again later opens a new session.
 *      Attach.  A present channel without a session gets the lowest free engine stream; its session starts at the
 *        start of this window, n0 = wW: the window is kept until its verdict, so no sample of it is lost.  No stream
 *        free: the channel's row is flagged NRSC5B_BAND_NO_SLOT.  Channels are taken in index order.
 *   4. Route: k_band_route appends the window's samples of every open session's channel to its engine stream, on the
 *      engine's CUDA stream, one launch per window; no channel data passes through the host.  A stream without room
 *      (its 4 MiB input buffer; a 512-symbol FM window is 4.4 MB) makes the engine run, and the route goes on in
 *      pieces: no sample is dropped.
 *   5. nrsc5b_process, then every open session's records are drained into a host buffer of its own.  A stream's record
 *      log (2 MiB) holds what one window's processing can emit; should it ever overflow, the push fails with
 *      NRSC5B_EOVERFLOW instead of truncating.
 * So a session's records are those of a cs16 engine of the same mode (and L2 setting) given channel samples
 * [n0, n1) by nrsc5b_push_cs16 and processed, except the positions in REC_BLOCK, which count from where the stream's
 * input buffer was last trimmed.  REC_L2's frame_off counts from the start of each nrsc5b_band_records output. */
typedef struct nrsc5b_band nrsc5b_band_t;
typedef struct {
    int device, mode, decim;        /* NRSC5B_MODE_FM: decim 8 | 16 | 32; NRSC5B_MODE_AM: 32 */
    uint32_t rate_hz;               /* 0: the plan's own rate, else the rate stage (nrsc5b_chan_create_rate*) */
    int input_cs16;
    const int *offsets; int nch;    /* NULL (nch = 0): every grid point the plan (and rate) takes, -lim ..= lim with lim =
                                     * 117 / 59 / 29 (FM, D = 32 / 16 / 8) or 74 (AM), or the rate stage's largest usable
                                     * |offset| where it is smaller.  Otherwise distinct offsets within that range */
    int window_symbols;             /* 32 ..= 512 */
    int hold_windows;               /* >= 1 */
    int max_stations;               /* engine streams, 1 ..= 4096 */
    int l2;
} nrsc5b_band_config_t;
enum {
    NRSC5B_BAND_DETECTED = 1,       /* the scan's verdict */
    NRSC5B_BAND_LEAKAGE = 2,        /* detected, but a stronger neighbour's leakage (not present) */
    NRSC5B_BAND_ATTACHED = 4,       /* a session holds the channel after this window's policy: the window is routed to it */
    NRSC5B_BAND_NO_SLOT = 8,        /* present without a session, and no engine stream was free */
};
typedef struct {
    int32_t id;                     /* 0, 1, ... in the order sessions open */
    int32_t channel, offset;        /* channel index and its offset (grid steps) */
    int32_t slot;                   /* engine stream; -1 once closed */
    int64_t n0, n1;                 /* channel samples [n0, n1) went to the engine; n1 = -1 while open */
    int64_t window;                 /* the window whose verdict opened it (n0 = window x W) */
    nrsc5b_scan_t verdict;          /* that window's row of the channel */
} nrsc5b_band_session_t;
/* EINVAL for a bad config (checked first, without a device), ENODEV without a device. */
int nrsc5b_band_create(nrsc5b_band_t **out, const nrsc5b_band_config_t *cfg);
void nrsc5b_band_destroy(nrsc5b_band_t *b);
/* The next nvalues of the capture: cu8 bytes or cs16 int16 values (the config's format), host or device memory, even.
 * Synchronous: returns once the capture has been read (the buffer may be reused at once, page-locked and device memory
 * included) and every window it completes has been scanned, routed and processed.  Odd nvalues, or a push after
 * nrsc5b_band_flush: NRSC5B_EINVAL, nothing changed. */
int nrsc5b_band_push(nrsc5b_band_t *b, const void *capture, size_t nvalues);
/* End of the capture: the partial window is routed (it gets no verdict), the engine runs and every session closes at
 * n1 = the last channel sample.  Later pushes are refused; a second flush does nothing. */
int nrsc5b_band_flush(nrsc5b_band_t *b);
/* Takes up to cap completed windows, oldest first: index[i], rows[i][nch], flags[i][nch] (NRSC5B_BAND_*; any pointer
 * may be NULL).  Returns the number taken; *pending (may be NULL) = windows waiting before the call.  Windows wait here
 * until taken (about 100 bytes per channel each: some 0.2 GB an hour for 235 FM channels at 128 symbols), so a
 * long-running caller takes them; one that does not want them discards them with index, rows and flags NULL and cap
 * at least the pending count. */
int nrsc5b_band_windows(nrsc5b_band_t *b, int64_t *index, nrsc5b_scan_t *rows, uint32_t *flags, int cap, int *pending);
/* Every session opened so far, by id (not drained): writes min(cap, *n) and returns that number. */
int nrsc5b_band_sessions(nrsc5b_band_t *b, nrsc5b_band_session_t *out, int cap, int *n);
/* Session id's records since the last call, in the engine's record format; as nrsc5b_drain: returns the bytes
 * written, *needed = the bytes waiting, NRSC5B_EFULL (nothing taken) if cap is smaller.  A closed session's buffer is
 * freed once taken. */
long nrsc5b_band_records(nrsc5b_band_t *b, int id, uint8_t *out, size_t cap, size_t *needed);
/* The channel offsets (offsets[nch], may be NULL) and their number. */
int nrsc5b_band_channels(nrsc5b_band_t *b, int *offsets, int *nch);
/* Device time per stage since create, from CUDA events on the handle's work: ms4 = {channelise (nrsc5b_chan_push*),
 * scan (push, result, reset: readback included), route (k_band_route), engine (nrsc5b_process)}; route_bytes = bytes
 * k_band_route read and wrote. */
int nrsc5b_band_times(nrsc5b_band_t *b, double *ms4, unsigned long long *route_bytes);

const char *nrsc5b_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NRSC5_B200_H */
