/* The seven input_* functions of the reference (src/input.c:96-188, declared src/input.h:37-43) on top of
 * the CUDA engine's C ABI (include/nrsc5_b200.h).  Linked with the reference's unmodified host-side
 * sources this gives a libnrsc5.so whose public API and event order are the reference's.
 *
 * input_push_cu8() never waits for the GPU: it copies the samples into the engine's page-locked staging area
 * (nrsc5b_stage_cu8, no CUDA call), replays the records of a batch that has finished meanwhile - in the reference's
 * call order, into frame_push() / pids_frame_push() / nrsc5_report_*() / output_advance() on the calling thread -
 * and, if the samples buffered by now complete a block and no batch is in flight, enqueues the next one
 * (nrsc5b_submit).  A push that completes no block (16 of 17 at the CLI's 32 768-byte pushes) makes no CUDA call at
 * all.  A source that delivers in real time finds every batch finished by its next push (a block takes the GPU
 * ~0.1 ms); a file is decoded as fast as the GPU goes, the pushes running ahead.  input_free() (nrsc5_close) and
 * input_reset() wait for what is in flight and deliver it: nothing is lost at the end of a stream.
 * NRSC5_B200_SYNC=1 restores the strictly synchronous behaviour (every push returns only after everything it
 * completed has been delivered), as does NRSC5_B200_DEVICE_L2=0, whose host-side L2 feeds back into the engine.
 *
 * L2 framing runs on the GPU as well (nrsc5b_enable_l2, csrc/l2.cuh).  The engine's REC_L2 record of a frame
 * holds what the reference's frame_process() (src/frame.c:516-643) would have called, in order; replay() makes
 * those calls - nrsc5_report_audio_service / output_align / output_aas_push / output_push - instead of
 * frame_push(), so the host does no L2 parsing.  NRSC5_B200_DEVICE_L2=0 puts the reference's own frame.c back on
 * the path (A/B checks).
 */
#include "config.h"

#include <assert.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "defines.h"
#include "input.h"
#include "private.h"

#include "nrsc5_b200.h"

/* Samples buffered on the GPU.  A file is pushed faster than it is decoded, so the buffer holds the part of the stream
 * the pushes are ahead by; when it is full the engine drops what the receiver's window has passed (a synchronous
 * step, once per buffer) and, if that frees nothing, the push waits for the batch in flight.  HBM is not scarce:
 * 256 MiB = 58 L1 frames of cu8.  (A real-time source never gets ahead by more than a block.) */
#define INPUT_CAPACITY (256u << 20)
#define RECORDS_CAPACITY (4u << 20)

static void fail(const char *what, int rc)
{
    fprintf(stderr, "libnrsc5 (GPU): %s failed (%d); there is no CPU path\n", what, rc);
    abort();
}

void input_set_sync_state(input_t *st, unsigned int new_state)
{
    /* reference src/input.c:172-188 for what the host side sees; the engine keeps the real state */
    if (st->sync_state == new_state)
        return;
    if (st->sync_state == SYNC_STATE_FINE)
        nrsc5_report_lost_sync(st->radio);
    st->sync_state = new_state;
    if (st->in_frame_push && st->engine)
    {
        /* frame.c:539 (L2 saw an audio frame whose header fails RS): the engine applies the same predicate
         * on the GPU; forcing the state covers the cases where the two disagree */
        int rc = nrsc5b_set_sync_state(st->engine, 0, (int)new_state);
        if (rc) fail("nrsc5b_set_sync_state", rc);
    }
}

static void unpack_bits(const uint8_t *packed, size_t nbits, uint8_t *bits)
{
    for (size_t i = 0; i < nbits; i++)
        bits[i] = (packed[i >> 3] >> (7 - (i & 7))) & 1;
}

/* the L2 -> L3 calls the device made of one frame (REC_L2 payload, include/nrsc5_b200.h), in call order */
static void replay_l2(input_t *st, const uint8_t *pay)
{
    uint32_t h[8];
    memcpy(h, pay, sizeof(h));
    const uint32_t flags = h[4], ev_len = h[6];
    const uint8_t *ev = pay + 32, *pdu = pay + 32 + ev_len;
    uint32_t off = 0;
    while (off + 8 <= ev_len)
    {
        uint32_t type, plen, v[8];
        memcpy(&type, ev + off, 4);
        memcpy(&plen, ev + off + 4, 4);
        const uint8_t *p = ev + off + 8;
        off += 8 + ((plen + 3) & ~3u);
        switch (type)
        {
        case 16:                                     /* frame.c:590 */
            memcpy(v, p, 32);
            nrsc5_report_audio_service(st->radio, v[0], v[1], v[2], v[3], v[4], (int)v[5], v[6], v[7]);
            break;
        case 17:                                     /* frame.c:606 */
            memcpy(v, p, 12);
            output_align(st->output, v[0], v[1], v[2]);
            break;
        case 18:                                     /* frame.c:365 */
            output_aas_push(st->output, (uint8_t *)p, plen);
            break;
        case 19:                                     /* frame.c:619-635 */
        {
            packet_ref_t ref;
            memcpy(v, p, 28);
            ref.program = v[0];
            ref.stream_id = v[1];
            ref.seq = v[2];
            ref.shape = v[3];
            ref.flags = v[4];
            ref.size = v[5];
            ref.data = (uint8_t *)pdu + v[6];
            output_push(st->output, &ref);
            break;
        }
        default:
            break;
        }
    }
    if (flags & 1)                                   /* frame.c:535-540: the first audio header of a P1 frame failed */
    {
        /* The engine applied this very predicate on the GPU when it decoded the frame and is long past it (batches
         * run ahead of the replay): only the host's view and the event follow here - forcing the engine's state now
         * would drop a sync it has regained since. */
        input_set_sync_state(st, SYNC_STATE_NONE);
    }
}

/* the REC_L2 record whose frame_off names the frame bits at `bits_off` of this drain */
static const uint8_t *find_l2(const uint8_t *rec, size_t n, size_t from, uint32_t bits_off)
{
    size_t off = from;
    while (off + 8 <= n)
    {
        uint32_t type, plen, frame_off;
        memcpy(&type, rec + off, 4);
        memcpy(&plen, rec + off + 4, 4);
        if (type == NRSC5B_REC_L2)
        {
            memcpy(&frame_off, rec + off + 8, 4);
            if (frame_off == bits_off)
                return rec + off + 8;
        }
        off += 8 + ((plen + 3) & ~3u);
    }
    return NULL;
}

static void replay(input_t *st, const uint8_t *rec, size_t n)
{
    size_t off = 0;
    while (off + 8 <= n)
    {
        uint32_t type, plen;
        memcpy(&type, rec + off, 4);
        memcpy(&plen, rec + off + 4, 4);
        const uint8_t *pay = rec + off + 8;
        off += 8 + ((plen + 3) & ~3u);
        switch (type)
        {
        case NRSC5B_REC_BLOCK:                       /* acquire.c:108 */
            output_advance(st->output);
            break;
        case NRSC5B_REC_SYNC:                        /* sync.c:403-409, input.c:180-186 */
        {
            float freq_offset;
            int psmi, flags[4] = { -1, -1, -1, -1 };     /* pli, hppi, aabi, rdbi: AM only (sync.c:230-236) */
            memcpy(&freq_offset, pay, 4);
            memcpy(&psmi, pay + 4, 4);
            if (plen >= 24) memcpy(flags, pay + 8, 16);
            if (st->sync_state == SYNC_STATE_FINE)
                nrsc5_report_lost_sync(st->radio);
            st->sync_state = SYNC_STATE_FINE;
            nrsc5_report_sync(st->radio, freq_offset, psmi, flags[0], flags[1], flags[2], flags[3]);
            pids_init(&st->pids, st);                /* decode_reset, decode.c:556-565 */
            frame_reset(&st->frame);
            break;
        }
        case NRSC5B_REC_PAD:                         /* an unused slot: no call */
            break;
        case NRSC5B_REC_LOST_SYNC:                   /* already reported if frame.c asked for it */
            if (st->sync_state == SYNC_STATE_FINE)
                nrsc5_report_lost_sync(st->radio);
            st->sync_state = SYNC_STATE_NONE;
            break;
        case NRSC5B_REC_MER:                         /* sync.c:490-497 */
        {
            float lo, up;
            memcpy(&lo, pay, 4);
            memcpy(&up, pay + 4, 4);
            nrsc5_report_mer(st->radio, lo, up);
            break;
        }
        case NRSC5B_REC_BER:                         /* decode.c:458 */
        {
            float cber;
            memcpy(&cber, pay, 4);
            nrsc5_report_ber(st->radio, cber);
            break;
        }
        case NRSC5B_REC_PIDS:                        /* decode.c:471 */
            unpack_bits(pay, 80, st->bits);
            pids_frame_push(&st->pids, st->bits);
            break;
        case NRSC5B_REC_FRAME:                       /* decode.c:460 */
        {
            uint32_t lc, nbits;
            memcpy(&lc, pay, 4);
            memcpy(&nbits, pay + 4, 4);
            if (st->device_l2)
            {
                /* L2 ran on the GPU at the end of the frame's pass: make its calls here, where frame_push() stood */
                const uint8_t *l2 = find_l2(rec, n, off, (uint32_t)(pay + 8 - rec));
                if (!l2) fail("REC_L2 of a frame", -1);
                replay_l2(st, l2);
                break;
            }
            unpack_bits(pay + 8, nbits, st->bits);
            st->in_frame_push = 1;
            frame_push(&st->frame, st->bits, nbits, (logical_channel_t)lc);
            st->in_frame_push = 0;
            break;
        }
        default:
            break;
        }
    }
}

static void engine_open(input_t *st, int cs16)
{
    const int am = st->radio->mode == NRSC5_MODE_AM;
    /* AM accepts both formats as well: cs16 at 46 511.72 S/s, or cu8 at 1 488 375 S/s which the engine decimates
     * by 32 on the device (src/input.c:71-89) */
    if (st->engine && st->engine_cs16 == cs16 && st->engine_am == am)
        return;
    /* the reference accepts cu8 and cs16 pushes on one handle; the engine is built for one format, so a
     * change of format starts a new engine (= input_reset) */
    if (st->engine)
        nrsc5b_destroy(st->engine);
    nrsc5b_config_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    const char *dev = getenv("NRSC5_B200_DEVICE");
    cfg.device = dev ? atoi(dev) : 0;
    cfg.nstreams = 1;
    cfg.mode = am ? NRSC5B_MODE_AM : NRSC5B_MODE_FM;
    cfg.input_capacity = INPUT_CAPACITY;
    cfg.log_capacity = RECORDS_CAPACITY;
    cfg.input_cs16 = cs16;
    int rc = nrsc5b_create(&st->engine, &cfg);
    if (rc) fail("nrsc5b_create", rc);
    st->engine_cs16 = cs16;
    st->engine_am = am;
    const char *dev_l2 = getenv("NRSC5_B200_DEVICE_L2");
    st->device_l2 = !(dev_l2 && !atoi(dev_l2));      /* default: on the device, FM and AM; 0: the reference's frame.c */
    st->trace = getenv("NRSC5_B200_TRACE") != NULL;
    const char *sync = getenv("NRSC5_B200_SYNC");
    st->pipelined = st->device_l2 && !(sync && atoi(sync));
    if (st->pipelined)
    {
        rc = nrsc5b_prepare_async(st->engine);       /* page-locked buffers now, not inside the first push */
        if (rc) fail("nrsc5b_prepare_async", rc);
    }
    if (st->device_l2)
    {
        rc = nrsc5b_enable_l2(st->engine, 1);
        if (rc) fail("nrsc5b_enable_l2", rc);
    }
}

static void run_and_replay(input_t *st)
{
    int rc = nrsc5b_process(st->engine);
    if (rc) fail("nrsc5b_process", rc);
    size_t need = 0;
    long got = nrsc5b_drain(st->engine, 0, st->records, st->records_cap, &need);
    if (got < 0) fail("nrsc5b_drain", (int)got);
    if (nrsc5b_take_overflow(st->engine, 0)) fail("record log overflow (RECORDS_CAPACITY)", -1);
    replay(st, st->records, (size_t)got);
}

static double seam_now(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

/* the records of a finished batch, straight from the page-locked memory the GPU exported them to */
static void deliver_batch(input_t *st)
{
    size_t n = 0;
    const uint8_t *rec = nrsc5b_batch_records(st->engine, 0, &n);
    if (nrsc5b_take_overflow(st->engine, 0)) fail("record log overflow (RECORDS_CAPACITY) or a frame exported undecoded", -1);
    const double t0 = st->trace ? seam_now() : 0;
    if (rec && n) replay(st, rec, n);
    if (st->trace) { st->trace_replay_s += seam_now() - t0; st->trace_batches++; st->trace_bytes += n; }
}

/* non-blocking: take what has finished, start what can start */
static void pump(input_t *st)
{
    int rc = nrsc5b_poll(st->engine, 0);
    if (rc < 0) fail("nrsc5b_poll", rc);
    if (rc == 1) deliver_batch(st);
    rc = nrsc5b_submit(st->engine, 0);
    if (rc < 0) fail("nrsc5b_submit", rc);
}

/* the device buffer is full of samples the GPU has not used yet: deliver the batch in flight and start the next */
static void wait_for_room(input_t *st)
{
    int rc = nrsc5b_poll(st->engine, 1);
    if (rc < 0) fail("nrsc5b_poll", rc);
    if (rc == 1) deliver_batch(st);
    rc = nrsc5b_submit(st->engine, 0);
    if (rc < 0) fail("nrsc5b_submit", rc);
    if (rc == 0 && nrsc5b_poll(st->engine, 0) == 0)
        fail("input buffer full although the GPU is idle (INPUT_CAPACITY)", NRSC5B_EFULL);
}

/* blocking: everything buffered so far is decoded and delivered */
static void pump_all(input_t *st)
{
    for (;;)
    {
        int rc = nrsc5b_poll(st->engine, 1);
        if (rc < 0) fail("nrsc5b_poll", rc);
        if (rc == 1) deliver_batch(st);
        rc = nrsc5b_submit(st->engine, 1);
        if (rc < 0) fail("nrsc5b_submit", rc);
        if (rc == 0) break;
    }
}

void input_push_cu8(input_t *st, const uint8_t *buf, const uint32_t len)
{
    nrsc5_report_iq(st->radio, buf, len);            /* input.c:101 */
    assert(len % 4 == 0);
    engine_open(st, 0);
    if (st->pipelined && !st->engine_am)
    {
        int rc = nrsc5b_stage_cu8(st->engine, 0, buf, len);
        while (rc == NRSC5B_EFULL)                   /* the GPU is a whole buffer behind: let it catch up */
        {
            wait_for_room(st);
            rc = nrsc5b_stage_cu8(st->engine, 0, NULL, 0);
        }
        if (rc) fail("nrsc5b_stage_cu8", rc);
        pump(st);
        return;
    }
    uint32_t done = 0;
    while (done < len)
    {
        /* synchronous mode (and AM cu8, which is decimated on arrival): at most a quarter block per round, so that a
         * host-side L2's sync-loss verdict (frame.c:538) always lands before the engine starts the following block */
        uint32_t n = len - done;
        if (n > 65536) n = 65536;
        int rc = nrsc5b_push_cu8(st->engine, 0, buf + done, n);
        if (rc) fail("nrsc5b_push_cu8", rc);
        run_and_replay(st);
        done += n;
    }
}

void input_push_cs16(input_t *st, const int16_t *buf, const uint32_t len)
{
    /* input.c:119-124: FM samples that are already at 744 187.5 S/s; len counts int16 values */
    assert(len % 2 == 0);
    engine_open(st, 1);
    if (st->pipelined)
    {
        int rc = nrsc5b_stage_cs16(st->engine, 0, buf, len);
        while (rc == NRSC5B_EFULL)
        {
            wait_for_room(st);
            rc = nrsc5b_stage_cs16(st->engine, 0, NULL, 0);
        }
        if (rc) fail("nrsc5b_stage_cs16", rc);
        pump(st);
        return;
    }
    uint32_t done = 0;
    while (done < len)
    {
        uint32_t n = len - done;
        if (n > 32768) n = 32768;
        int rc = nrsc5b_push_cs16(st->engine, 0, buf + done, n);
        if (rc) fail("nrsc5b_push_cs16", rc);
        run_and_replay(st);
        done += n;
    }
}

void input_reset(input_t *st)
{
    /* input.c:126-138 (buffered samples and what they would have decoded to are dropped, as in the reference) */
    if (st->sync_state == SYNC_STATE_FINE)
        nrsc5_report_lost_sync(st->radio);
    st->sync_state = SYNC_STATE_NONE;
    int rc = nrsc5b_reset(st->engine, 0);
    if (rc) fail("nrsc5b_reset", rc);
    pids_init(&st->pids, st);
    frame_reset(&st->frame);
}

void input_init(input_t *st, nrsc5_t *radio, output_t *output)
{
    memset(st, 0, sizeof(*st));
    st->radio = radio;
    st->output = output;
    st->sync_state = SYNC_STATE_NONE;

    engine_open(st, 0);
    st->records_cap = RECORDS_CAPACITY + 64;
    st->records = malloc(st->records_cap);
    st->bits = malloc(P1_FRAME_LEN_FM);
    if (!st->records || !st->bits) fail("malloc", -1);

    frame_init(&st->frame, st);
    input_reset(st);
}

void input_set_mode(input_t *st)
{
    /* acquire_set_mode + input_reset (input.c:159-163): AM and FM use different engines */
    engine_open(st, st->radio->mode == NRSC5_MODE_AM ? 1 : st->engine_cs16);
    input_reset(st);
}

void input_free(input_t *st)
{
    /* the reference has no flush and decodes inside the pushes; here the tail of the stream may still be on its way:
     * deliver it before the handle goes (nrsc5_close -> input_free, nrsc5.c:429) */
    const double t0 = st->trace ? seam_now() : 0;
    if (st->engine && st->pipelined)
        pump_all(st);
    const double t1 = st->trace ? seam_now() : 0;
    if (st->trace)
        fprintf(stderr, "libnrsc5 (GPU) trace: %lu batches delivered, %lu record bytes, %.6f s in the replay (callbacks included), "
                        "%.6f s in the final flush\n", st->trace_batches, st->trace_bytes, st->trace_replay_s, t1 - t0);
    frame_free(&st->frame);
    nrsc5b_destroy(st->engine);
    if (st->trace)
        fprintf(stderr, "libnrsc5 (GPU) trace: %.6f s in nrsc5b_destroy\n", seam_now() - t1);
    free(st->records);
    free(st->bits);
}
