/* input.h of the drop-in libnrsc5.so: the seam between the reference's unmodified host side (nrsc5.c,
 * frame.c, pids.c, output.c, ... compiled from the reference tree as they are) and the CUDA engine.
 *
 * It replaces reference src/input.h:1-43.  The host side only ever touches four members of input_t -
 * `radio`, `output`, `frame` (frame.c:746, decode.c:460) and, through pids_init(), `pids` - and calls the
 * seven input_* functions declared at the bottom (nrsc5.c:127,181,190,221,429,469,548,606,613,637,642;
 * frame.c:539).  Everything between input_push_cu8() and frame_push()/pids_frame_push() - decimation,
 * acquisition, OFDM demodulation, synchronisation, deinterleaving, Viterbi - runs on the GPU behind
 * include/nrsc5_b200.h. */
#pragma once

#include <stdint.h>
#include <complex.h>

#include <nrsc5.h>

#include "defines.h"
#include "frame.h"
#include "output.h"
#include "pids.h"

enum { SYNC_STATE_NONE, SYNC_STATE_COARSE, SYNC_STATE_FINE };

struct nrsc5b_engine;

typedef struct input_t
{
    nrsc5_t *radio;
    output_t *output;
    unsigned int sync_state;            /* as last reported downstream */

    frame_t frame;
    pids_t pids;

    struct nrsc5b_engine *engine;       /* one stream on one GPU */
    int engine_cs16;                    /* the format that engine was built for */
    int engine_am;                      /* ... and the mode */
    uint8_t *records;                   /* drained record stream of the last push */
    size_t records_cap;
    uint8_t *bits;                      /* one bit per byte, as frame_push()/pids_frame_push() take them */
    int in_frame_push;
    int device_l2;                      /* L2 framing runs on the GPU (FM): replay REC_L2 instead of calling frame_push() */
    int pipelined;                      /* pushes stage samples and return; batches complete behind them (default) */
    int trace;                          /* NRSC5_B200_TRACE: time spent delivering records, printed by input_free() */
    unsigned long trace_batches, trace_bytes;
    double trace_replay_s;
} input_t;

void input_init(input_t *st, nrsc5_t *radio, output_t *output);
void input_set_mode(input_t *st);
void input_reset(input_t *st);
void input_free(input_t *st);
void input_set_sync_state(input_t *st, unsigned int new_state);
void input_push_cu8(input_t *st, const uint8_t *buf, uint32_t len);
void input_push_cs16(input_t *st, const int16_t *buf, uint32_t len);
