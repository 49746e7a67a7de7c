/* bench_pipe: one capture through the PUBLIC libnrsc5 API exactly as the reference's CLI feeds a file
 * (reference src/main.c:1097-1119: fread 32 768 bytes -> nrsc5_pipe_samples_cu8, then nrsc5_stop / nrsc5_close),
 * with the library given on the command line and loaded with dlopen - so the very same binary times the drop-in
 * (nrsc5_b200/dropin/_build/libnrsc5.so, CUDA engine underneath) and the unmodified reference
 * (oracle/_ref/libnrsc5_ref.so, CPU) on the same bytes.  Prints one JSON object: wall seconds of the push loop
 * (input already in memory; open and close outside / inside as stated), event counts and an FNV-1a digest of all
 * HDC packets so that the two runs can be compared.
 *
 *   bench_pipe <libnrsc5.so> <capture.cu8 | capture.cs16> [--cs16] [--am] [--chunk BYTES] [--reps N]
 */
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <nrsc5.h>

typedef int (*open_pipe_t)(nrsc5_t **);
typedef void (*close_t)(nrsc5_t *);
typedef void (*startstop_t)(nrsc5_t *);
typedef int (*set_mode_t)(nrsc5_t *, int);
typedef void (*set_cb_t)(nrsc5_t *, nrsc5_callback_t, void *);
typedef int (*pipe_cu8_t)(nrsc5_t *, const uint8_t *, unsigned int);
typedef int (*pipe_cs16_t)(nrsc5_t *, const int16_t *, unsigned int);

struct tally {
    unsigned long n[64];
    unsigned long hdc_bytes;
    uint32_t hdc_fnv;
    unsigned long audio_service, id3;
};

static void on_event(const nrsc5_event_t *evt, void *opaque)
{
    struct tally *t = (struct tally *)opaque;
    if (evt->event < 64) t->n[evt->event]++;
    if (evt->event == NRSC5_EVENT_HDC) {
        uint32_t h = t->hdc_fnv;
        for (size_t i = 0; i < evt->hdc.count; i++) h = (h ^ evt->hdc.data[i]) * 0x01000193u;
        t->hdc_fnv = h;
        t->hdc_bytes += evt->hdc.count;
    }
}

static double now(void)
{
    struct timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return (double)ts.tv_sec + 1e-9 * (double)ts.tv_nsec;
}

int main(int argc, char **argv)
{
    if (argc < 3) {
        fprintf(stderr, "usage: %s <libnrsc5.so> <capture> [--cs16] [--am] [--chunk BYTES] [--reps N]\n", argv[0]);
        return 2;
    }
    int cs16 = 0, am = 0, reps = 1;
    size_t chunk = 32768;
    for (int i = 3; i < argc; i++) {
        if (!strcmp(argv[i], "--cs16")) cs16 = 1;
        else if (!strcmp(argv[i], "--am")) am = 1;
        else if (!strcmp(argv[i], "--chunk") && i + 1 < argc) chunk = (size_t)atol(argv[++i]);
        else if (!strcmp(argv[i], "--reps") && i + 1 < argc) reps = atoi(argv[++i]);
    }
    void *lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
    if (!lib) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 1; }
    open_pipe_t p_open = (open_pipe_t)dlsym(lib, "nrsc5_open_pipe");
    close_t p_close = (close_t)dlsym(lib, "nrsc5_close");
    startstop_t p_start = (startstop_t)dlsym(lib, "nrsc5_start"), p_stop = (startstop_t)dlsym(lib, "nrsc5_stop");
    set_mode_t p_mode = (set_mode_t)dlsym(lib, "nrsc5_set_mode");
    set_cb_t p_cb = (set_cb_t)dlsym(lib, "nrsc5_set_callback");
    pipe_cu8_t p_cu8 = (pipe_cu8_t)dlsym(lib, "nrsc5_pipe_samples_cu8");
    pipe_cs16_t p_cs16 = (pipe_cs16_t)dlsym(lib, "nrsc5_pipe_samples_cs16");
    if (!p_open || !p_close || !p_cb || !p_cu8 || !p_cs16 || !p_start || !p_stop || !p_mode) {
        fprintf(stderr, "missing public symbols in %s\n", argv[1]);
        return 1;
    }
    FILE *fp = fopen(argv[2], "rb");
    if (!fp) { perror(argv[2]); return 1; }
    fseek(fp, 0, SEEK_END);
    size_t nbytes = (size_t)ftell(fp);
    fseek(fp, 0, SEEK_SET);
    uint8_t *buf = (uint8_t *)malloc(nbytes);
    if (!buf || fread(buf, 1, nbytes, fp) != nbytes) { fprintf(stderr, "read failed\n"); return 1; }
    fclose(fp);
    nbytes &= ~(size_t)3;

    double best = 1e30, first = 0, open_s = 0;
    struct tally tl;
    for (int r = 0; r < reps + 1; r++) {                   /* the first pass is a warm-up (CUDA context, page faults) */
        memset(&tl, 0, sizeof(tl));
        tl.hdc_fnv = 0x811C9DC5u;
        nrsc5_t *radio = NULL;
        const double t_open = now();
        if (p_open(&radio) != 0 || !radio) { fprintf(stderr, "nrsc5_open_pipe failed\n"); return 1; }
        if (am) p_mode(radio, NRSC5_MODE_AM);
        p_cb(radio, on_event, &tl);
        p_start(radio);
        const double t0 = now();
        for (size_t off = 0; off < nbytes; off += chunk) {
            const size_t n = nbytes - off < chunk ? nbytes - off : chunk;
            if (cs16) p_cs16(radio, (const int16_t *)(buf + off), (unsigned int)(n / 2));
            else p_cu8(radio, buf + off, (unsigned int)n);
        }
        p_stop(radio);                                     /* everything buffered is decoded and delivered by now ... */
        p_close(radio);                                    /* ... or by here (reference: stop is a no-op in pipe mode) */
        const double t1 = now();
        if (r == 0) { first = t1 - t0; open_s = t0 - t_open; continue; }
        if (t1 - t0 < best) best = t1 - t0;
    }
    const double samples = cs16 ? (double)nbytes / 4 * 2 : (double)nbytes / 2;    /* in cu8-rate complex samples (FM) */
    const double rate = am && cs16 ? 46511.71875 : 1488375.0;
    const double signal_s = (am && cs16 ? (double)nbytes / 4 : samples) / rate;
    printf("{\"seconds\": %.6f, \"first_pass_seconds\": %.6f, \"open_seconds\": %.6f, \"signal_seconds\": %.4f, \"x_realtime\": %.2f, "
           "\"msamples_per_s\": %.3f, \"pushes\": %zu, \"chunk_bytes\": %zu, \"sync\": %lu, \"lost_sync\": %lu, \"mer\": %lu, \"ber\": %lu, "
           "\"hdc\": %lu, \"hdc_bytes\": %lu, \"hdc_fnv\": \"%08x\", \"id3\": %lu, \"sis\": %lu, \"audio_service\": %lu}\n",
           best, first, open_s, signal_s, signal_s / best, samples / best / 1e6, (nbytes + chunk - 1) / chunk, chunk,
           tl.n[NRSC5_EVENT_SYNC], tl.n[NRSC5_EVENT_LOST_SYNC], tl.n[NRSC5_EVENT_MER], tl.n[NRSC5_EVENT_BER], tl.n[NRSC5_EVENT_HDC],
           tl.hdc_bytes, tl.hdc_fnv, tl.n[NRSC5_EVENT_ID3], tl.n[NRSC5_EVENT_SIS], tl.n[NRSC5_EVENT_AUDIO_SERVICE]);
    free(buf);
    return 0;
}
