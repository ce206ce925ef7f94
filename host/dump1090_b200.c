/* dump1090-b200 — C host for the H100 demodulator: the --ifile side of
 * dump1090's command line (dump1090.c:2849-3010) over the C ABI of
 * include/modes_b200.h.  Reads 8-bit unsigned I/Q at 2 MHz from a file (or '-'
 * for stdin; --sample-rate and --iformat below for other captures), feeds it to the device library, prints what the reference prints.
 *
 * Supported options (same spelling and meaning as the reference):
 *   --ifile <file>  --raw  --onlyaddr  --no-fix  --no-crc-check  --aggressive  --stats
 * Additions: --drop-eof-buffer (reproduce the stock binary's usual EOF race
 * outcome), --device <n>, --gpus <n> (deal the buffers to n GPUs starting at --device, one copy
 * stream per GPU), --chunk <bytes> (read size); --sbs prints the SBS (BaseStation)
 * line of every message instead (what the reference writes to port 30003, dump1090.c:2396) and
 * --aircraft-json prints the tracked aircraft as the reference's /data.json at the end (:2505),
 * both with stream time (MODES_STREAM_EPOCH_MS + sample position / 2 MHz) as the clock.
 * --beast writes one Beast binary frame per message instead (what the dump1090 descendants send on
 * port 30005: 12 MHz timestamp = 6 x sample position, signal level measured on the GPU); it excludes
 * --raw, --onlyaddr, --sbs and --aircraft-json, which write to stdout as well.
 * --arrival refines the Beast timestamps to a sixth of a sample with the arrival time measured on the
 * GPU (modes_set_arrival); it needs --beast, the only output mode that prints a time.
 * --levels measures every decoded buffer's noise, peak and clipping on the GPU and prints one
 * summary line on stderr at the end (buffers, samples, noise floor and peak in dBFS on the scale of
 * the Beast signal level, clipped samples and their fraction); it combines with every output mode
 * and leaves stdout as it is.
 * --recover adds weak DF17/DF18 frames of already known aircraft that a soft-decision search on the
 * GPU repairs (include/modes_b200.h, modes_set_recovery); they are not the reference's messages.  It
 * combines with every output mode; with --stats the reference's lines stay as they are on stdout and
 * one recovery line goes to stderr.  --gpu-resolve runs the order-dependent half on the GPU too
 * (modes_config.gpu_resolve); it has no recovery rule, so it is refused together with --recover.
 * --recover-weak implies --recover and also searches weak preambles, positions the reference's
 * preamble test rejects (modes_set_weak_preambles); with --stats a second line goes to stderr.
 * --sample-rate <hz> gives the rate of the file: 2000000 (the default), 2400000, what dump1090-fa and
 * readsb record (modes_set_input_rate: resampled to 2 MHz on the GPU, sample positions and Beast
 * timestamps on the same 2 MHz / 12 MHz clocks), or 4000000, 6000000, 8000000 or 10000000, what Airspy,
 * SDRplay and USRP radios usually record (decimated to 2 MHz on the GPU, on the same clocks).  It
 * combines with every output mode and switch.
 * --iformat UC8|SC16|SC16Q11 gives the sample format of the file, as dump1090-fa spells it: 8-bit
 * unsigned (the default), or signed 16-bit I/Q (SoapySDR and Airspy-class tools; bladeRF's 12-bit values),
 * converted to 8 bits on the GPU (modes_set_input_format).  --iformat-shift <0..15> replaces the
 * format's default shift (SC16 8, SC16Q11 4; not with UC8): a smaller one for a quiet capture, checked
 * with the clipping count of --levels.  Both combine with --sample-rate, every output mode and switch.
 * --input-offset <hz> says where 1090 MHz sits in the file's baseband, for a radio tuned off the channel
 * (+2000000: tuned to 1088 MHz, as zero-IF radios are to keep their DC spike away from it): the input is
 * shifted back by that much on the GPU as it is decimated (modes_set_input_offset).  It needs
 * --sample-rate 4000000 to 10000000, and |hz| at most half the rate less 1 MHz (1, 2, 3 or 4 MHz).
 * --spectrum measures every decoded buffer's input power spectrum on the GPU (modes_set_spectrum), before
 * resampling, decimation and the offset, and prints one summary line on stderr at the end, as --levels
 * does: the noise floor, the DC bin's excess over bins 126 and 130 (a zero-IF radio's spike) and the centre of
 * the 2 MHz band with the most power above the floor (where the channel most likely sits: the value for
 * --input-offset).  It combines with every --sample-rate, --iformat and --input-offset and leaves stdout
 * as it is.
 * --carrier measures every decoded frame's carrier frequency on the GPU (modes_set_carrier) and prints one
 * summary line on stderr at the end, as --levels does: the messages and aircraft measured and the receiver's
 * offset, the median over aircraft of each aircraft's median carrier, in Hz and in ppm of 1090 MHz (the
 * receiver's tuning error; carrier_summary in dump1090_b200/api.py is the same computation).  It combines with
 * every --sample-rate, --iformat, --input-offset and output mode and leaves stdout as it is; the device
 * resolve has no room for it, so it is refused together with --gpu-resolve.
 * --pool decodes every --ifile (given once per file) at once, each as one receiver of a receiver pool
 * (modes_pool_*: one buffer of every file per batch, each file finished with its tail by modes_pool_finish),
 * and prints exactly what one run per file prints, file by file in command-line order.  It takes the text
 * outputs (the default, --raw, --onlyaddr), --stats, --no-fix, --no-crc-check, --aggressive,
 * --drop-eof-buffer, --sample-rate 2000000 or 2400000, --iformat, --iformat-shift and --device; every other
 * option, and --ifile - (stdin), is refused with it.  Without --pool a repeated --ifile means the last one.
 * The live-radio, networking and interactive options are out of scope.
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include "modes_b200.h"

static int opt_raw = 0, opt_onlyaddr = 0, opt_stats = 0, opt_check_crc = 1, opt_sbs = 0, opt_json = 0, opt_beast = 0;
static int opt_levels = 0, opt_recover = 0, opt_weak = 0, opt_arrival = 0, opt_spectrum = 0, opt_carrier = 0;
static modes_tracker *tracker = NULL;

/* --levels: totals over the records taken so far */
static struct { long long buffers; unsigned long long samples, clipped; unsigned __int128 power; unsigned peak; } lv;

static void take_levels(modes_ctx *ctx) {
    modes_level r[256];
    size_t n;
    while ((n = modes_take_levels(ctx, r, 256)) > 0)
        for (size_t i = 0; i < n; i++) {
            lv.buffers++;
            lv.samples += r[i].n_samples;
            lv.clipped += r[i].clipped;
            lv.power += r[i].sum_power;
            if (r[i].peak > lv.peak) lv.peak = r[i].peak;
        }
}

static void print_levels(void) {
    fprintf(stderr, "levels: %lld buffers, %llu samples, ", lv.buffers, lv.samples);
    if (!lv.samples) { fprintf(stderr, "noise n/a, peak n/a, clipped 0\n"); return; }
    const double fs2 = 65535.0 * 65535.0;
    const double noise = lv.power ? 10.0 * log10((double)lv.power / (double)lv.samples / fs2) : -INFINITY;
    const double peak = lv.peak ? 20.0 * log10(lv.peak / 65535.0) : -INFINITY;
    fprintf(stderr, "noise %.2f dBFS, peak %.2f dBFS, clipped %llu (%.6f)\n", noise, peak, lv.clipped,
            (double)lv.clipped / (double)lv.samples);
}

/* --spectrum: per-bin totals over the records taken so far (spectrum_summary in dump1090_b200/api.py is the
 * same computation; the floor and the band search are exact on the integer sums) */
static struct { long long buffers; unsigned long long frames; unsigned __int128 power[MODES_SPECTRUM_BINS]; } sp;

static void take_spectra(modes_ctx *ctx) {
    static modes_spectrum r[64];
    size_t n;
    while ((n = modes_take_spectra(ctx, r, 64)) > 0)
        for (size_t i = 0; i < n; i++) {
            sp.buffers++;
            sp.frames += r[i].frames;
            for (int k = 0; k < MODES_SPECTRUM_BINS; k++) sp.power[k] += r[i].power[k];
        }
}

static int cmp_u128(const void *a, const void *b) {
    const unsigned __int128 x = *(const unsigned __int128 *)a, y = *(const unsigned __int128 *)b;
    return x < y ? -1 : x > y;
}

static void print_spectrum(unsigned long fs) {
    enum { N = MODES_SPECTRUM_BINS };
    fprintf(stderr, "spectrum: %lld buffers, %llu frames, ", sp.buffers, sp.frames);
    if (!sp.frames) { fprintf(stderr, "floor n/a\n"); return; }
    const unsigned __int128 dc = 2 * sp.power[N / 2], nb = sp.power[N / 2 - 2] + sp.power[N / 2 + 2];
    const double dc_db = dc == nb ? 0.0 : !nb ? INFINITY : !dc ? -INFINITY : 10.0 * log10((double)dc / (double)nb);
    unsigned __int128 t2[N], srt[N];
    for (int i = 0; i < N; i++) t2[i] = 2 * sp.power[i];
    t2[N / 2 - 1] = t2[N / 2] = t2[N / 2 + 1] = nb;          /* DC and the window's main lobe around it */
    memcpy(srt, t2, sizeof(srt));
    qsort(srt, N, sizeof(srt[0]), cmp_u128);
    const unsigned __int128 floor4 = srt[N / 2 - 1] + srt[N / 2];
    const double floor_db = floor4 ? 10.0 * log10((double)floor4 / 4.0 / (double)sp.frames) : -INFINITY;
    const int w = (int)((unsigned long long)N * 2000000ull / fs);
    unsigned __int128 best = 0;
    int at = -1;
    for (int i0 = 0; i0 + w <= N; i0++) {
        unsigned __int128 score = 0;
        for (int i = i0; i < i0 + w; i++) score += 2 * t2[i] > floor4 ? 2 * t2[i] - floor4 : 0;
        if (at < 0 || score > best) { best = score; at = i0; }
    }
    fprintf(stderr, "floor %.2f dB, DC %+.2f dB over its neighbours, strongest 2 MHz band at %+.0f Hz\n", floor_db, dc_db,
            (at + (w - 1) / 2.0 - N / 2) * (double)fs / N);
}

/* --carrier: (address, code) of every measured message, summarised at the end */
static struct { uint64_t *v; size_t n, cap; } cr;

static void take_carrier(const modes_message *mm) {
    if (!mm->carrier) return;
    if (cr.n == cr.cap) {
        const size_t cap = cr.cap ? 2 * cr.cap : 4096;
        uint64_t *v = (uint64_t *)realloc(cr.v, cap * sizeof(uint64_t));
        if (!v) return;
        cr.v = v; cr.cap = cap;
    }
    const uint32_t addr = ((uint32_t)mm->aa1 << 16) | ((uint32_t)mm->aa2 << 8) | (uint32_t)mm->aa3;
    cr.v[cr.n++] = ((uint64_t)addr << 16) | (uint16_t)mm->carrier;
}

static int cmp_u64(const void *a, const void *b) {
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : x > y;
}

static int cmp_double(const void *a, const void *b) {
    const double x = *(const double *)a, y = *(const double *)b;
    return x < y ? -1 : x > y;
}

/* the median of n sorted values (the mean of the middle two for even n) */
static double median_of(const double *v, size_t n) { return n & 1 ? v[n / 2] : 0.5 * (v[n / 2 - 1] + v[n / 2]); }

static void print_carrier(void) {
    qsort(cr.v, cr.n, sizeof(uint64_t), cmp_u64);            /* by address, then by code */
    double *per = (double *)malloc((cr.n ? cr.n : 1) * sizeof(double)), *hz = (double *)malloc((cr.n ? cr.n : 1) * sizeof(double));
    size_t n_ac = 0;
    for (size_t i = 0; per && hz && i < cr.n;) {
        size_t k = 0;
        for (const uint64_t a = cr.v[i] >> 16; i < cr.n && cr.v[i] >> 16 == a; i++)
            hz[k++] = ((double)(cr.v[i] & 0xffffu) - 16384.0) * 100.0;
        per[n_ac++] = median_of(hz, k);
    }
    fprintf(stderr, "carrier: %zu messages, %zu aircraft, ", cr.n, n_ac);
    if (!n_ac) fprintf(stderr, "receiver offset n/a\n");
    else {
        qsort(per, n_ac, sizeof(double), cmp_double);
        const double f = median_of(per, n_ac);
        fprintf(stderr, "receiver offset %+.0f Hz (%+.3f ppm of 1090 MHz)\n", f, f / 1090.0);
    }
    free(per); free(hz); free(cr.v);
}

/* Message sink: the --raw / --onlyaddr forms of displayModesMessage
 * (dump1090.c:1318-1331) and, by default, the full text (:1314-1450) via modes_format_message(). */
static void on_message(void *user, const modes_message *mm) {
    (void)user;
    if (opt_carrier) take_carrier(mm);
    if (opt_stats) return;                                  /* dump1090.c:1803 */
    if (opt_beast) {
        uint8_t frame[64];
        size_t n = modes_format_beast(mm, frame, sizeof(frame));
        fwrite(frame, 1, n, stdout);
        return;
    }
    if (tracker) {                                          /* dump1090.c:1806-1809 */
        const modes_aircraft *a = modes_tracker_update(tracker, mm, MODES_STREAM_EPOCH_MS + mm->sample_pos / 2000);
        if (a && opt_sbs) {
            char line[512];
            size_t n = modes_format_sbs(mm, a, line, sizeof(line));
            fwrite(line, 1, n < sizeof(line) ? n : sizeof(line) - 1, stdout);
        }
        if (opt_sbs || opt_json) return;
    }
    if (opt_onlyaddr) {
        printf("%02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
        return;
    }
    if (!opt_raw) {                                         /* the full text, dump1090.c:1314-1450 */
        char text[2048];
        size_t n = modes_format_message(mm, opt_check_crc, text, sizeof(text));
        fwrite(text, 1, n < sizeof(text) ? n : sizeof(text) - 1, stdout);
        return;
    }
    printf("*");
    for (int j = 0; j < mm->msgbits / 8; j++) printf("%02x", mm->msg[j]);
    printf(";\n");
    if (opt_raw) return;
}

/* The reference's --stats lines (dump1090.c:2993-3006). */
static void print_stats(const modes_stats *st) {
    printf("%lld valid preambles\n", (long long)st->v[0]);
    printf("%lld demodulated again after phase correction\n", (long long)st->v[1]);
    printf("%lld demodulated with zero errors\n", (long long)st->v[2]);
    printf("%lld with good crc\n", (long long)st->v[3]);
    printf("%lld with bad crc\n", (long long)st->v[4]);
    printf("%lld errors corrected\n", (long long)st->v[5]);
    printf("%lld single bit errors\n", (long long)st->v[6]);
    printf("%lld two bits errors\n", (long long)st->v[7]);
    printf("%lld total usable messages\n", (long long)(st->v[3] + st->v[5]));
}

/* --pool: each file's lines, held until every file is done */
static struct text { char *v; size_t n, cap; } *pool_text;

static void on_pool_message(void *user, uint32_t receiver, const modes_message *mm) {
    (void)user;
    if (opt_stats) return;                                  /* dump1090.c:1803 */
    char line[2048];
    size_t n = 0;
    if (opt_onlyaddr) n = (size_t)snprintf(line, sizeof(line), "%02x%02x%02x\n", mm->aa1, mm->aa2, mm->aa3);
    else if (!opt_raw) {
        n = modes_format_message(mm, opt_check_crc, line, sizeof(line));
        if (n >= sizeof(line)) n = sizeof(line) - 1;
    } else {
        line[n++] = '*';
        for (int j = 0; j < mm->msgbits / 8; j++) n += (size_t)snprintf(line + n, sizeof(line) - n, "%02x", mm->msg[j]);
        line[n++] = ';';
        line[n++] = '\n';
    }
    struct text *t = &pool_text[receiver];
    if (t->n + n > t->cap) {
        const size_t cap = 2 * (t->n + n) + 4096;
        char *v = (char *)realloc(t->v, cap);
        if (!v) { fprintf(stderr, "out of memory\n"); exit(1); }
        t->v = v; t->cap = cap;
    }
    memcpy(t->v + t->n, line, n);
    t->n += n;
}

/* --pool: every file one receiver, fed one buffer per file and call, then finished with its tail. */
static int run_pool(const modes_config *cfg, char **files, size_t n, uint32_t rate, uint32_t format, int32_t shift) {
    const size_t full = (size_t)MODES_BUFFER_BYTES * (format == MODES_INPUT_UC8 ? 1 : 2);
    FILE **f = (FILE **)calloc(n, sizeof(FILE *));
    if (!f) { fprintf(stderr, "out of memory\n"); return 1; }
    for (size_t i = 0; i < n; i++) {
        f[i] = fopen(files[i], "rb");
        if (!f[i]) { perror("Opening data file"); return 1; }
    }
    size_t *tail = (size_t *)calloc(n, sizeof(size_t));
    uint32_t *ids = (uint32_t *)malloc(n * sizeof(uint32_t));
    const uint8_t **iq = (const uint8_t **)malloc(n * sizeof(uint8_t *));
    int *done = (int *)calloc(n, sizeof(int));
    pool_text = (struct text *)calloc(n, sizeof(struct text));
    unsigned char *bufs = (unsigned char *)modes_host_alloc(n * full);
    unsigned char *tails = (unsigned char *)malloc(n * full);
    if (!tail || !ids || !iq || !done || !pool_text || !bufs || !tails) { fprintf(stderr, "out of memory\n"); return 1; }
    modes_pool *p = modes_pool_create(cfg, n, n);
    if (!p) { fprintf(stderr, "modes_pool_create failed\n"); return 1; }
    for (uint32_t i = 0; i < n; i++) {
        if (modes_pool_set_input_rate(p, i, rate)) { fprintf(stderr, "--sample-rate: %s\n", modes_pool_last_error(p)); return 1; }
        if (modes_pool_set_input_format(p, i, format, shift)) { fprintf(stderr, "--iformat: %s\n", modes_pool_last_error(p)); return 1; }
    }
    for (;;) {
        size_t k = 0;
        for (uint32_t i = 0; i < n; i++) {
            if (done[i]) continue;
            unsigned char *b = bufs + k * full;
            const size_t got = fread(b, 1, full, f[i]);
            if (got == full) { ids[k] = i; iq[k++] = b; continue; }
            memcpy(tails + i * full, b, got);                  /* a short read: the file's tail */
            tail[i] = got;
            done[i] = 1;
        }
        if (!k) break;
        if (modes_pool_ingest(p, ids, iq, k, on_pool_message, NULL)) { fprintf(stderr, "modes_pool_ingest: %s\n", modes_pool_last_error(p)); return 1; }
    }
    for (uint32_t i = 0; i < n; i++) { ids[i] = i; iq[i] = tails + i * full; }
    if (modes_pool_finish(p, ids, iq, tail, n, on_pool_message, NULL)) { fprintf(stderr, "modes_pool_finish: %s\n", modes_pool_last_error(p)); return 1; }
    for (uint32_t i = 0; i < n; i++) {
        fwrite(pool_text[i].v, 1, pool_text[i].n, stdout);
        if (opt_stats) {
            modes_stats st;
            modes_pool_stats(p, i, &st);
            print_stats(&st);
        }
        free(pool_text[i].v);
        fclose(f[i]);
    }
    modes_pool_destroy(p);
    modes_host_free(bufs);
    free(tails); free(pool_text); free(done); free(iq); free(ids); free(tail); free(f);
    return 0;
}

int main(int argc, char **argv) {
    modes_config cfg;
    const char *filename = NULL;
    size_t chunk = 16u << 20;
    unsigned long sample_rate = 2000000;
    const char *iformat = "UC8";
    const char *iformat_shift = NULL;
    const char *input_offset = NULL;
    int opt_pool = 0;
    const char *pool_refused = NULL;                        /* the first option --pool does not take */
    char **files = (char **)malloc((size_t)argc * sizeof(char *));
    size_t n_files = 0;
    if (!files) { fprintf(stderr, "out of memory\n"); return 1; }
    modes_default_config(&cfg);
    for (int j = 1; j < argc; j++) {
        int more = j + 1 < argc;
        if (!pool_refused && (!strcmp(argv[j], "--sbs") || !strcmp(argv[j], "--aircraft-json") || !strcmp(argv[j], "--beast") ||
                              !strcmp(argv[j], "--arrival") || !strcmp(argv[j], "--levels") || !strcmp(argv[j], "--spectrum") ||
                              !strcmp(argv[j], "--carrier") || !strcmp(argv[j], "--recover") ||
                              !strcmp(argv[j], "--recover-weak") || !strcmp(argv[j], "--gpu-resolve") ||
                              !strcmp(argv[j], "--gpus") || !strcmp(argv[j], "--chunk") || !strcmp(argv[j], "--input-offset")))
            pool_refused = argv[j];
        if (!strcmp(argv[j], "--ifile") && more) filename = files[n_files++] = argv[++j];
        else if (!strcmp(argv[j], "--pool")) opt_pool = 1;
        else if (!strcmp(argv[j], "--raw")) opt_raw = 1;
        else if (!strcmp(argv[j], "--onlyaddr")) opt_onlyaddr = 1;
        else if (!strcmp(argv[j], "--no-fix")) cfg.fix_errors = 0;
        else if (!strcmp(argv[j], "--no-crc-check")) { cfg.check_crc = 0; opt_check_crc = 0; }
        else if (!strcmp(argv[j], "--aggressive")) cfg.aggressive = 1;
        else if (!strcmp(argv[j], "--stats")) opt_stats = 1;
        else if (!strcmp(argv[j], "--drop-eof-buffer")) cfg.drop_eof_buffer = 1;
        else if (!strcmp(argv[j], "--sbs")) opt_sbs = 1;
        else if (!strcmp(argv[j], "--aircraft-json")) opt_json = 1;
        else if (!strcmp(argv[j], "--beast")) opt_beast = 1;
        else if (!strcmp(argv[j], "--arrival")) opt_arrival = 1;
        else if (!strcmp(argv[j], "--levels")) opt_levels = 1;
        else if (!strcmp(argv[j], "--spectrum")) opt_spectrum = 1;
        else if (!strcmp(argv[j], "--carrier")) opt_carrier = 1;
        else if (!strcmp(argv[j], "--recover")) opt_recover = 1;
        else if (!strcmp(argv[j], "--recover-weak")) opt_recover = opt_weak = 1;
        else if (!strcmp(argv[j], "--gpu-resolve")) cfg.gpu_resolve = 1;
        else if (!strcmp(argv[j], "--device") && more) cfg.device = atoi(argv[++j]);
        else if (!strcmp(argv[j], "--gpus") && more) cfg.n_gpus = atoi(argv[++j]);
        else if (!strcmp(argv[j], "--chunk") && more) chunk = (size_t)strtoull(argv[++j], NULL, 10);
        else if (!strcmp(argv[j], "--sample-rate") && more) sample_rate = strtoul(argv[++j], NULL, 10);
        else if (!strcmp(argv[j], "--iformat") && more) iformat = argv[++j];
        else if (!strcmp(argv[j], "--iformat-shift") && more) iformat_shift = argv[++j];
        else if (!strcmp(argv[j], "--input-offset") && more) input_offset = argv[++j];
        else {
            fprintf(stderr, "Unknown or not enough arguments for option '%s'.\n", argv[j]);
            return 1;
        }
    }
    if (!filename) { fprintf(stderr, "--ifile <filename> is required (use '-' for stdin)\n"); return 1; }
    if (opt_pool) {
        if (pool_refused) {
            fprintf(stderr, "--pool cannot be combined with %s: it takes the text outputs, --stats, --no-fix, --no-crc-check, "
                            "--aggressive, --drop-eof-buffer, --sample-rate, --iformat, --iformat-shift and --device\n", pool_refused);
            return 1;
        }
        for (size_t i = 0; i < n_files; i++)
            if (!strcmp(files[i], "-")) {
                fprintf(stderr, "--pool decodes files: --ifile - (stdin) cannot be combined with --pool\n");
                return 1;
            }
        if (sample_rate != 2000000 && sample_rate != 2400000) {
            fprintf(stderr, "--pool takes --sample-rate 2000000 or 2400000\n");
            return 1;
        }
    }
    if (sample_rate != 2000000 && sample_rate != 2400000 && sample_rate != 4000000 && sample_rate != 6000000 &&
        sample_rate != 8000000 && sample_rate != 10000000) {
        fprintf(stderr, "--sample-rate takes 2000000, 2400000, 4000000, 6000000, 8000000 or 10000000\n");
        return 1;
    }
    uint32_t format;
    if (!strcasecmp(iformat, "UC8")) format = MODES_INPUT_UC8;
    else if (!strcasecmp(iformat, "SC16")) format = MODES_INPUT_SC16;
    else if (!strcasecmp(iformat, "SC16Q11")) format = MODES_INPUT_SC16Q11;
    else {
        fprintf(stderr, "--iformat takes UC8, SC16 or SC16Q11\n");
        return 1;
    }
    int32_t shift = -1;
    if (iformat_shift) {
        char *end;
        const long v = strtol(iformat_shift, &end, 10);
        if (!*iformat_shift || *end || v < 0 || v > 15) {
            fprintf(stderr, "--iformat-shift takes a whole number from 0 to 15\n");
            return 1;
        }
        if (format == MODES_INPUT_UC8) {
            fprintf(stderr, "--iformat-shift needs --iformat SC16 or SC16Q11: UC8 input is not shifted\n");
            return 1;
        }
        shift = (int32_t)v;
    }
    int32_t offset_hz = 0;
    if (input_offset) {
        char *end;
        const long v = strtol(input_offset, &end, 10);
        if (!*input_offset || *end || v < -4000000 || v > 4000000) {
            fprintf(stderr, "--input-offset takes a whole number of Hz from -4000000 to 4000000\n");
            return 1;
        }
        if (v && sample_rate < 4000000) {
            fprintf(stderr, "--input-offset needs --sample-rate 4000000, 6000000, 8000000 or 10000000\n");
            return 1;
        }
        offset_hz = (int32_t)v;
    }
    if (opt_beast && (opt_raw || opt_onlyaddr || opt_sbs || opt_json)) {
        fprintf(stderr, "--beast writes binary frames to stdout: it cannot be combined with --raw, --onlyaddr, --sbs or --aircraft-json\n");
        return 1;
    }
    if (opt_arrival && !opt_beast) {
        fprintf(stderr, "--arrival refines the timestamps of --beast, the only output mode that prints a time: it needs --beast\n");
        return 1;
    }
    if (opt_recover && cfg.gpu_resolve) {
        if (opt_weak) fprintf(stderr, "--recover-weak implies --recover: ");
        fprintf(stderr, "--recover cannot be combined with --gpu-resolve: the device resolve has no recovery rule\n");
        return 1;
    }
    if (opt_carrier && cfg.gpu_resolve) {
        fprintf(stderr, "--carrier cannot be combined with --gpu-resolve: the device resolve's delivery records have no room for it\n");
        return 1;
    }
    if (opt_pool) {
        const int rc = run_pool(&cfg, files, n_files, (uint32_t)sample_rate, format, shift);
        free(files);
        return rc;
    }
    free(files);
    FILE *f = (filename[0] == '-' && filename[1] == 0) ? stdin : fopen(filename, "rb");
    if (!f) { perror("Opening data file"); return 1; }

    modes_ctx *ctx = modes_create(&cfg);
    if (!ctx) { fprintf(stderr, "modes_create: %s\n", modes_last_error(NULL)); return 1; }
    if (opt_sbs || opt_json) {
        tracker = modes_tracker_create(cfg.check_crc);
        if (!tracker) { fprintf(stderr, "out of memory\n"); return 1; }
    }
    if (modes_set_input_rate(ctx, (uint32_t)sample_rate)) { fprintf(stderr, "--sample-rate: %s\n", modes_last_error(ctx)); return 1; }
    if (modes_set_input_format(ctx, format, shift)) { fprintf(stderr, "--iformat: %s\n", modes_last_error(ctx)); return 1; }
    if (modes_set_input_offset(ctx, offset_hz)) { fprintf(stderr, "--input-offset: %s\n", modes_last_error(ctx)); return 1; }
    if (opt_beast) modes_set_signal(ctx, 1);
    if (opt_arrival) modes_set_arrival(ctx, 1);
    if (opt_levels) modes_set_levels(ctx, 1);
    if (opt_spectrum) modes_set_spectrum(ctx, 1);
    if (opt_carrier && modes_set_carrier(ctx, 1)) { fprintf(stderr, "--carrier: %s\n", modes_last_error(ctx)); return 1; }
    if (opt_recover && modes_set_recovery(ctx, 1)) { fprintf(stderr, "--recover: %s\n", modes_last_error(ctx)); return 1; }
    if (opt_weak && modes_set_weak_preambles(ctx, 1)) { fprintf(stderr, "--recover-weak: %s\n", modes_last_error(ctx)); return 1; }
    modes_set_sink(ctx, on_message, NULL);
    unsigned char *buf = (unsigned char *)modes_host_alloc(chunk);
    if (!buf) { fprintf(stderr, "out of memory\n"); return 1; }
    size_t n;
    while ((n = fread(buf, 1, chunk, f)) > 0) {
        if (modes_process(ctx, buf, n)) { fprintf(stderr, "modes_process: %s\n", modes_last_error(ctx)); return 1; }
        if (opt_levels) take_levels(ctx);
        if (opt_spectrum) take_spectra(ctx);
    }
    if (modes_finish(ctx)) { fprintf(stderr, "modes_finish: %s\n", modes_last_error(ctx)); return 1; }
    if (opt_levels) { take_levels(ctx); print_levels(); }
    if (opt_spectrum) { take_spectra(ctx); print_spectrum(sample_rate); }
    if (opt_carrier) print_carrier();
    if (opt_stats) {                                        /* dump1090.c:2993-3006 */
        modes_stats st;
        modes_get_stats(ctx, &st);
        print_stats(&st);
        if (opt_recover) {
            modes_recovery_stats rs;
            modes_get_recovery_stats(ctx, &rs);
            fprintf(stderr, "recovery: %lld considered, %lld found, %lld ambiguous, %lld unknown address, %lld dropped, %lld delivered\n",
                    (long long)rs.considered, (long long)rs.found, (long long)rs.ambiguous, (long long)rs.unknown_address,
                    (long long)rs.dropped, (long long)rs.delivered);
        }
        if (opt_weak) {
            modes_recovery_stats ws;
            modes_get_weak_recovery_stats(ctx, &ws);
            fprintf(stderr, "weak preambles: %lld considered, %lld found, %lld ambiguous, %lld unknown address, %lld dropped, %lld delivered\n",
                    (long long)ws.considered, (long long)ws.found, (long long)ws.ambiguous, (long long)ws.unknown_address,
                    (long long)ws.dropped, (long long)ws.delivered);
        }
    }
    if (opt_json) {
        size_t need = modes_tracker_format_json(tracker, 0, NULL, 0);
        char *json = (char *)malloc(need + 1);
        if (json) { modes_tracker_format_json(tracker, 0, json, need + 1); fwrite(json, 1, need, stdout); free(json); }
    }
    modes_tracker_destroy(tracker);
    modes_host_free(buf);
    modes_destroy(ctx);
    if (f != stdin) fclose(f);
    return 0;
}
