/* dump1090-b200 — C host for the H100 demodulator: the --ifile side of
 * dump1090's command line (dump1090.c:2849-3010) over the C ABI of
 * include/modes_b200.h.  Reads 8-bit unsigned I/Q at 2 MHz from a file (or '-'
 * for stdin), feeds it to the device library, prints what the reference prints.
 *
 * Supported options (same spelling and meaning as the reference):
 *   --ifile <file>  --raw  --onlyaddr  --no-fix  --no-crc-check  --aggressive  --stats
 * Additions: --drop-eof-buffer (reproduce the stock binary's usual EOF race
 * outcome), --device <n>, --gpus <n> (deal the buffers to n GPUs starting at --device, one copy
 * stream per GPU), --chunk <bytes> (read size); --sbs prints the SBS (BaseStation)
 * line of every message instead (what the reference writes to port 30003, dump1090.c:2396) and
 * --aircraft-json prints the tracked aircraft as the reference's /data.json at the end (:2505),
 * both with stream time (MODES_STREAM_EPOCH_MS + sample position / 2 MHz) as the clock.
 * The live-radio, networking and interactive options are out of scope.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "modes_b200.h"

static int opt_raw = 0, opt_onlyaddr = 0, opt_stats = 0, opt_check_crc = 1, opt_sbs = 0, opt_json = 0;
static modes_tracker *tracker = NULL;

/* Message sink: the --raw / --onlyaddr forms of displayModesMessage
 * (dump1090.c:1318-1331) and, by default, the full text (:1314-1450) via modes_format_message(). */
static void on_message(void *user, const modes_message *mm) {
    (void)user;
    if (opt_stats) return;                                  /* dump1090.c:1803 */
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

int main(int argc, char **argv) {
    modes_config cfg;
    const char *filename = NULL;
    size_t chunk = 16u << 20;
    modes_default_config(&cfg);
    for (int j = 1; j < argc; j++) {
        int more = j + 1 < argc;
        if (!strcmp(argv[j], "--ifile") && more) filename = argv[++j];
        else if (!strcmp(argv[j], "--raw")) opt_raw = 1;
        else if (!strcmp(argv[j], "--onlyaddr")) opt_onlyaddr = 1;
        else if (!strcmp(argv[j], "--no-fix")) cfg.fix_errors = 0;
        else if (!strcmp(argv[j], "--no-crc-check")) { cfg.check_crc = 0; opt_check_crc = 0; }
        else if (!strcmp(argv[j], "--aggressive")) cfg.aggressive = 1;
        else if (!strcmp(argv[j], "--stats")) opt_stats = 1;
        else if (!strcmp(argv[j], "--drop-eof-buffer")) cfg.drop_eof_buffer = 1;
        else if (!strcmp(argv[j], "--sbs")) opt_sbs = 1;
        else if (!strcmp(argv[j], "--aircraft-json")) opt_json = 1;
        else if (!strcmp(argv[j], "--device") && more) cfg.device = atoi(argv[++j]);
        else if (!strcmp(argv[j], "--gpus") && more) cfg.n_gpus = atoi(argv[++j]);
        else if (!strcmp(argv[j], "--chunk") && more) chunk = (size_t)strtoull(argv[++j], NULL, 10);
        else {
            fprintf(stderr, "Unknown or not enough arguments for option '%s'.\n", argv[j]);
            return 1;
        }
    }
    if (!filename) { fprintf(stderr, "--ifile <filename> is required (use '-' for stdin)\n"); return 1; }
    FILE *f = (filename[0] == '-' && filename[1] == 0) ? stdin : fopen(filename, "rb");
    if (!f) { perror("Opening data file"); return 1; }

    modes_ctx *ctx = modes_create(&cfg);
    if (!ctx) { fprintf(stderr, "modes_create: %s\n", modes_last_error(NULL)); return 1; }
    if (opt_sbs || opt_json) {
        tracker = modes_tracker_create(cfg.check_crc);
        if (!tracker) { fprintf(stderr, "out of memory\n"); return 1; }
    }
    modes_set_sink(ctx, on_message, NULL);
    unsigned char *buf = (unsigned char *)modes_host_alloc(chunk);
    if (!buf) { fprintf(stderr, "out of memory\n"); return 1; }
    size_t n;
    while ((n = fread(buf, 1, chunk, f)) > 0) {
        if (modes_process(ctx, buf, n)) { fprintf(stderr, "modes_process: %s\n", modes_last_error(ctx)); return 1; }
    }
    if (modes_finish(ctx)) { fprintf(stderr, "modes_finish: %s\n", modes_last_error(ctx)); return 1; }
    if (opt_stats) {                                        /* dump1090.c:2993-3006 */
        modes_stats st;
        modes_get_stats(ctx, &st);
        printf("%lld valid preambles\n", (long long)st.v[0]);
        printf("%lld demodulated again after phase correction\n", (long long)st.v[1]);
        printf("%lld demodulated with zero errors\n", (long long)st.v[2]);
        printf("%lld with good crc\n", (long long)st.v[3]);
        printf("%lld with bad crc\n", (long long)st.v[4]);
        printf("%lld errors corrected\n", (long long)st.v[5]);
        printf("%lld single bit errors\n", (long long)st.v[6]);
        printf("%lld two bits errors\n", (long long)st.v[7]);
        printf("%lld total usable messages\n", (long long)(st.v[3] + st.v[5]));
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
