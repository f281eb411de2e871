/* TEST INFRASTRUCTURE -- not product code.
 *
 * ref_dump (ref_dump.c, unchanged) with one more option, --time-overwrite: the producer runs with
 * simulator_t.time_overwrite set, which is what the reference's `-s now` does besides reading the clock
 * (gps-sim.c:89-102). The explicit -s date stands in for the clock reading, so the reference's ephemeris and UTC time
 * overwrite (gps.c:2531-2561) runs verbatim at a chosen instant. Without --time-overwrite the binary is ref_dump.
 *
 * ref_dump.c keeps its simulator_t on main's stack and hands it to gps_thread_ep through pthread_create; that call is
 * the one place the flag can be set from outside, so it is routed through oracle_pthread_create below.
 */
#include <pthread.h>
#include <string.h>

static int oracle_time_overwrite;
static int oracle_pthread_create(pthread_t *th, const pthread_attr_t *attr, void *(*fn)(void *), void *arg);

#define pthread_create oracle_pthread_create
#define main ref_dump_main
#include "ref_dump.c"
#undef main
#undef pthread_create

static int oracle_pthread_create(pthread_t *th, const pthread_attr_t *attr, void *(*fn)(void *), void *arg) {
    if (fn == gps_thread_ep && oracle_time_overwrite) ((simulator_t *) arg)->time_overwrite = true;
    return pthread_create(th, attr, fn, arg);
}

int main(int argc, char **argv) {
    int n = 0;
    for (int i = 0; i < argc; i++) {
        if (i > 0 && !strcmp(argv[i], "--time-overwrite")) oracle_time_overwrite = 1;
        else argv[n++] = argv[i];
    }
    argv[n] = NULL;
    return ref_dump_main(n, argv);
}
