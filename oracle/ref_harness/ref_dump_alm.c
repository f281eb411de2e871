/* TEST INFRASTRUCTURE -- not product code.
 *
 * ref_dump.c (the UNMODIFIED reference producer behind the recording FIFO) with the reference's own default
 * almanac_enable = true (gps-sim.c:189) instead of the false that ref_dump.c sets: the producer then reads
 * ./almanac.sem (almanac.c:78), checks its toa against the start (gps.c:2637-2651) and sends it in subframes 4 and 5
 * (gps.c:772-883). ref_dump.c and the reference sources are compiled unmodified; the one hook is the start of the
 * producer thread, where the flag is set on the simulator_t handed to gps_thread_ep. Same command line as ref_dump.
 * Built by oracle/Makefile.almanac. */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <zlib.h>

/* same first inclusion order of the reference headers as ref_dump.c */
#include "gps.h"
#include "gps-sim.h"

static int alm_pthread_create(pthread_t *th, const pthread_attr_t *attr, void *(*fn)(void *), void *arg) {
    ((simulator_t *) arg)->almanac_enable = true;
    return pthread_create(th, attr, fn, arg);
}
#define pthread_create alm_pthread_create

#include "ref_dump.c"
