/* TEST INFRASTRUCTURE -- not product code.
 *
 * Prints the almanac that the UNMODIFIED reference parser (almanac.c, almanac_read_file) reads from ./almanac.sem:
 *   line 1:  <almanac valid flag> <return code of almanac_read_file>
 *   then one line per record sv[0..31]:
 *            svid svn ura health config_code valid toa.week  e delta_i omegadot sqrta omega0 aop m0 af0 af1 toa.sec
 * Doubles are printed as C99 hex floats (%a) so that they compare bit for bit. */
#include <stdio.h>
#include "gps-sim.h"
#include "almanac.h"

int main(void) {
    almanac_gps_t *alm = almanac_init();    /* the parser fills this (static) almanac */
    const int rc = (int) almanac_read_file();
    printf("%u %d\n", alm->valid, rc);
    for (int sv = 0; sv < MAX_SAT; sv++) {
        const almanac_prn_t *a = &alm->sv[sv];
        printf("%u %u %u %u %u %u %d %a %a %a %a %a %a %a %a %a %a\n", a->svid, a->svn, a->ura, a->health, a->config_code,
               a->valid, a->toa.week, a->e, a->delta_i, a->omegadot, a->sqrta, a->omega0, a->aop, a->m0, a->af0, a->af1,
               a->toa.sec);
    }
    return 0;
}
