/* agrep_b200/csrc/pattern_internal.h -- private to libagrepb200 */
#ifndef AGB_PATTERN_INTERNAL_H
#define AGB_PATTERN_INTERNAL_H
#include "agrep_b200.h"
#ifdef __cplusplus
extern "C" {
#endif
struct agb_pattern { agb_desc d; agb_regex rx; agb_wide wide; };
int  agbi_build(const char *pattern, const agb_options *o, agb_desc *d, char *err, size_t errlen);
/* as agbi_build; a regular expression (o->regex) also fills *rx, and a simple literal of more than 63 positions *wide
 * (refused where wide is NULL) */
int  agbi_build_rx(const char *pattern, const agb_options *o, agb_desc *d, agb_regex *rx, agb_wide *wide, char *err, size_t errlen);
/* Next(S) of a regular expression of M positions */
uint64_t agbi_regex_next(const agb_regex *rx, int M, uint64_t S);
int  agbi_derive(agb_desc *d, char *err, size_t errlen);   /* delim_kind, reset[], start[], nrows from the words */
void agbi_step(const agb_desc *d, const uint64_t *B, uint64_t *A, uint64_t cm);
void agbi_lut_lower1(unsigned char lut[256]);
#ifdef __cplusplus
}
#endif
#endif
