/* include/agrep_b200_dropin.h -- the drop-in layer (libagrepb200_dropin.so).
 *
 * These are the reference's OWN entry points for the scan path, same names, same K&R argument lists, same
 * return convention (0 = done, -1 = error with errno = AGREP_ERROR 123), same global side effects
 * (num_of_matched, CurrentByteOffset, NEW_FILE, calls to output()).  exec() (agrep.c:3332) is their only
 * caller (agrep.c:3359-3360, 3430-3431, 3607-3608, 3696-3700); file_out() and newmgrep.c also use fill_buf().
 *
 *   symbol      replaces (reference file:line)        what it does here
 *   ---------   ----------------------------------   ------------------------------------------------------
 *   bitap       bitap.c:78-448                        dispatcher + exact shift-and scan on the GPU; regex: re() on the GPU, re1()
 *   asearch     asearch.c:32-572                      k = 1..4 scan on the GPU
 *   asearch0    asearch.c:574-982                     k = 5..8 scan on the GPU
 *   asearch1    asearch1.c:28-435                     -I/-S/-D cost scan on the GPU
 *   sgrep       sgrep.c:262-682 (+ bm() :694)         simple-literal scan on the GPU
 *   fill_buf    bitap.c:450-477                       read(2) loop (still used by file_out(), mgrep)
 *   alloc_buf   bitap.c:484-494                       unchanged contract
 *   free_buf    bitap.c:496-505                       unchanged contract
 *
 * The library expects the reference's globals (agrep.c:113-140, 135-140: Mask[], Init[], Init1, NO_ERR_MASK,
 * endposition, D_endpos, wildmask, AND, INVERSE, DELIMITER, I, S, DD, JUMP, REGEX, COUNT, ... and output(),
 * re(), re1()) to be provided by the program it is linked into, exactly as the replaced objects did.
 */
#ifndef AGREP_B200_DROPIN_H
#define AGREP_B200_DROPIN_H
#ifdef __cplusplus
extern "C" {
#endif
int  bitap(char old_D_pat[], char *Pattern, int fd, int M, int D);
int  asearch(unsigned char old_D_pat[], int text, unsigned D);
int  asearch0(unsigned char old_D_pat[], int text, unsigned D);
int  asearch1(char old_D_pat[], int Text, unsigned D);
int  sgrep(unsigned char *in_pat, int in_m, int fd, int D, int samepattern);
int  fill_buf(int fd, unsigned char *buf, int record_size);
void alloc_buf(int fd, unsigned char **buf, int size);
void free_buf(int fd, char *buf);
#ifdef __cplusplus
}
#endif
#endif
