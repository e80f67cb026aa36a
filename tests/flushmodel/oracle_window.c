/* oracle_window.c -- TEST INFRASTRUCTURE ONLY.  Compiles the oracle's deflate unchanged and adds read-only accessors to its state:
 * the window buffer (2 * w_size bytes) and the bytes slid out of it, so tests/flushmodel can compare the stale bytes zb_bgzf.h's
 * rule predicts with what the oracle's window holds after each full flush. */
#include "../../oracle/zo_deflate.c"

const uint8_t *fm_oracle_window(const zo_stream *strm) { return ((const dstate *)strm->state)->window; }
uint64_t fm_oracle_abs_base(const zo_stream *strm) { return ((const dstate *)strm->state)->abs_base; }
