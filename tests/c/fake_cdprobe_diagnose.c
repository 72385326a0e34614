/* fake_cdprobe_diagnose.c — TEST DOUBLE: fake_cdprobe.c plus cdprobe_diagnose, for the daemon's diagnosis log
 * (tests/test_diagnose_cpu.py).  Everything of fake_cdprobe.c applies; one more script item:
 *
 *   corrupt : a passing-looking pass except that read cell 1 -> 0 is unreachable with its mapping up.
 *             cdprobe_diagnose then reports 3 flipped words (bit 17 twice, bit 8 once) when the issuer reads the
 *             cell, and a clean region when the target does: the bytes went wrong in transit.
 *
 * Built with -DFAKE_CDPROBE_NO_DIAGNOSE it exports no cdprobe_diagnose (a library from before the call existed).
 */
#define cdprobe_run fake_base_run
#include "fake_cdprobe.c"
#undef cdprobe_run

static int g_corrupt;  /* the last cdprobe_run played the "corrupt" item */

CDPROBE_API int cdprobe_run(cdprobe_t* h, cdprobe_result_t* r) {
  char item[32];
  script_item(g_runs, item, sizeof(item));
  const int rc = fake_base_run(h, r);
  r->row_mask = 3;
  g_corrupt = !strcmp(item, "corrupt");
  if (g_corrupt) {
    r->reach_read[1 * CDPROBE_MAX_GPUS + 0] = 0;
    r->unreachable_pairs = 1;
    r->verdict = 0;
  }
  return rc;
}

#ifndef FAKE_CDPROBE_NO_DIAGNOSE
CDPROBE_API int cdprobe_diagnose(cdprobe_t* h, uint32_t op, uint32_t issuer, uint32_t target, uint32_t reader,
                                 cdprobe_diag_t* out) {
  if (!h || !out) return CDPROBE_ERR_ARG;
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->op = op;
  out->issuer = issuer;
  out->target = target;
  out->reader = reader;
  out->first_bad = UINT64_MAX;
  if (issuer >= 2 || target >= 2 || reader >= 2) return CDPROBE_ERR_ARG;
  logline("diagnose", (int)(op * 100 + issuer * 10 + target) * 10 + (int)reader);
  out->run_seq = (uint64_t)g_runs;
  out->bytes = 1ull << 30;
  if (g_corrupt && op == CDPROBE_OP_READ && issuer == 1 && target == 0 && reader == 1) {
    out->bad_words = 3;
    out->bad_granules = 2;
    out->first_bad = 4104;
    out->last_bad = 20480;
    out->kind_count[CDPROBE_DIAG_FLIP] = 3;
    out->bit_flips[17] = 2;
    out->bit_flips[8] = 1;
    out->n_samples = 3;
  }
  return CDPROBE_OK;
}
#endif
