/* fake_cdprobe.c — TEST DOUBLE of libcdprobe.so for the daemon's run loop (tests/test_daemon.py), so that
 * `cdprobe-daemon run` (open / run / reopen-after-timeout / signals / periodic passes / verdict writing) is
 * exercised on a box without a GPU.  It implements only what the daemon binds (include/cdprobe.h) and moves no
 * bytes: it is never built into, linked with or loaded by the product.
 *
 *   FAKE_CDPROBE_SCRIPT = comma list consumed one item per cdprobe_run: ok | slow | unreachable | timeout | state
 *                         (the last item repeats);  a leading "openfail" / "unsupported" makes cdprobe_open fail.
 *   FAKE_CDPROBE_LOG    = file that receives one line per open / run / close.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/cdprobe.h"

struct cdprobe {
  int id;
};
static int g_opens, g_runs;
static char g_err[128];

static void logline(const char* what, int a) {
  const char* p = getenv("FAKE_CDPROBE_LOG");
  if (!p) return;
  FILE* f = fopen(p, "a");
  if (!f) return;
  fprintf(f, "%s %d\n", what, a);
  fclose(f);
}

static const char* script_item(int k, char* buf, size_t n) {
  const char* s = getenv("FAKE_CDPROBE_SCRIPT");
  if (!s || !*s) s = "ok";
  const char* last = s;
  for (int i = 0; *s; ++i) {
    const char* e = strchr(s, ',');
    size_t len = e ? (size_t)(e - s) : strlen(s);
    if (strncmp(s, "openfail", len) != 0 && strncmp(s, "unsupported", len) != 0) {
      last = s;
      if (k == 0) break;
      --k;
    }
    if (!e) break;
    s = e + 1;
  }
  const char* e = strchr(last, ',');
  size_t len = e ? (size_t)(e - last) : strlen(last);
  if (len >= n) len = n - 1;
  memcpy(buf, last, len);
  buf[len] = 0;
  return buf;
}

CDPROBE_API uint32_t cdprobe_abi_version(void) { return CDPROBE_ABI_VERSION; }
CDPROBE_API const char* cdprobe_strerror(int rc) {
  switch (rc) {
    case CDPROBE_OK: return "ok";
    case CDPROBE_ERR_TIMEOUT: return "probe timed out";
    case CDPROBE_ERR_STATE: return "handle is in an unusable state";
    case CDPROBE_ERR_CUDA: return "CUDA call failed";
    case CDPROBE_ERR_UNSUPPORTED: return "device or driver lacks a required feature";
    default: return "error";
  }
}
CDPROBE_API const char* cdprobe_last_error(void) { return g_err; }

CDPROBE_API int cdprobe_open(const cdprobe_config_t* cfg, cdprobe_t** out) {
  const char* s = getenv("FAKE_CDPROBE_SCRIPT");
  g_err[0] = 0;
  if (!cfg || !out || cfg->abi != CDPROBE_ABI_VERSION) return CDPROBE_ERR_ABI;
  if (s && strncmp(s, "unsupported", 11) == 0) {
    snprintf(g_err, sizeof(g_err), "fake: no sm_90 device");
    return CDPROBE_ERR_UNSUPPORTED;
  }
  if (s && strncmp(s, "openfail", 8) == 0) {
    snprintf(g_err, sizeof(g_err), "fake: cuMemCreate: CUDA_ERROR_OUT_OF_MEMORY");
    return CDPROBE_ERR_CUDA;
  }
  struct cdprobe* h = (struct cdprobe*)calloc(1, sizeof(*h));
  h->id = ++g_opens;
  logline("open", h->id);
  *out = h;
  return CDPROBE_OK;
}

CDPROBE_API int cdprobe_run(cdprobe_t* h, cdprobe_result_t* r) {
  char item[32];
  script_item(g_runs++, item, sizeof(item));
  logline(item, h ? h->id : -1);
  memset(r, 0, sizeof(*r));
  r->abi = CDPROBE_ABI_VERSION;
  r->n = 2;
  r->bytes_per_pair = 1ull << 30;
  g_err[0] = 0;
  if (!strcmp(item, "timeout")) {
    snprintf(g_err, sizeof(g_err), "device watchdog fired (a peer did not reach a barrier within timeout_ms)");
    r->aborted = 1;
    return CDPROBE_ERR_TIMEOUT;
  }
  if (!strcmp(item, "state")) {
    snprintf(g_err, sizeof(g_err), "handle is unusable after an earlier timeout or CUDA error: close it and open a new one");
    return CDPROBE_ERR_STATE;
  }
  for (int i = 0; i < 2; ++i)
    for (int j = 0; j < 2; ++j) {
      int c = i * CDPROBE_MAX_GPUS + j;
      r->reach_read[c] = 1;
      r->reach_write[c] = (i == j || strcmp(item, "unreachable")) ? 1 : 0;
      r->gbps_read[c] = i == j ? 0.f : (!strcmp(item, "slow") ? 310.f : 674.f);
      r->gbps_write[c] = i == j ? 0.f : 705.f;
    }
  r->min_gbps_read = !strcmp(item, "slow") ? 310.f : 674.f;
  r->min_gbps_write = 705.f;
  r->gate_gbps_read = 604.f;
  r->gate_gbps_write = 631.f;
  r->unreachable_pairs = !strcmp(item, "unreachable") ? 2 : 0;
  r->slow_pairs = !strcmp(item, "slow") ? 2 : 0;
  r->verdict = (!strcmp(item, "ok")) ? 1 : 0;
  r->probe_ms = 3.14;
  r->run_seq = (uint64_t)g_runs;
  return CDPROBE_OK;
}

CDPROBE_API void cdprobe_close(cdprobe_t* h) {
  if (!h) return;
  logline("close", h->id);
  free(h);
}
