/*
 * fake_nvml_links.c — the scriptable fake libnvidia-ml.so.1 of fake_nvml.c, plus the per-link counter entry points
 * that CDPROBE_OPT_LINK_COUNTERS reads (test fixture).  fake_nvml.c is compiled into this translation unit unchanged,
 * so every scenario it knows reads the same here; tests build this file on their own (tests/test_links_*.py), next
 * to the fake the oracle builds.
 *
 * Extra directives, in the same scenario file (FAKE_NVML_SCENARIO); fake_nvml.c skips them:
 *   field G L ID START STEP      field ID of link L (scopeId) of GPU G reads START + STEP x (earlier
 *                                nvmlDeviceGetFieldValues calls on GPU G); an unscripted field reads 0
 *   field_fail G L ID RET        that field returns nvmlReturn_t RET
 *   link_down_after G L          link L of GPU G is active at its first nvmlDeviceGetNvLinkState query only
 *   remote G L BUSID             remote PCI bus id of link L of GPU G (unscripted: NOT_SUPPORTED)
 *   fail fields RET              nvmlDeviceGetFieldValues returns RET
 *   uuid_alias G UUID            nvmlDeviceGetHandleByUUID(UUID) finds GPU G too
 *   field_delay_us N             every nvmlDeviceGetFieldValues call takes N us longer
 * and "unsupported nvlink" also makes every field and remote bus id NOT_SUPPORTED (a PCIe card).
 */
#define nvmlInitWithFlags fake_base_init_with_flags
#define nvmlDeviceGetNvLinkState fake_base_nvlink_state
#include "fake_nvml.c"
#undef nvmlInitWithFlags
#undef nvmlDeviceGetNvLinkState

#include <time.h>

#define MAXF 64

static struct {
  struct {
    int g, l;
    unsigned id;
    unsigned long long start, step;
    int ret;
  } field[MAXF];
  int n_field;
  int fail_fields;
  unsigned char down_after[MAXG][MAXL];
  int state_queries[MAXG][MAXL];
  int field_calls[MAXG];
  char remote[MAXG][MAXL][32];
  char alias[MAXG][96];
  long field_delay_us;
} X;

static void load_links(void) {
  memset(&X, 0, sizeof(X));
  const char* path = getenv("FAKE_NVML_SCENARIO");
  if (!path) return;
  FILE* f = fopen(path, "r");
  if (!f) return;
  char line[256];
  while (fgets(line, sizeof(line), f)) {
    char a[64];
    int x, y, z;
    unsigned id;
    unsigned long long st, sp;
    if (sscanf(line, "field_fail %d %d %u %d", &x, &y, &id, &z) == 4) {
      if (X.n_field < MAXF) {
        X.field[X.n_field].g = x, X.field[X.n_field].l = y, X.field[X.n_field].id = id;
        X.field[X.n_field++].ret = z;
      }
    } else if (sscanf(line, "field %d %d %u %llu %llu", &x, &y, &id, &st, &sp) == 5) {
      if (X.n_field < MAXF) {
        X.field[X.n_field].g = x, X.field[X.n_field].l = y, X.field[X.n_field].id = id;
        X.field[X.n_field].start = st, X.field[X.n_field++].step = sp;
      }
    } else if (sscanf(line, "link_down_after %d %d", &x, &y) == 2) {
      if (x >= 0 && x < MAXG && y >= 0 && y < MAXL) X.down_after[x][y] = 1;
    } else if (sscanf(line, "remote %d %d %31s", &x, &y, a) == 3) {
      if (x >= 0 && x < MAXG && y >= 0 && y < MAXL) snprintf(X.remote[x][y], sizeof(X.remote[x][y]), "%s", a);
    } else if (sscanf(line, "fail fields %d", &x) == 1) {
      X.fail_fields = x;
    } else if (sscanf(line, "uuid_alias %d %63s", &x, a) == 2) {
      if (x >= 0 && x < MAXG) snprintf(X.alias[x], sizeof(X.alias[x]), "%s", a);
    } else if (sscanf(line, "field_delay_us %d", &x) == 1) {
      X.field_delay_us = x;
    }
  }
  fclose(f);
}

nvmlReturn_t nvmlInitWithFlags(unsigned int flags) {
  load_links();
  return fake_base_init_with_flags(flags);
}

nvmlReturn_t nvmlDeviceGetNvLinkState(nvmlDevice_t d, unsigned int link, nvmlEnableState_t* st) {
  const nvmlReturn_t r = fake_base_nvlink_state(d, link, st);
  if (r != NVML_SUCCESS) return r;
  const int g = idx_of(d);
  if (X.state_queries[g][link]++ > 0 && X.down_after[g][link]) *st = NVML_FEATURE_DISABLED;
  return NVML_SUCCESS;
}

nvmlReturn_t nvmlDeviceGetHandleByUUID(const char* uuid, nvmlDevice_t* d) {
  load();
  char buf[96];
  for (int i = 0; i < S.gpus; ++i) {
    nvmlDeviceGetUUID((nvmlDevice_t)(size_t)(i + 1), buf, sizeof(buf));
    if (!strcmp(buf, uuid) || (X.alias[i][0] && !strcmp(X.alias[i], uuid))) {
      *d = (nvmlDevice_t)(size_t)(i + 1);
      return NVML_SUCCESS;
    }
  }
  return NVML_ERROR_NOT_FOUND;
}

nvmlReturn_t nvmlDeviceGetFieldValues(nvmlDevice_t d, int count, nvmlFieldValue_t* v) {
  if (X.field_delay_us > 0) {
    struct timespec ts = {X.field_delay_us / 1000000, (X.field_delay_us % 1000000) * 1000};
    nanosleep(&ts, NULL);
  }
  if (X.fail_fields) return (nvmlReturn_t)X.fail_fields;
  const int g = idx_of(d);
  const unsigned long long k = (unsigned long long)X.field_calls[g]++;
  for (int i = 0; i < count; ++i) {
    v[i].valueType = NVML_VALUE_TYPE_UNSIGNED_LONG_LONG;
    v[i].value.ullVal = 0;
    v[i].nvmlReturn = S.unsup_nvlink ? NVML_ERROR_NOT_SUPPORTED : NVML_SUCCESS;
    for (int f = 0; f < X.n_field && !S.unsup_nvlink; ++f) {
      if (X.field[f].g != g || X.field[f].l != (int)v[i].scopeId || X.field[f].id != v[i].fieldId) continue;
      if (X.field[f].ret) v[i].nvmlReturn = (nvmlReturn_t)X.field[f].ret;
      else v[i].value.ullVal = X.field[f].start + X.field[f].step * k;
    }
  }
  return NVML_SUCCESS;
}

nvmlReturn_t nvmlDeviceGetNvLinkRemotePciInfo_v2(nvmlDevice_t d, unsigned int link, nvmlPciInfo_t* p) {
  const int g = idx_of(d);
  if (S.unsup_nvlink || link >= MAXL || !X.remote[g][link][0]) return NVML_ERROR_NOT_SUPPORTED;
  memset(p, 0, sizeof(*p));
  snprintf(p->busId, sizeof(p->busId), "%s", X.remote[g][link]);
  return NVML_SUCCESS;
}
