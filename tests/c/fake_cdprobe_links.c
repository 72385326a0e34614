/* fake_cdprobe_links.c — the library test double of fake_cdprobe.c, plus cdprobe_set_option and cdprobe_links, for
 * the daemon's link-counter report (tests/test_links_cpu.py).  fake_cdprobe.c is compiled into this translation unit
 * unchanged; built alone, it is a library without cdprobe_links.
 *
 *   FAKE_CDPROBE_LOG    = also receives one "set_option OPTION VALUE" line per cdprobe_set_option.
 *   FAKE_CDPROBE_LINKS  = what cdprobe_links reports for the pass's two GPUs: clean (DATA moved, no error) or error
 *                         (GPU 1: link 7 replay +312 crc +41 to 0000:05:00.0, link 11 lost).
 */
#include "fake_cdprobe.c"

CDPROBE_API int cdprobe_set_option(cdprobe_t* h, uint32_t option, uint64_t value) {
  const char* p = getenv("FAKE_CDPROBE_LOG");
  FILE* f = p ? fopen(p, "a") : NULL;
  if (f) {
    fprintf(f, "set_option %u %llu\n", option, (unsigned long long)value);
    fclose(f);
  }
  return h ? CDPROBE_OK : CDPROBE_ERR_ARG;
}

CDPROBE_API int cdprobe_links(cdprobe_t* h, cdprobe_links_t* out) {
  if (!h || !out) return CDPROBE_ERR_ARG;
  const char* s = getenv("FAKE_CDPROBE_LINKS");
  memset(out, 0, sizeof(*out));
  out->abi = CDPROBE_ABI_VERSION;
  out->n_devices = 2;
  out->run_seq = (uint64_t)g_runs;
  out->sample_ms = 0.5;
  for (int d = 0; d < 2; ++d) {
    cdprobe_link_device_t* x = &out->dev[d];
    x->rank_mask = 1u << d;
    snprintf(x->uuid, sizeof(x->uuid), "GPU-fa4e0000-0000-0000-0000-%012d", d);
    x->link_mask = (1u << CDPROBE_NVLINK_MAX_LINKS) - 1u;
    x->expected_tx_kib = x->expected_rx_kib = 1048576;
    for (int l = 0; l < CDPROBE_NVLINK_MAX_LINKS; ++l) {
      x->tx_kib[l] = 1024;
      x->rx_kib[l] = 2048;
    }
  }
  if (s && !strcmp(s, "error")) {
    cdprobe_link_device_t* x = &out->dev[1];
    x->errors[7][CDPROBE_LINK_REPLAY] = 312;
    x->errors[7][CDPROBE_LINK_CRC] = 41;
    x->error_mask = 1u << 7;
    x->lost_mask = 1u << 11;
    snprintf(x->remote_bus_id[7], sizeof(x->remote_bus_id[7]), "0000:05:00.0");
  }
  return CDPROBE_OK;
}
