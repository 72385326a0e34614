// daemon_main.cc — `cdprobe-daemon {run,check}`: the fabric-probe slice of
// cmd/compute-domain-daemon, in C++ because the image has no Go toolchain
// (SURVEY.md §8f n1; the Go patch itself is in INTEGRATION.md §2).
//
// It mirrors the reference's interface for this path — same sub-commands, same
// env contract (cmd/compute-domain-daemon/main.go:104-166: CLIQUE_ID,
// COMPUTE_DOMAIN_UUID, …), same texts and exit codes:
//
//   check  (main.go:435-459)  CLIQUE_ID == ""  -> prints
//          "check succeeded (noop, clique ID is empty)"; otherwise runs
//          `nvidia-imex-ctl -c /imexd/imexd.cfg -q` and requires exactly
//          "READY\n".  THEN (new) consults the cached probe verdict; a missing
//          verdict does not gate (probe unsupported / not run yet).
//          exit 0 = ready, exit 1 = not ready (error text on stderr, as
//          urfave/cli prints a returned error).
//   run    (main.go:212-347)  requires COMPUTE_DOMAIN_UUID ("CDI container
//          edits did not apply…"), REMOVES any verdict a previous pod left in
//          the per-domain host-path mount (computedomain.go:170-177 survives
//          restarts), opens the probe through the C ABI (dlopen libcdprobe.so,
//          like the Go shim), runs it at start, on every SIGUSR1 (stand-in for
//          the daemon-set update the Go update loops deliver) and every
//          FABRIC_PROBE_INTERVAL_S seconds when set, writes the verdict
//          atomically (stamped with POD_UID + boot id so `check` ignores one it
//          does not own), reopens the handle after a timeout, exits on
//          SIGTERM/SIGINT.  `--once` runs one pass.
//
// The verdict file is ONE schema shared with the Go patch
// (integration/cmd/compute-domain-daemon/fabricprobe.go, struct
// fabricProbeVerdict): tests/test_daemon.py parses the Go struct tags and
// checks what this binary writes against them.
//
// The binary contains no CUDA: everything device-side is behind libcdprobe.so.
#include <dlfcn.h>
#include <errno.h>
#include <poll.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <string>

#include "../../include/cdprobe.h"

namespace {

const char* kImexCtl = "nvidia-imex-ctl";          // main.go:47 imexCtlBinaryName
const char* kImexCfg = "/imexd/imexd.cfg";         // main.go:44-51
const char* kDefaultVerdict = "/imexd/fabricprobe.json";

std::string env_or(const char* name, const char* dflt) {
  const char* v = getenv(name);
  return (v && *v) ? v : dflt;
}

// ---- check -----------------------------------------------------------------
// Returns 0 when stdout+stderr of the child is exactly "READY\n" and it exited 0.
int imex_daemon_ready(std::string* why) {
  const std::string bin = env_or("CDPROBE_IMEX_CTL", kImexCtl);  // test hook
  int pfd[2];
  if (pipe(pfd) != 0) {
    *why = std::string("IMEX daemon check failed: error running ") + bin + ": " + strerror(errno);
    return 1;
  }
  const pid_t pid = fork();
  if (pid < 0) {
    *why = std::string("IMEX daemon check failed: error running ") + bin + ": " + strerror(errno);
    return 1;
  }
  if (pid == 0) {
    dup2(pfd[1], 1);
    dup2(pfd[1], 2);
    close(pfd[0]);
    close(pfd[1]);
    execlp(bin.c_str(), bin.c_str(), "-c", kImexCfg, "-q", (char*)nullptr);
    fprintf(stderr, "exec: %s", strerror(errno));
    _exit(127);
  }
  close(pfd[1]);
  std::string out;
  char buf[512];
  ssize_t k;
  while ((k = read(pfd[0], buf, sizeof(buf))) > 0) out.append(buf, (size_t)k);
  close(pfd[0]);
  int st = 0;
  waitpid(pid, &st, 0);
  if (!WIFEXITED(st) || WEXITSTATUS(st) != 0) {
    *why = "IMEX daemon check failed: error running " + bin + ": exit status " +
           std::to_string(WIFEXITED(st) ? WEXITSTATUS(st) : -1);
    return 1;
  }
  if (out != "READY\n") {
    *why = "IMEX daemon not ready: " + out;
    return 1;
  }
  return 0;
}

// Minimal reader of the verdict file this binary writes (flat JSON, known keys).
bool json_field(const std::string& doc, const char* key, std::string* val) {
  const std::string k = std::string("\"") + key + "\":";
  size_t p = doc.find(k);
  if (p == std::string::npos) return false;
  p += k.size();
  while (p < doc.size() && doc[p] == ' ') ++p;
  size_t e = p;
  if (p < doc.size() && doc[p] == '"') {
    e = doc.find('"', p + 1);
    if (e == std::string::npos) return false;
    *val = doc.substr(p + 1, e - p - 1);
    return true;
  }
  while (e < doc.size() && doc[e] != ',' && doc[e] != '}' && doc[e] != '\n') ++e;
  *val = doc.substr(p, e - p);
  return true;
}

std::string boot_id() {
  FILE* f = fopen("/proc/sys/kernel/random/boot_id", "r");
  if (f == nullptr) return "";
  char buf[80] = {0};
  if (fgets(buf, sizeof(buf), f) == nullptr) buf[0] = 0;
  fclose(f);
  std::string b = buf;
  while (!b.empty() && (b.back() == '\n' || b.back() == ' ')) b.pop_back();
  return b;
}

int cmd_check() {
  const std::string clique = env_or("CLIQUE_ID", "");
  if (clique.empty()) {
    printf("check succeeded (noop, clique ID is empty)\n");  // main.go:437
  } else {
    std::string why;
    if (imex_daemon_ready(&why) != 0) {
      fprintf(stderr, "%s\n", why.c_str());
      return 1;
    }
  }
  // the fabric-probe verdict written by `run`
  const std::string path = env_or("FABRIC_PROBE_VERDICT_PATH", kDefaultVerdict);
  FILE* f = fopen(path.c_str(), "r");
  if (f == nullptr) return 0;  // no verdict: probe unsupported or not run yet — do not gate
  std::string doc;
  char buf[4096];
  size_t k;
  while ((k = fread(buf, 1, sizeof(buf), f)) > 0) doc.append(buf, k);
  fclose(f);
  std::string ok, err, t, unreachable, slow, minr, minw, owner, boot;
  if (!json_field(doc, "ok", &ok)) {
    fprintf(stderr, "fabric probe verdict unreadable: %s\n", path.c_str());
    return 1;
  }
  // a verdict written by another pod (the mount outlives pods) or before a reboot says nothing about
  // THIS pod's fabric: treated like a missing one
  const std::string my_uid = env_or("POD_UID", "");
  if (json_field(doc, "pod_uid", &owner) && !owner.empty() && !my_uid.empty() && owner != my_uid) return 0;
  const std::string my_boot = boot_id();
  if (json_field(doc, "boot_id", &boot) && !boot.empty() && !my_boot.empty() && boot != my_boot) return 0;
  long max_age = atol(env_or("FABRIC_PROBE_MAX_AGE_S", "0").c_str());
  const long interval = atol(env_or("FABRIC_PROBE_INTERVAL_S", "0").c_str());
  if (max_age <= 0 && interval > 0) max_age = 3 * interval + 60;  // periodic re-probe on: a verdict must keep coming
  if (max_age > 0 && json_field(doc, "time_unix", &t) && time(nullptr) - atol(t.c_str()) > max_age) {
    fprintf(stderr, "fabric probe verdict is stale (%ld s old)\n", (long)(time(nullptr) - atol(t.c_str())));
    return 1;
  }
  if (ok != "true") {
    json_field(doc, "error", &err);
    json_field(doc, "unreachable_pairs", &unreachable);
    if (!json_field(doc, "slow_pairs", &slow)) slow = "0";
    json_field(doc, "min_gbps_read", &minr);
    json_field(doc, "min_gbps_write", &minw);
    fprintf(stderr, "fabric probe failed: %s unreachable pair(s), %s slow pair(s), min read %.0f GB/s, min write %.0f GB/s%s%s\n",
            unreachable.c_str(), slow.c_str(), atof(minr.c_str()), atof(minw.c_str()), err.empty() ? "" : ": ", err.c_str());
    return 1;
  }
  return 0;
}

// ---- run -------------------------------------------------------------------
struct Lib {
  void* dl = nullptr;
  int (*open)(const cdprobe_config_t*, cdprobe_t**) = nullptr;
  int (*run)(cdprobe_t*, cdprobe_result_t*) = nullptr;
  void (*close)(cdprobe_t*) = nullptr;
  const char* (*strerror_)(int) = nullptr;
  const char* (*last_error)(void) = nullptr;
  uint32_t (*abi)(void) = nullptr;
  int (*topology)(uint32_t, cdprobe_topology_t*) = nullptr;
  int (*diagnose)(cdprobe_t*, uint32_t, uint32_t, uint32_t, uint32_t, cdprobe_diag_t*) = nullptr;  // optional
  int (*set_option)(cdprobe_t*, uint32_t, uint64_t) = nullptr;                                      // optional
  int (*links)(cdprobe_t*, cdprobe_links_t*) = nullptr;                                             // optional
};

bool load_lib(Lib* L, std::string* why) {
  const std::string path = env_or("CDPROBE_LIBRARY", "libcdprobe.so");
  L->dl = dlopen(path.c_str(), RTLD_LAZY | RTLD_GLOBAL);
  if (L->dl == nullptr) {
    *why = std::string("cannot load ") + path + ": " + dlerror();
    return false;
  }
  *(void**)&L->open = dlsym(L->dl, "cdprobe_open");
  *(void**)&L->run = dlsym(L->dl, "cdprobe_run");
  *(void**)&L->close = dlsym(L->dl, "cdprobe_close");
  *(void**)&L->strerror_ = dlsym(L->dl, "cdprobe_strerror");
  *(void**)&L->last_error = dlsym(L->dl, "cdprobe_last_error");
  *(void**)&L->abi = dlsym(L->dl, "cdprobe_abi_version");
  *(void**)&L->topology = dlsym(L->dl, "cdprobe_topology");
  *(void**)&L->diagnose = dlsym(L->dl, "cdprobe_diagnose");
  *(void**)&L->set_option = dlsym(L->dl, "cdprobe_set_option");
  *(void**)&L->links = dlsym(L->dl, "cdprobe_links");
  if (!L->open || !L->run || !L->close || !L->strerror_ || !L->last_error || !L->abi) {
    *why = "libcdprobe.so lacks an ABI symbol";
    return false;
  }
  if (L->abi() != CDPROBE_ABI_VERSION) {
    *why = "libcdprobe.so ABI version mismatch";
    return false;
  }
  return true;
}

volatile sig_atomic_t g_stop = 0, g_rerun = 0;
int ppoll_nofd(const timespec* ts, const sigset_t* mask) { return ppoll(nullptr, 0, ts, mask); }
void on_term(int) { g_stop = 1; }
void on_usr1(int) { g_rerun = 1; }

bool env_on(const char* name) {
  const std::string v = env_or(name, "");
  return v == "1" || v == "true" || v == "TRUE" || v == "True";
}

bool write_verdict(const std::string& path, const cdprobe_result_t* r, int rc, const char* err,
                   const cdprobe_links_t* links = nullptr) {
  const std::string tmp = path + ".tmp";
  FILE* f = fopen(tmp.c_str(), "w");
  if (f == nullptr) return false;
  const bool ok = rc == CDPROBE_OK && r != nullptr && r->verdict != 0;
  const unsigned unreachable = r ? r->unreachable_pairs : 0u;
  // schema 2 — field for field the Go struct fabricProbeVerdict (integration/cmd/compute-domain-daemon/fabricprobe.go)
  fprintf(f, "{\"schema\": 2,\n \"time_unix\": %ld,\n \"pod_uid\": \"%s\",\n \"boot_id\": \"%s\",\n \"ok\": %s,\n \"n\": %u,\n",
          (long)time(nullptr), env_or("POD_UID", "").c_str(), boot_id().c_str(), ok ? "true" : "false", r ? r->n : 0u);
  fprintf(f, " \"unreachable_pairs\": %u,\n \"slow_pairs\": %u,\n", unreachable, r ? r->slow_pairs : 0u);
  fprintf(f, " \"min_gbps_read\": %.1f,\n \"min_gbps_write\": %.1f,\n \"gate_gbps_read\": %.1f,\n \"gate_gbps_write\": %.1f,\n",
          r ? r->min_gbps_read : 0.f, r ? r->min_gbps_write : 0.f, r ? r->gate_gbps_read : 0.f, r ? r->gate_gbps_write : 0.f);
  fprintf(f, " \"probe_ms\": %.3f,\n \"bytes_per_pair\": %llu,\n", r ? r->probe_ms : 0.0,
          r ? (unsigned long long)r->bytes_per_pair : 0ull);
  // the matrices themselves (row-major n x n; reach cells are 0/1 integers), for operators: the CRD status
  // stays Ready/NotReady
  {
    const uint32_t n = r ? r->n : 0u;
    const char* names[4] = {"reach_read", "reach_write", "gbps_read", "gbps_write"};
    for (int k = 0; k < 4; ++k) {
      fprintf(f, " \"%s\": [", names[k]);
      for (uint32_t i = 0; i < n; ++i)
        for (uint32_t j = 0; j < n; ++j) {
          const uint32_t c = i * CDPROBE_MAX_GPUS + j;
          if (k == 0) fprintf(f, "%u", (unsigned)r->reach_read[c]);
          else if (k == 1) fprintf(f, "%u", (unsigned)r->reach_write[c]);
          else fprintf(f, "%.1f", k == 2 ? r->gbps_read[c] : r->gbps_write[c]);
          if (!(i == n - 1 && j == n - 1)) fputc(',', f);
        }
      fprintf(f, "],\n");
    }
  }
  std::string e = err ? err : "";
  for (char& c : e)
    if (c == '"' || c == '\\' || c == '\n') c = ' ';
  fprintf(f, " \"error\": \"%s\"}\n", e.c_str());
  fclose(f);
  if (rename(tmp.c_str(), path.c_str()) != 0) return false;
  // Prometheus textfile (INTEGRATION.md §4): same series the Go daemon would register in pkg/metrics
  const std::string mpath = env_or("FABRIC_PROBE_METRICS_PATH", "");
  if (!mpath.empty() && r != nullptr) {
    const std::string mtmp = mpath + ".tmp";
    FILE* m = fopen(mtmp.c_str(), "w");
    if (m != nullptr) {
      fprintf(m, "# TYPE nvidia_dra_fabric_probe_duration_seconds gauge\nnvidia_dra_fabric_probe_duration_seconds %.6f\n",
              r->probe_ms / 1e3);
      fprintf(m, "# TYPE nvidia_dra_fabric_probe_unreachable_pairs gauge\nnvidia_dra_fabric_probe_unreachable_pairs %u\n",
              unreachable);
      fprintf(m, "# TYPE nvidia_dra_fabric_probe_slow_pairs gauge\nnvidia_dra_fabric_probe_slow_pairs %u\n", r->slow_pairs);
      fprintf(m, "# TYPE nvidia_dra_fabric_probe_ok gauge\nnvidia_dra_fabric_probe_ok %d\n", ok ? 1 : 0);
      fprintf(m, "# TYPE nvidia_dra_fabric_probe_pair_gbps gauge\n");
      for (uint32_t i = 0; i < r->n; ++i)
        for (uint32_t j = 0; j < r->n; ++j) {
          if (i == j && r->n > 1) continue;
          const uint32_t c = i * CDPROBE_MAX_GPUS + j;
          fprintf(m, "nvidia_dra_fabric_probe_pair_gbps{src=\"%u\",dst=\"%u\",op=\"read\"} %.1f\n", i, j, r->gbps_read[c]);
          fprintf(m, "nvidia_dra_fabric_probe_pair_gbps{src=\"%u\",dst=\"%u\",op=\"write\"} %.1f\n", i, j, r->gbps_write[c]);
        }
      if (links != nullptr) {  // per-link NVLink counters of the pass, for the GPUs NVML could sample
        const std::string node = env_or("NODE_NAME", "");
        const char* dirs[2] = {"tx", "rx"};
        const char* counters[3] = {"replay", "recovery", "crc"};
        fprintf(m, "# TYPE nvidia_dra_fabric_probe_link_kib gauge\n");
        for (uint32_t d = 0; d < links->n_devices; ++d)
          for (int l = 0; l < CDPROBE_NVLINK_MAX_LINKS && links->dev[d].status == 0; ++l)
            for (int k = 0; k < 2; ++k)
              fprintf(m, "nvidia_dra_fabric_probe_link_kib{node=\"%s\",gpu=\"%s\",link=\"%d\",dir=\"%s\"} %llu\n",
                      node.c_str(), links->dev[d].uuid, l, dirs[k],
                      (unsigned long long)(k == 0 ? links->dev[d].tx_kib[l] : links->dev[d].rx_kib[l]));
        fprintf(m, "# TYPE nvidia_dra_fabric_probe_link_errors gauge\n");
        for (uint32_t d = 0; d < links->n_devices; ++d)
          for (int l = 0; l < CDPROBE_NVLINK_MAX_LINKS && links->dev[d].status == 0; ++l)
            for (int k = 0; k < 3; ++k)
              fprintf(m, "nvidia_dra_fabric_probe_link_errors{node=\"%s\",gpu=\"%s\",link=\"%d\",counter=\"%s\"} %llu\n",
                      node.c_str(), links->dev[d].uuid, l, counters[k], (unsigned long long)links->dev[d].errors[l][k]);
      }
      fclose(m);
      rename(mtmp.c_str(), mpath.c_str());
    }
  }
  return true;
}

// One log line per cell, for at most 8 unreachable cells whose mapping is up (an integrity failure, not a torn-down
// peer): where the cell's bytes went wrong and how (cdprobe_diagnose).  Read cells are re-read by the issuer (what
// crossed the fabric) and, when the target is a rank of this process, by the target too (what is at rest); write
// cells by the target, which holds the landing slot.
void log_diagnoses(const Lib& L, cdprobe_t* h, const cdprobe_result_t& r) {
  int left = 8;
  for (uint32_t i = 0; i < r.n; ++i)
    for (uint32_t j = 0; j < r.n; ++j)
      for (uint32_t op = CDPROBE_OP_READ; op <= CDPROBE_OP_WRITE; ++op) {
        const uint32_t c = i * CDPROBE_MAX_GPUS + j;
        if ((i == j && r.n > 1) || !((r.row_mask >> i) & 1u) || left == 0) continue;
        if (r.status[c] != 0 || r.status[j * CDPROBE_MAX_GPUS + i] != 0) continue;
        if ((op == CDPROBE_OP_READ ? r.reach_read[c] : r.reach_write[c]) != 0) continue;
        --left;
        const char* opname = op == CDPROBE_OP_READ ? "read" : "write";
        const uint32_t reader = op == CDPROBE_OP_READ ? i : j;
        cdprobe_diag_t d;
        int rc = L.diagnose(h, op, i, j, reader, &d);
        if (rc != CDPROBE_OK) {
          fprintf(stderr, "fabric probe diagnosis: %s %u -> %u, reader %u: %s: %s\n", opname, i, j, reader, L.strerror_(rc),
                  L.last_error());
          continue;
        }
        std::string first = d.bad_words ? std::to_string((unsigned long long)d.first_bad) : "none";
        std::string bits;
        int order[64];
        for (int b = 0; b < 64; ++b) order[b] = b;
        std::stable_sort(order, order + 64, [&](int a, int b) { return d.bit_flips[a] > d.bit_flips[b]; });
        for (int k = 0; k < 8 && d.bit_flips[order[k]] != 0; ++k)
          bits += " " + std::to_string(order[k]) + ":" + std::to_string((unsigned long long)d.bit_flips[order[k]]);
        if (bits.empty()) bits = " none";
        std::string where;
        cdprobe_diag_t t;
        if (op == CDPROBE_OP_READ && i != j && L.diagnose(h, op, i, j, j, &t) == CDPROBE_OK) {
          if (d.bad_words != 0 && t.bad_words == 0) where = "; in transit";
          else if (t.bad_words == d.bad_words && t.first_bad == d.first_bad && t.last_bad == d.last_bad) where = "; at rest";
          else where = "; the target reads " + std::to_string((unsigned long long)t.bad_words) + " bad word(s)";
        }
        fprintf(stderr,
                "fabric probe diagnosis: %s %u -> %u, reader %u: %llu/%llu bad words, %llu bad granule(s), first bad byte %s; "
                "flip %llu zero %llu displaced %llu stale %llu foreign %llu; bits%s%s\n",
                opname, i, j, reader, (unsigned long long)d.bad_words, (unsigned long long)(d.bytes / 8),
                (unsigned long long)d.bad_granules, first.c_str(), (unsigned long long)d.kind_count[CDPROBE_DIAG_FLIP],
                (unsigned long long)d.kind_count[CDPROBE_DIAG_ZERO], (unsigned long long)d.kind_count[CDPROBE_DIAG_DISPLACED],
                (unsigned long long)d.kind_count[CDPROBE_DIAG_STALE], (unsigned long long)d.kind_count[CDPROBE_DIAG_FOREIGN],
                bits.c_str(), where.c_str());
      }
}

// One log line per GPU of the pass with a link lost or an error counter risen, e.g.
//   fabric probe links: GPU-… link 7 (remote 0000:05:00.0): replay +312 recovery +0 crc +41; link 11 lost
void log_links(const cdprobe_links_t& k) {
  for (uint32_t d = 0; d < k.n_devices; ++d) {
    const cdprobe_link_device_t& x = k.dev[d];
    if (x.status != 0 || (x.lost_mask == 0 && x.error_mask == 0)) continue;
    std::string line;
    for (int l = 0; l < CDPROBE_NVLINK_MAX_LINKS; ++l) {
      if ((x.error_mask >> l) & 1u) {
        char buf[160];
        snprintf(buf, sizeof(buf), "link %d%s%s%s: replay +%llu recovery +%llu crc +%llu", l,
                 x.remote_bus_id[l][0] ? " (remote " : "", x.remote_bus_id[l], x.remote_bus_id[l][0] ? ")" : "",
                 (unsigned long long)x.errors[l][CDPROBE_LINK_REPLAY],
                 (unsigned long long)x.errors[l][CDPROBE_LINK_RECOVERY], (unsigned long long)x.errors[l][CDPROBE_LINK_CRC]);
        line += (line.empty() ? "" : "; ") + std::string(buf);
      }
      if ((x.lost_mask >> l) & 1u) line += (line.empty() ? "" : "; ") + std::string("link ") + std::to_string(l) + " lost";
    }
    fprintf(stderr, "fabric probe links: %s %s\n", x.uuid, line.c_str());
  }
}

// Turns the link counters on for a freshly opened handle, when asked for and the library has them.
void enable_links(const Lib& L, cdprobe_t* h, bool want) {
  if (!want || !L.set_option || !L.links) return;
  if (L.set_option(h, CDPROBE_OPT_LINK_COUNTERS, 1) != CDPROBE_OK)
    fprintf(stderr, "fabric probe links: cannot enable the link counters: %s\n", L.last_error());
}

// Signals are blocked for the whole of run() and only delivered inside sigsuspend/sigtimedwait-style waits:
// the "check the flag, then sleep" sequence cannot lose a SIGTERM or SIGUSR1 that lands in between.
int wait_for_signal(const sigset_t* unblocked, long timeout_s) {
  if (timeout_s <= 0) {
    sigsuspend(unblocked);  // returns after a handler ran
    return 0;
  }
  // ppoll with no fds == an interruptible sleep that atomically installs the unblocked mask
  timespec ts = {timeout_s, 0};
  return ppoll_nofd(&ts, unblocked);
}

int cmd_run(bool once) {
  if (env_or("COMPUTE_DOMAIN_UUID", "").empty()) {  // main.go:217-219
    fprintf(stderr, "CDI container edits did not apply -- is CDI enabled in your container runtime?\n");
    return 1;
  }
  const std::string verdict_path = env_or("FABRIC_PROBE_VERDICT_PATH", kDefaultVerdict);
  // /imexd is a per-domain host-path mount that outlives pods and container restarts: whatever verdict is there
  // was not produced by this process.  Until this run has probed there is no verdict (check does not gate).
  if (unlink(verdict_path.c_str()) != 0 && errno != ENOENT)
    fprintf(stderr, "cannot remove stale %s: %s\n", verdict_path.c_str(), strerror(errno));
  Lib L;
  std::string why;
  if (!load_lib(&L, &why)) {
    // ErrUnsupported: log and carry on without a verdict; check() will not gate on it
    fprintf(stderr, "fabric probe not supported on this node: %s\n", why.c_str());
    return 0;
  }
  cdprobe_config_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.abi = CDPROBE_ABI_VERSION;
  cfg.n_gpus = 0;  // every GPU the management CDI device exposes (cdi.go:270-275)
  cfg.bytes = strtoull(env_or("FABRIC_PROBE_BYTES", "1073741824").c_str(), nullptr, 10);
  const std::string mode = env_or("FABRIC_PROBE_MODE", "sliced");
  cfg.mode = mode == "full" ? CDPROBE_MODE_FULL : mode == "reach-only" ? CDPROBE_MODE_REACH_ONLY : CDPROBE_MODE_SLICED;
  cfg.min_fraction = (float)atof(env_or("FABRIC_PROBE_MIN_FRACTION", "0").c_str());
  cfg.link_peak_gbps = (float)atof(env_or("FABRIC_PROBE_LINK_PEAK_GBPS", "0").c_str());
  cfg.timeout_ms = (uint32_t)atol(env_or("FABRIC_PROBE_TIMEOUT_MS", "5000").c_str());
  cfg.flags = CDPROBE_FLAG_FABRIC_HANDLES | CDPROBE_FLAG_MIG_AWARE;
  const long interval_s = atol(env_or("FABRIC_PROBE_INTERVAL_S", "0").c_str());
  const bool want_links = env_on("FABRIC_PROBE_LINK_COUNTERS");
  if (L.topology) {
    cdprobe_topology_t topo;
    if (L.topology(1, &topo) == CDPROBE_OK && topo.clique_error[0] == '\0')
      fprintf(stderr, "identified fabric clique: \"%s\" (%u GPU(s))\n", topo.clique_id, topo.n);  // cf. nvlib.go:247,336
  }
  cdprobe_t* h = nullptr;
  int rc = L.open(&cfg, &h);
  if (rc == CDPROBE_ERR_NO_DEVICE || rc == CDPROBE_ERR_UNSUPPORTED) {
    fprintf(stderr, "fabric probe not supported on this node: %s: %s\n", L.strerror_(rc), L.last_error());
    return 0;
  }
  if (rc != CDPROBE_OK) {
    // a node whose probe cannot even be set up is not Ready: say so in the verdict instead of leaving none
    fprintf(stderr, "error opening fabric probe: %s: %s\n", L.strerror_(rc), L.last_error());
    const std::string e = std::string("cdprobe_open: ") + L.strerror_(rc) + ": " + L.last_error();
    write_verdict(verdict_path, nullptr, rc, e.c_str());
    return 1;
  }
  enable_links(L, h, want_links);
  sigset_t block, orig;
  sigemptyset(&block);
  sigaddset(&block, SIGTERM);
  sigaddset(&block, SIGINT);
  sigaddset(&block, SIGUSR1);
  sigprocmask(SIG_BLOCK, &block, &orig);
  sigdelset(&orig, SIGTERM);  // the mask the waits install: our three signals deliverable
  sigdelset(&orig, SIGINT);
  sigdelset(&orig, SIGUSR1);
  struct sigaction sa;
  memset(&sa, 0, sizeof(sa));
  sa.sa_handler = on_term;
  sigaction(SIGTERM, &sa, nullptr);
  sigaction(SIGINT, &sa, nullptr);
  sa.sa_handler = on_usr1;
  sigaction(SIGUSR1, &sa, nullptr);

  int status = 0;
  g_rerun = 1;
  while (!g_stop) {
    if (g_rerun) {
      g_rerun = 0;
      cdprobe_result_t res{};
      if (h == nullptr) {  // the previous pass left the handle unusable: a fresh one for this pass
        rc = L.open(&cfg, &h);
        if (rc != CDPROBE_OK) {
          fprintf(stderr, "error reopening fabric probe: %s: %s\n", L.strerror_(rc), L.last_error());
          const std::string e = std::string("cdprobe_open: ") + L.strerror_(rc) + ": " + L.last_error();
          write_verdict(verdict_path, nullptr, rc, e.c_str());
          h = nullptr;
          status = 2;
          if (once) break;
          wait_for_signal(&orig, interval_s > 0 ? interval_s : 30);
          if (!g_stop) g_rerun = 1;
          continue;
        }
        enable_links(L, h, want_links);
      }
      const timespec t0 = [] { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t; }();
      rc = L.run(h, &res);
      timespec t1;
      clock_gettime(CLOCK_MONOTONIC, &t1);
      fprintf(stderr, "t_fabric_probe %.6f s\n", (t1.tv_sec - t0.tv_sec) + (t1.tv_nsec - t0.tv_nsec) / 1e9);
      const std::string run_err = rc == CDPROBE_OK ? "" : std::string(L.strerror_(rc)) + ": " + L.last_error();
      cdprobe_links_t links;
      const bool have_links = want_links && L.set_option && L.links && L.links(h, &links) == CDPROBE_OK &&
                              links.run_seq != 0 && links.run_seq == res.run_seq;
      if (!write_verdict(verdict_path, &res, rc, run_err.c_str(), have_links ? &links : nullptr))
        fprintf(stderr, "cannot write %s: %s\n", verdict_path.c_str(), strerror(errno));
      fprintf(stderr,
              "fabric probe: verdict %s, %u GPU(s), %u unreachable pair(s), %u slow pair(s), min read %.0f GB/s, min write "
              "%.0f GB/s, %.3f ms\n",
              (rc == CDPROBE_OK && res.verdict) ? "ok" : "FAILED", res.n, res.unreachable_pairs, res.slow_pairs,
              res.min_gbps_read, res.min_gbps_write, res.probe_ms);
      status = (rc == CDPROBE_OK && res.verdict) ? 0 : 2;
      if (have_links) log_links(links);
      if (L.diagnose && rc == CDPROBE_OK && !res.aborted && !res.verdict && res.unreachable_pairs > 0)
        log_diagnoses(L, h, res);
      if (rc == CDPROBE_ERR_TIMEOUT || rc == CDPROBE_ERR_STATE || rc == CDPROBE_ERR_CUDA) {
        // a timed-out or failed pass may leave the handle sticky (cdprobe_run then only returns ERR_STATE):
        // close it; the next pass opens a fresh one
        L.close(h);
        h = nullptr;
      }
      if (once) break;
    }
    if (!g_stop && !g_rerun) {
      wait_for_signal(&orig, interval_s);
      if (interval_s > 0 && !g_stop) g_rerun = 1;  // periodic re-probe (or an early SIGUSR1: same thing)
    }
  }
  if (h != nullptr) L.close(h);
  fprintf(stderr, "Exiting\n");
  return once ? status : 0;
}

// Test hook (tests/test_daemon.py): writes the verdict of a synthetic 2-GPU result through the same writer
// `run` uses, so the schema can be checked against the Go struct without a GPU.
int cmd_selftest_verdict(const char* path, bool ok) {
  cdprobe_result_t r{};
  r.abi = CDPROBE_ABI_VERSION;
  r.n = 2;
  r.verdict = ok ? 1u : 0u;
  for (uint32_t i = 0; i < 2; ++i)
    for (uint32_t j = 0; j < 2; ++j) {
      const uint32_t c = i * CDPROBE_MAX_GPUS + j;
      r.reach_read[c] = 1;
      r.reach_write[c] = (ok || i == j) ? 1 : 0;
      r.gbps_read[c] = i == j ? 0.f : 671.5f;
      r.gbps_write[c] = i == j ? 0.f : 702.25f;
    }
  r.unreachable_pairs = ok ? 0u : 2u;
  r.slow_pairs = 0;
  r.min_gbps_read = 671.5f;
  r.min_gbps_write = 702.25f;
  r.gate_gbps_read = 598.1f;
  r.gate_gbps_write = 625.7f;
  r.probe_ms = 3.21;
  r.bytes_per_pair = 1073741824ull;
  return write_verdict(path, &r, CDPROBE_OK, ok ? "" : "synthetic \"failure\"") ? 0 : 1;
}

}  // namespace

int main(int argc, char** argv) {
  if (argc >= 2 && strcmp(argv[1], "check") == 0) return cmd_check();
  if (argc >= 2 && strcmp(argv[1], "run") == 0) return cmd_run(argc >= 3 && strcmp(argv[2], "--once") == 0);
  if (argc >= 4 && strcmp(argv[1], "selftest-verdict") == 0) return cmd_selftest_verdict(argv[2], strcmp(argv[3], "ok") == 0);
  fprintf(stderr, "usage: cdprobe-daemon {run [--once] | check}\n");
  return 2;
}
