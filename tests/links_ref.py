"""Restatement of cdprobe_links' rules (DESIGN §5o), for tests: the payload a probe pass moves between devices, from the
plan's partner table alone, and the delta and mask rules of two NVML samples of one device."""

OP_READ, OP_WRITE = 1, 2
LINKS = 18
FIELDS = ("tx", "rx", "replay", "recovery", "crc")  # bit f of failed_fields is FIELDS[f]
ERR_UNSUPPORTED = -8


def payload(partner, rounds, n, bpp, ops, dev, warm_bytes=0, down=(), ran=None):
    """(tx, rx) bytes per device id of one pass.  partner[r][g] is rank g's partner in round r (-1: idle); dev[g] is
    rank g's device; down holds ordered pairs (issuer, owner) whose mapping is down, which takes both cells of the pair
    out of the schedule; ran is the set of ranks whose kernel ran (default: all).

    In every round a rank writes the slot it owns in its partner (write: its tx, the partner's rx) and reads its slice
    from the partner (read: the partner's tx, its rx); the wake-up before round 0 reads min(warm_bytes, bpp) from the
    round-0 partner.  The loop-back diagonal stays on one device and so does everything between ranks that share one."""
    ran = set(range(n)) if ran is None else set(ran)
    tx, rx = {}, {}

    def add(src, dst, b):
        if dev[src] != dev[dst] and b:
            tx[dev[src]] = tx.get(dev[src], 0) + b
            rx[dev[dst]] = rx.get(dev[dst], 0) + b

    def ok(a, b):
        return (a, b) not in down and (b, a) not in down

    for g in range(n):
        if g not in ran:
            continue
        for r in range(rounds):
            p = partner[r][g]
            if p < 0 or not ok(g, p):
                continue
            if r == 0:
                add(p, g, min(warm_bytes, bpp))
            if ops & OP_WRITE:
                add(g, p, bpp)
            if ops & OP_READ:
                add(p, g, bpp)
    return tx, rx


def delta(before, after):
    """The device row of two samples, each a dict: status, link_mask, value[l][f], failed[l] (bits), remote[l].  A field
    that failed in either sample, or that went backwards, reads 0; failed_fields is the union of the two samples'."""
    status = before["status"] or after["status"]
    row = {"status": status, "link_mask": 0, "lost_mask": 0, "error_mask": 0, "tx_kib": [0] * LINKS,
           "rx_kib": [0] * LINKS, "errors": [[0, 0, 0] for _ in range(LINKS)], "failed_fields": [0] * LINKS,
           "remote_bus_id": [""] * LINKS}
    if status:
        return row
    row["link_mask"] = before["link_mask"]
    row["lost_mask"] = before["link_mask"] & ~after["link_mask"]
    for l in range(LINKS):
        failed = before["failed"][l] | after["failed"][l]
        row["failed_fields"][l] = failed
        row["remote_bus_id"][l] = before["remote"][l]
        d = [0 if (failed >> f) & 1 or after["value"][l][f] < before["value"][l][f]
             else after["value"][l][f] - before["value"][l][f] for f in range(len(FIELDS))]
        row["tx_kib"][l], row["rx_kib"][l] = d[0], d[1]
        row["errors"][l] = d[2:]
        if any(d[2:]):
            row["error_mask"] |= 1 << l
    return row
