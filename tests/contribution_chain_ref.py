"""Reference of the two phase-2 ceremony calls in the exponent, shared by the CPU and GPU tiers.

A point is its discrete log over the group's generator (0 = the identity).  A record is a dict of the exponents of its five
members (after_g1, s_g1, s_x_g1 over g1; r_g2, r_x_g2 over g2).
  contribute_key      g16_pk_contribute on a key given by its exponents (pk_verify_ref.key_exponents): delta_g1 and
                      delta_g2 times delta, h_query and l_query times delta^-1, nothing else touched
  record / chain      what honest contributors publish: after = x D, s_x = x s, r_x = x r
  verdict             what g16_contribution_chain_pairs decides: its refusal message, or the exponents p, q of its 4 count
                      G1 and 4 count G2 output points; equation k holds iff p_2k q_2k = p_2k+1 q_2k+1 mod r (bilinearity)
  tamperings          the cases every tier checks, each with the refusal or the exact set of broken equations it causes."""

MEMBERS = ("after_g1", "s_g1", "s_x_g1", "r_g2", "r_x_g2")


def contribute_key(k, delta, r):
    """the exponents of g16_pk_contribute(delta) applied to key exponents k"""
    di = pow(delta, -1, r)
    out = dict(k)
    out["h_query"] = [x * di % r for x in k["h_query"]]
    out["l_query"] = [x * di % r for x in k["l_query"]]
    out["delta_g1"] = k["delta_g1"] * delta % r
    out["delta_g2"] = k["delta_g2"] * delta % r
    return out


def record(d, x, s, rr, r):
    """contributor's record for secret x on running point d, chosen point s, hash point rr"""
    return dict(after_g1=d * x % r, s_g1=s % r, s_x_g1=s * x % r, r_g2=rr % r, r_x_g2=rr * x % r)


def chain(start, xs, r, seed=1):
    """(end, records) of honest contributions xs from start; s and r of record i are fixed functions of the seed"""
    d, recs = start % r, []
    for i, x in enumerate(xs):
        recs.append(record(d, x, 0x5A17 * (seed + 7 * i) + 3, 0x4A5B * (seed + 11 * i) + 5, r))
        d = recs[-1]["after_g1"]
    return d, recs


def verdict(start, end, recs, r):
    """("refuse", message) as the call words it, or ("pairs", p, q)"""
    named = [("start_g1", start), ("end_g1", end)] + [(f"records[{i}].{m}", c[m]) for i, c in enumerate(recs) for m in MEMBERS]
    for name, e in named:
        if e % r == 0:
            return ("refuse", f"{name}: point is the identity")
    if end % r != recs[-1]["after_g1"] % r:
        return ("refuse", f"records[{len(recs) - 1}].after_g1: not end_g1")
    p, q = [], []
    d = start
    for c in recs:
        p += [c["s_g1"], c["s_x_g1"], d, c["after_g1"]]
        q += [c["r_x_g2"], c["r_g2"], c["r_x_g2"], c["r_g2"]]
        d = c["after_g1"]
    return ("pairs", [x % r for x in p], [x % r for x in q])


def failing(p, q, r):
    """the equations k with p_2k q_2k != p_2k+1 q_2k+1"""
    return {k for k in range(len(p) // 2) if p[2 * k] * q[2 * k] % r != p[2 * k + 1] * q[2 * k + 1] % r}


def outcome(start, end, recs, r):
    """the refusal message, or the set of failing equations"""
    v = verdict(start, end, recs, r)
    return v[1] if v[0] == "refuse" else failing(v[1], v[2], r)


def tamperings(start, xs, r, other_start):
    """(name, start, end, records, expected) for a chain of len(xs) >= 3 honest contributions; expected is the refusal
    message or the exact set of failing equations"""
    n = len(xs)
    assert n >= 3
    end, recs = chain(start, xs, r)
    cp = lambda: [dict(c) for c in recs]
    out = []
    t = cp()   # s_x of another secret: record 1's proof of knowledge alone
    t[1]["s_x_g1"] = t[1]["s_g1"] * (xs[1] + 1) % r
    out.append(("s_x of another x", start, end, t, {2}))
    t = cp()   # after_g1 of record 0 not x D: its step and the next one
    t[0]["after_g1"] = t[0]["after_g1"] * 3 % r
    out.append(("after_g1 not x D", start, end, t, {1, 3}))
    t = cp()   # records 0 and 1 swapped: the step of each and of the record after them (the proofs of knowledge are still
    t[0], t[1] = t[1], t[0]   # each contributor's own)
    out.append(("two records swapped", start, end, t, {1, 3, 5}))
    t = cp()   # record 1 dropped: the step of the record that follows it
    del t[1]
    out.append(("a record dropped", start, end, t, {3}))
    _, foreign = chain(other_start, xs, r, seed=9)   # record 1 replayed from a chain with another start
    t = cp()
    t[1] = dict(foreign[1])
    out.append(("a record replayed from another chain", start, end, t, {3, 5}))
    t = cp()
    out.append(("end_g1 not the chain's end", start, end * 2 % r, t, f"records[{n - 1}].after_g1: not end_g1"))
    t = cp()   # the last record dropped: the chain stops short of end_g1
    out.append(("the last record dropped", start, end, t[:-1], f"records[{n - 2}].after_g1: not end_g1"))
    for i, m in ((1, "r_x_g2"), (0, "s_g1"), (n - 1, "r_g2")):
        t = cp()
        t[i][m] = 0
        out.append((f"records[{i}].{m} the identity", start, end, t, f"records[{i}].{m}: point is the identity"))
    out.append(("start_g1 the identity", 0, end, cp(), "start_g1: point is the identity"))
    return out


def phase1_chains(tau0, alpha0, beta0, contributions, r):
    """the three phase-1 chains over contributions (tau_k, alpha_k, beta_k) to T(tau0, alpha0, beta0): for each of
    tau_g1[1], alpha_tau_g1[0], beta_tau_g1[0], (start, end, records)"""
    out = {}
    for j, (name, x0) in enumerate((("tau_g1[1]", tau0), ("alpha_tau_g1[0]", alpha0), ("beta_tau_g1[0]", beta0))):
        xs = [c[j] for c in contributions]
        end, recs = chain(x0, xs, r, seed=3 + j)
        out[name] = (x0 % r, end, recs)
    return out
