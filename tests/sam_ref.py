"""TEST INFRASTRUCTURE: an independent Python renderer of the SAM rules in DESIGN.md "SAM output", and a structural
validator of SAM text.  Written from the rules, not from salmon_b200/csrc/sam_core.h."""

ACGT = "ACGT"
COMP = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}


def seq_str(codes):
    return "".join(ACGT[c] if c < 4 else "N" for c in codes)


def _cigar(p, L, ref_len):
    lc = min(-p, L) if p < 0 else 0
    rc = min(max(p + L - ref_len, 0), L - lc)
    m = L - lc - rc
    if m == 0:
        return "*"
    return (f"{lc}S" if lc else "") + f"{m}M" + (f"{rc}S" if rc else "")


def render_fragment(name, alns, left, right, ref_names, ref_lens, paired, qual_left=None, qual_right=None):
    """alns: list of (tid, pos, mate_pos, flags, flen, score1, score2); left / right: code arrays of the mapped bases;
    qual_*: bytes or None.  -> the fragment's SAM lines."""
    L = len(left)
    out = []
    nh = len(alns)
    seqs = [seq_str(left), seq_str(right) if right is not None else None]
    quals = [qual_left, qual_right]
    for i, (tid, pos, mpos, fl, flen, s1, s2) in enumerate(alns):
        status = (fl >> 2) & 3
        fw_first, fw_mate = bool(fl & 1), bool(fl & 2)
        if not paired or status == 1:
            mates = {0: (pos, not fw_first)}
        elif status == 2:
            mates = {1: (pos, not fw_first)}
        else:
            mates = {0: (pos, not fw_first), 1: (mpos, not fw_mate)}
        pos1 = lambda p: max(p, 0) + 1
        for m in (0, 1) if paired else (0,):
            o = 1 - m
            flag = 0x100 if i else 0
            if m in mates:
                p, rev = mates[m]
                POS, cig, mapq = pos1(p), _cigar(p, L, ref_lens[tid]), 255
                if rev:
                    flag |= 0x10
            else:
                p, rev = mates[o][0], False
                POS, cig, mapq = pos1(p), "*", 255
                flag |= 0x4
            tlen, rnext, pnext = 0, "*", 0
            if paired:
                flag |= 0x1 | (0x80 if m else 0x40)
                rnext = "="
                if len(mates) == 2:
                    flag |= 0x2
                    if mates[o][1]:
                        flag |= 0x20
                    pnext = pos1(mates[o][0])
                    left_most = mates[m][0] < mates[o][0] or (mates[m][0] == mates[o][0] and m == 0)
                    tlen = flen if left_most else -flen
                elif m in mates:
                    flag |= 0x8
                    pnext = POS
                else:
                    if mates[o][1]:
                        flag |= 0x20
                    pnext = POS
            s = seqs[m]
            q = quals[m]
            if rev:
                s = "".join(COMP[c] for c in reversed(s))
                q = q[::-1] if q is not None else None
            qs = q.decode() if q is not None else "*"
            tags = f"NH:i:{nh}" + (f"\tAS:i:{(s1, s2)[m]}" if m in mates else "")
            out.append("\t".join([name, str(flag), ref_names[tid], str(POS), str(mapq), cig, rnext, str(pnext),
                                  str(tlen), s, qs, tags]))
    return out


def unmapped_type(n_out, decoy, first_flags, paired):
    if decoy:
        return "d"
    if n_out == 0:
        return "u"
    if not paired:
        return None
    st = (first_flags >> 2) & 3
    return None if st == 0 else ("m1" if st == 1 else "m2")


def _cigar_qlen(c):
    import re
    return sum(int(n) for n, op in re.findall(r"(\d+)([MIDNSHP=X])", c) if op in "MIS=X")


def validate(text, n_refs=None):
    """structural checks over a whole SAM file; returns the records grouped by fragment (QNAME runs)"""
    lines = text.splitlines()
    body = [ln for ln in lines if not ln.startswith("@")]
    hdr = [ln for ln in lines if ln.startswith("@")]
    assert hdr and hdr[0].startswith("@HD\tVN:1.0\tSO:unknown")
    sq = [ln for ln in hdr if ln.startswith("@SQ")]
    if n_refs is not None:
        assert len(sq) == n_refs
    assert any(ln.startswith("@PG\tID:salmon") for ln in hdr)
    frags = []
    for ln in body:
        f = ln.split("\t")
        assert len(f) >= 11, ln
        if not frags or frags[-1][0][0] != f[0]:
            frags.append([])
        frags[-1].append(f)
    for recs in frags:
        nh = {int(t[5:]) for r in recs for t in r[11:] if t.startswith("NH:i:")}
        assert len(nh) == 1
        paired = int(recs[0][1]) & 1
        per = 2 if paired else 1
        assert len(recs) == per * nh.pop()
        for k, r in enumerate(recs):
            flag = int(r[1])
            assert bool(flag & 0x100) == (k >= per), recs
            if r[5] != "*":
                assert _cigar_qlen(r[5]) == len(r[9]), r
            if r[10] != "*":
                assert len(r[10]) == len(r[9])
        if paired:
            for a in range(0, len(recs), 2):
                r1, r2 = recs[a], recs[a + 1]
                f1, f2 = int(r1[1]), int(r2[1])
                assert f1 & 0x40 and f2 & 0x80
                assert r1[6] == r2[6] == "="
                assert r1[7] == r2[3] and r2[7] == r1[3], (r1, r2)
                assert int(r1[8]) == -int(r2[8])
                assert bool(f1 & 0x10) == bool(f2 & 0x20) or f2 & 0x4 or f1 & 0x4
    return frags
