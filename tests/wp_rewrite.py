"""Rewrites an H.264 stream so that its B slices carry explicit weights (weighted_bipred_idc 1), without touching their slice data.

Weights never change how slice data is parsed, so the rewrite only has to change two things:
- every PPS: weighted_bipred_idc becomes 1 (a fixed-length field, overwritten in place);
- every B slice header: a pred_weight_table() is inserted after ref_pic_list_modification().  The rest of the slice is copied bit for
  bit: under CAVLC the slice data moves by the inserted bits and gets new rbsp_trailing_bits; under CABAC the header is followed by new
  cabac_alignment_one_bits and the byte-aligned arithmetic-coded data is copied as it is.
Emulation prevention is removed before and redone after.  I and P slices and every other NAL unit are copied unchanged.

The tables are drawn from a seed: denominators 0-7, weights and offsets in [-128, 127] with extremes drawn often, some flags off (the
default weight 2^denominator and offset 0), and every (list-0, list-1) pair of luma or chroma weights within the bound of 8.4.2.3,
-128 <= w0 + w1 <= (denominator == 7 ? 127 : 128), so the stream stays conforming.  `neutral_table` gives denominators 5 and every flag
off: weights 32 and offsets 0, which reproduce default prediction exactly for every partition shape.

Plain Python (no reference sources, no compiled code), so it runs wherever the tests run.
"""
import random

__all__ = ["rewrite", "neutral_table", "random_table", "nal_units", "unescape", "escape"]


# ---- NAL units and emulation prevention ---------------------------------------------------------------------------------

def nal_units(bs):
    """Annex-B stream -> list of (start code bytes, NAL unit bytes incl. header)"""
    bs = bytes(bs)
    starts, i, n = [], 0, len(bs)
    while i + 3 <= n:
        if bs[i] == 0 and bs[i + 1] == 0 and bs[i + 2] == 1:
            starts.append((i - 1 if i > 0 and bs[i - 1] == 0 else i, i + 3))
            i += 3
        else:
            i += 1
    out = []
    for k, (sc, payload) in enumerate(starts):
        end = starts[k + 1][0] if k + 1 < len(starts) else n
        out.append((bs[sc:payload], bs[payload:end]))
    return out


def unescape(ebsp):
    """NAL payload -> RBSP (drops emulation_prevention_three_byte)"""
    out, zeros = bytearray(), 0
    for b in ebsp:
        if zeros >= 2 and b == 3:
            zeros = 0
            continue
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


def escape(rbsp):
    """RBSP -> NAL payload (inserts emulation_prevention_three_byte, also after trailing zero bytes)"""
    out, zeros = bytearray(), 0
    for b in rbsp:
        if zeros >= 2 and b <= 3:
            out.append(3)
            zeros = 0
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    if out and out[-1] == 0:
        out.append(3)
    return bytes(out)


# ---- bits ---------------------------------------------------------------------------------------------------------------

class Reader:
    def __init__(self, data):
        self.bits = "".join(format(b, "08b") for b in data)
        self.pos = 0

    def u(self, n):
        if self.pos + n > len(self.bits):
            raise ValueError("truncated")
        v = int(self.bits[self.pos:self.pos + n], 2) if n else 0
        self.pos += n
        return v

    def ue(self):
        z = 0
        while self.u(1) == 0:
            z += 1
            if z > 31:
                raise ValueError("bad exp-Golomb code")
        return (1 << z) - 1 + self.u(z)

    def se(self):
        k = self.ue()
        return (k + 1) // 2 if k & 1 else -(k // 2)


def ue_bits(v):
    s = format(v + 1, "b")
    return "0" * (len(s) - 1) + s


def se_bits(v):
    return ue_bits(2 * v - 1 if v > 0 else -2 * v)


def to_bytes(bits):
    assert len(bits) % 8 == 0
    return bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8))


# ---- parameter sets -----------------------------------------------------------------------------------------------------

def parse_sps(rbsp):
    r = Reader(rbsp)
    profile = r.u(8)
    r.u(16)                                                       # constraint flags, level_idc
    sps_id = r.ue()
    sps = {"profile": profile}
    if profile in (100, 110, 122, 244, 44, 83, 86, 118, 128, 138, 139, 134, 135):
        cf = r.ue()
        if cf == 3:
            r.u(1)
        r.ue(); r.ue(); r.u(1)                                    # bit depths, qpprime_y_zero_transform_bypass_flag
        if r.u(1):
            raise ValueError("scaling matrices are not rewritten")
    sps["log2_max_frame_num"] = r.ue() + 4
    sps["poc_type"] = r.ue()
    if sps["poc_type"] == 0:
        sps["log2_max_poc_lsb"] = r.ue() + 4
    elif sps["poc_type"] == 1:
        sps["delta_pic_order_always_zero"] = r.u(1)
        r.se(); r.se()
        for _ in range(r.ue()):
            r.se()
    r.ue(); r.u(1); r.ue(); r.ue()                                # max_num_ref_frames, gaps, width, height
    sps["frame_mbs_only"] = r.u(1)
    if not sps["frame_mbs_only"]:
        raise ValueError("field streams are not rewritten")
    return sps_id, sps


def parse_pps(rbsp):
    """-> (pps_id, fields, bit position of weighted_bipred_idc)"""
    r = Reader(rbsp)
    pps_id, sps_id = r.ue(), r.ue()
    p = {"sps_id": sps_id, "cabac": r.u(1), "bottom_field_poc": r.u(1)}
    if r.ue() != 0:
        raise ValueError("slice groups are not rewritten")
    p["n_ref_l0"], p["n_ref_l1"] = r.ue() + 1, r.ue() + 1
    p["weighted_pred"] = r.u(1)
    wbi_pos = r.pos
    p["weighted_bipred_idc"] = r.u(2)
    r.se(); r.se(); r.se()                                        # pic_init_qp, pic_init_qs, chroma_qp_index_offset
    p["deblocking_control"] = r.u(1)
    r.u(1)                                                        # constrained_intra_pred_flag
    p["redundant_pic_cnt"] = r.u(1)
    return pps_id, p, wbi_pos


# ---- pred_weight_table --------------------------------------------------------------------------------------------------

def neutral_table(n_ref):
    """denominators 5, every flag off: w = 32, o = 0 everywhere"""
    return {"ld": (5, 5), "lists": [[(None, None) for _ in range(n)] for n in n_ref]}


def _bound(ld):
    return 127 if ld == 7 else 128


def random_table(rng, n_ref):
    """seeded table for a B slice with n_ref = (entries of list 0, entries of list 1).  Entry = (luma, chroma): luma None (flag off) or
    (w, o); chroma None or ((w_cb, o_cb), (w_cr, o_cr))."""
    ld = (rng.randint(0, 7), rng.randint(0, 7))

    def value():
        t = rng.random()
        return -128 if t < 0.12 else 127 if t < 0.24 else rng.randint(-128, 127)

    def weight(lo, hi, ldp):
        """a weight in [lo, hi], or None (flag off) when the default 2^ld is in range and the draw says so"""
        if lo <= (1 << ldp) <= hi and rng.random() < 0.25:
            return None
        t = rng.random()
        if t < 0.15 and lo <= -128:
            return -128
        if t < 0.3 and hi >= 127:
            return 127
        if t < 0.6:                                               # near the neutral weight: moderate, mostly visible pictures
            c = 1 << ldp
            return max(lo, min(hi, c + rng.randint(-c // 2 - 1, c // 2 + 1)))
        return rng.randint(lo, hi)

    lists = [[], []]
    # plane 0 luma, 1 Cb, 2 Cr: weights of list 0 first, then list 1 within the pair bound against every list-0 weight
    w = [[[None] * 3 for _ in range(n_ref[l])] for l in range(2)]
    for pl in range(3):
        ldp = ld[0 if pl == 0 else 1]
        b = _bound(ldp)
        for i in range(n_ref[0]):
            w[0][i][pl] = weight(-128, 127, ldp)
        eff0 = [(1 << ldp) if w[0][i][pl] is None else w[0][i][pl] for i in range(n_ref[0])]
        lo, hi = max(-128, -128 - min(eff0)), min(127, b - max(eff0))
        for j in range(n_ref[1]):
            w[1][j][pl] = weight(lo, hi, ldp)
    for l in range(2):
        for i in range(n_ref[l]):
            ws = w[l][i]
            luma = None if ws[0] is None else (ws[0], value())
            if ws[1] is None and ws[2] is None:
                chroma = None
            else:                                                 # one flag for both chroma planes: a None one gets its default
                chroma = tuple(((1 << ld[1]) if ws[pl] is None else ws[pl], value()) for pl in (1, 2))
            lists[l].append((luma, chroma))
    return {"ld": ld, "lists": lists}


def table_bits(t):
    bits = ue_bits(t["ld"][0]) + ue_bits(t["ld"][1])
    for entries in t["lists"]:
        for luma, chroma in entries:
            bits += "0" if luma is None else "1" + se_bits(luma[0]) + se_bits(luma[1])
            bits += "0" if chroma is None else "1" + "".join(se_bits(w) + se_bits(o) for w, o in chroma)
    return bits


# ---- slices -------------------------------------------------------------------------------------------------------------

def _skip_list_modification(r):
    if r.u(1):
        while True:
            idc = r.ue()
            if idc == 3:
                break
            if idc > 5:
                raise ValueError("bad modification_of_pic_nums_idc")
            r.ue()


def _rewrite_b_slice(nal_hdr, rbsp, spss, ppss, make_table, cut):
    nal_type, ref_idc = nal_hdr & 31, (nal_hdr >> 5) & 3
    r = Reader(rbsp)
    r.ue()                                                        # first_mb_in_slice
    slice_type = r.ue() % 5
    pps = ppss[r.ue()]
    if slice_type != 1:
        return None
    sps = spss[pps["sps_id"]]
    r.u(sps["log2_max_frame_num"])
    if nal_type == 5:
        r.ue()
    if sps["poc_type"] == 0:
        r.u(sps["log2_max_poc_lsb"])
        if pps["bottom_field_poc"]:
            r.se()
    elif sps["poc_type"] == 1 and not sps["delta_pic_order_always_zero"]:
        r.se()
        if pps["bottom_field_poc"]:
            r.se()
    if pps["redundant_pic_cnt"]:
        r.ue()
    r.u(1)                                                        # direct_spatial_mv_pred_flag
    n_ref = [pps["n_ref_l0"], pps["n_ref_l1"]]
    if r.u(1):                                                    # num_ref_idx_active_override_flag
        n_ref = [r.ue() + 1, r.ue() + 1]
    _skip_list_modification(r)
    _skip_list_modification(r)
    insert_at = r.pos
    if pps["weighted_bipred_idc"] == 1:
        raise ValueError("the stream already carries explicit B weights")
    table = table_bits(make_table(n_ref))
    if cut:                                                       # a slice that ends inside its table
        body = r.bits[:insert_at] + table[:len(table) // 2] + "1"
        return to_bytes(body + "0" * (-len(body) % 8))
    if ref_idc:                                                   # dec_ref_pic_marking()
        if nal_type == 5:
            r.u(2)
        elif r.u(1):
            while True:
                op = r.ue()
                if op == 0:
                    break
                if op in (1, 3):
                    r.ue()
                if op == 2:
                    r.ue()
                if op in (3, 6):
                    r.ue()
                if op == 4:
                    r.ue()
    if pps["cabac"]:
        r.ue()                                                    # cabac_init_idc
    r.se()                                                        # slice_qp_delta
    if pps["deblocking_control"] and r.ue() != 1:
        r.se(); r.se()
    header_end = r.pos
    bits = r.bits
    if pps["cabac"]:
        data_start = (header_end + 7) // 8 * 8                    # after the old cabac_alignment_one_bits
        if bits[header_end:data_start] != "1" * (data_start - header_end):
            raise ValueError("cabac_alignment_one_bit")
        head = bits[:insert_at] + table + bits[insert_at:header_end]
        head += "1" * (-len(head) % 8)
        return to_bytes(head) + rbsp[data_start // 8:]
    stop = bits.rindex("1")                                       # rbsp_stop_one_bit
    body = bits[:insert_at] + table + bits[insert_at:stop] + "1"
    body += "0" * (-len(body) % 8)
    return to_bytes(body)


def rewrite(bs, seed=None, make_table=None, cut=False):
    """the stream `bs` with explicit weights in its B slices: tables from random_table(seed), or neutral ones for seed None, or from
    make_table(n_ref) when given; `cut`: every B slice ends halfway through its table (a truncated slice)"""
    rng = random.Random(seed)
    if make_table is None:
        make_table = neutral_table if seed is None else (lambda n_ref: random_table(rng, n_ref))
    spss, ppss, out = {}, {}, bytearray()
    for sc, nal in nal_units(bs):
        hdr, rbsp = nal[0], unescape(nal[1:])
        t = hdr & 31
        new = None
        if t == 7:
            sid, sps = parse_sps(rbsp)
            spss[sid] = sps
        elif t == 8:
            pid, pps, wbi_pos = parse_pps(rbsp)
            ppss[pid] = dict(pps)
            bits = Reader(rbsp).bits
            new = to_bytes(bits[:wbi_pos] + "01" + bits[wbi_pos + 2:])
        elif t in (1, 5):
            new = _rewrite_b_slice(hdr, rbsp, spss, ppss, make_table, cut)
        if new is None:
            out += sc + nal
        else:
            out += sc + bytes([hdr]) + escape(new)
    return bytes(out)
