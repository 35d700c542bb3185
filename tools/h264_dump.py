"""Minimal Annex-B inspector (NAL list, SPS/PPS/slice-header fields) used while debugging bit-exactness."""
import sys


class BR:
    def __init__(self, data):
        self.d, self.p = data, 0

    def u(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | ((self.d[self.p >> 3] >> (7 - (self.p & 7))) & 1)
            self.p += 1
        return v

    def ue(self):
        z = 0
        while self.u(1) == 0:
            z += 1
        return (1 << z) - 1 + (self.u(z) if z else 0)

    def se(self):
        k = self.ue()
        return (k + 1) // 2 if k & 1 else -(k // 2)


def split_nals(bs):
    i, n, out = 0, len(bs), []
    starts = []
    while i + 3 <= n:
        if bs[i] == 0 and bs[i + 1] == 0 and bs[i + 2] == 1:
            starts.append((i - 1 if i > 0 and bs[i - 1] == 0 else i, i + 3))
            i += 3
        else:
            i += 1
    for k, (s, p) in enumerate(starts):
        e = starts[k + 1][0] if k + 1 < len(starts) else n
        out.append((s, bs[p:e]))
    return out


def unescape(nal):
    out, z = bytearray(), 0
    for b in nal:
        if z >= 2 and b == 3:
            z = 0
            continue
        out.append(b)
        z = z + 1 if b == 0 else 0
    return bytes(out)


def dump(bs, verbose=True):
    sps = {}
    res = []
    for off, nal in split_nals(bs):
        hdr = nal[0]
        t, ref = hdr & 31, (hdr >> 5) & 3
        r = BR(unescape(nal[1:]) + b"\0\0\0\0")
        info = {"off": off, "type": t, "ref_idc": ref, "size": len(nal)}
        if t == 7:
            info["profile"] = r.u(8); info["constraints"] = r.u(8); info["level"] = r.u(8); info["sps_id"] = r.ue()
            if info["profile"] in (100, 110, 122, 244, 44, 83, 86, 118, 128):
                info["chroma_format"] = r.ue(); info["bit_depth"] = (r.ue() + 8, r.ue() + 8); info["bypass"] = r.u(1)
                info["scaling_matrix"] = r.u(1)
                if info["scaling_matrix"]:
                    for k in range(8):
                        if r.u(1):
                            last = nxt = 8
                            for _ in range(16 if k < 6 else 64):
                                if nxt: nxt = (last + r.se() + 256) % 256
                                last = nxt if nxt else last
            info["log2_max_frame_num"] = r.ue() + 4; info["poc_type"] = r.ue()
            if info["poc_type"] == 0: info["log2_max_poc_lsb"] = r.ue() + 4
            info["num_ref"] = r.ue(); info["gaps"] = r.u(1); info["mbw"] = r.ue() + 1; info["mbh"] = r.ue() + 1
            info["frame_mbs_only"] = r.u(1); info["d8x8"] = r.u(1); info["crop"] = r.u(1)
            if info["crop"]: info["crop_lrtb"] = [r.ue() for _ in range(4)]
            info["vui"] = r.u(1)
            sps = info
        elif t == 8:
            info["pps_id"] = r.ue(); info["sps_id"] = r.ue(); info["cabac"] = r.u(1); info["pic_order_present"] = r.u(1)
            info["slice_groups"] = r.ue() + 1; info["nref0"] = r.ue() + 1; info["nref1"] = r.ue() + 1
            info["wp"] = r.u(1); info["wbi"] = r.u(2); info["init_qp"] = r.se() + 26; info["init_qs"] = r.se() + 26
            info["cqp_off"] = r.se(); info["dbf_ctrl"] = r.u(1); info["cip"] = r.u(1); info["red"] = r.u(1)
            if r.p + 8 < 8 * (len(nal) - 1):
                info["t8x8"] = r.u(1); info["pps_scaling"] = r.u(1)
            pps = info
        elif t in (1, 5):
            info["first_mb"] = r.ue(); info["slice_type"] = r.ue(); info["pps_id"] = r.ue()
            info["frame_num"] = r.u(sps.get("log2_max_frame_num", 15))
            if t == 5: info["idr_pic_id"] = r.ue()
            if sps.get("poc_type", 2) == 0: info["poc_lsb"] = r.u(sps["log2_max_poc_lsb"])
            if info["slice_type"] % 5 == 1:
                info["direct_spatial"] = r.u(1)
            if info["slice_type"] % 5 in (0, 1):
                info["num_ref_override"] = r.u(1)
                if info["num_ref_override"]: info["nref"] = r.ue() + 1
                info["reorder"] = r.u(1)
                if info["reorder"]:
                    cmds = []
                    while True:
                        idc = r.ue()
                        if idc == 3: break
                        cmds.append((idc, r.ue()))
                    info["reorder_cmds"] = cmds
            if ref:
                if t == 5: info["no_out_prior"] = r.u(1); info["long_term"] = r.u(1)
                else:
                    info["adaptive_marking"] = r.u(1)
                    if info["adaptive_marking"]:
                        ops = []
                        while True:
                            op = r.ue()
                            if op == 0: break
                            ops.append((op, r.ue(), r.ue()) if op == 3 else (op, r.ue()))
                        info["mmco"] = ops
            info["qp_delta"] = r.se()
            info["dbf_idc"] = r.ue()
            if info["dbf_idc"] != 1: info["alpha"] = r.se(); info["beta"] = r.se()
            info["hdr_bits"] = r.p
        res.append(info)
        if verbose:
            print(info)
    return res


if __name__ == "__main__":
    dump(open(sys.argv[1], "rb").read())
