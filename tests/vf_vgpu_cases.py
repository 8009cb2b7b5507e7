"""Inputs for the vGPU-on-VF tests (kxpu_vf_vgpu_types, kxpu_classify_vf_vgpu): side-record and walk builders, the hand
cases and hypothesis strategies, shared by the CPU and the GPU tests."""
import numpy as np
from hypothesis import strategies as st

import viab_cases as VC
from oracle import xpu_oracle as XO
from kxpu_b200.binding import VFVGPUREC_DTYPE, VGPUKEY_DTYPE

READ, CUR_ERR = 0x01, 0x02
NONE, NAMED, UNNAMED, BAD = 0, 1, 2, 3
HEADER = b"ID    : vGPU Name\n"
# two passthrough rules and one vGPU rule on the manager's driver (bit 2)
RULES = [(b"10de", b"vfio-pci"), (b"1002", b"vfio-pci"), (b"10de", b"nvidia")]
VGPU_BIT = 1 << 2


def vt(cur=None, flags=None):
    """One kxpu_vfvgpurec: cur = the bytes of current_vgpu_type (None: not read)."""
    r = np.zeros(1, VFVGPUREC_DTYPE)[0]
    if cur is None:
        r["flags"] = flags or 0
        return r
    r["cur_txt"][:min(len(cur), 16)] = np.frombuffer(cur[:16], np.uint8)
    r["cur_len"] = min(len(cur), 17)
    r["flags"] = READ if flags is None else flags
    return r


def vts(*rs):
    return np.array(list(rs), VFVGPUREC_DTYPE)


def key(k):
    """The 48-byte key row of key bytes k (b"": the all-zero row)."""
    row = np.zeros(1, VGPUKEY_DTYPE)[0]
    row["key"][:len(k)] = np.frombuffer(k, np.uint8)
    row["len"] = len(k)
    return row


# name -> (tables, [current_vgpu_type bytes or None], [(status, type_id, key)])
HAND = {
    "header_and_lines": ([HEADER + b"557  : NVIDIA H100-4C\n558 : NVIDIA H100-8C\n"], [b"557\n", b"558"],
                         [(NAMED, 557, b"NVIDIA_H100-4C"), (NAMED, 558, b"NVIDIA_H100-8C")]),
    "crlf_and_tabs": ([b"ID : Name\r\n\t557\t:\tGRID A\r\n 558 :B \t\r\n"], [b"557\n", b"558\n"],
                      [(NAMED, 557, b"GRID_A"), (NAMED, 558, b"B")]),
    "leading_zero_id_is_no_line": ([b"0557 : A\n"], [b"557"], [(UNNAMED, 557, b"")]),
    "id_zero_in_a_table": ([b"0 : Zero\n557 : A\n"], [b"0\n", b"557"], [(NONE, 0, b""), (NAMED, 557, b"A")]),
    "first_table_wins": ([b"557 : First\n", b"557 : Second\n557 : Third\n"], [b"557"], [(NAMED, 557, b"First")]),
    "first_line_wins": ([b"557 : One\n557 : Two"], [b"557"], [(NAMED, 557, b"One")]),
    "two_ids_one_key": ([b"557 : H100 4C\n558 : H100-4C?\n559 : H100_4C\n"], [b"557", b"559"],
                        [(NAMED, 557, b"H100_4C"), (NAMED, 559, b"H100_4C")]),
    "name_of_41_bytes": ([b"557 : " + b"A" * 41 + b"\n557 : short\n"], [b"557"], [(NAMED, 557, b"short")]),
    "name_of_40_bytes": ([b"557 : " + b"A" * 40], [b"557"], [(NAMED, 557, b"A" * 40)]),
    "name_sanitised_to_empty": ([b"557 : ###\n"], [b"557"], [(UNNAMED, 557, b"")]),
    "no_name": ([b"557 :\n557:   \n"], [b"557"], [(UNNAMED, 557, b"")]),
    "colon_in_name": ([b"557 : a:b\n"], [b"557"], [(NAMED, 557, b"ab")]),
    "largest_id": ([b"4294967295 : Max\n4294967296 : Over\n"], [b"4294967295"], [(NAMED, 4294967295, b"Max")]),
    "last_line_without_newline": ([b"557 : A\n558 : B"], [b"558"], [(NAMED, 558, b"B")]),
    "no_tables": ([], [b"557"], [(UNNAMED, 557, b"")]),
    "empty_tables": ([b"", b"", b"557 : A"], [b"557"], [(NAMED, 557, b"A")]),
    "table_without_final_newline_does_not_join": ([b"557 : A", b"\n558 : B\n"], [b"558", b"557"],
                                                 [(NAMED, 558, b"B"), (NAMED, 557, b"A")]),
}

# current_vgpu_type shapes: (bytes or None, flags or None) -> (status, type_id) with the table "557 : A"
CURRENT = [
    ((b"557", None), (NAMED, 557)), ((b"557\n", None), (NAMED, 557)), ((b"557\n\n", None), (BAD, 0)),
    ((b" 557", None), (BAD, 0)), ((b"0", None), (NONE, 0)), ((b"0\n", None), (NONE, 0)), ((b"00", None), (BAD, 0)),
    ((b"0557", None), (BAD, 0)), ((b"4294967295", None), (UNNAMED, 4294967295)), ((b"4294967296", None), (BAD, 0)),
    ((b"1" * 17, None), (BAD, 0)), ((b"1" * 16, None), (BAD, 0)), ((b"", None), (BAD, 0)), ((b"\n", None), (BAD, 0)),
    ((b"-1", None), (BAD, 0)), ((b"557", READ | CUR_ERR), (BAD, 0)), ((b"", READ | CUR_ERR), (BAD, 0)),
    ((None, None), (NONE, 0)), ((None, CUR_ERR), (NONE, 0)), ((b"557", 0), (NONE, 0)), ((b"12", None), (UNNAMED, 12)),
]


def cur_record(cur, flags):
    return vt(cur, flags)


_NAMES = st.sampled_from([b"NVIDIA H100-4C", b"NVIDIA H100-8C", b"H100_4C", b"GRID A", b" x ", b"###", b"A" * 40,
                          b"A" * 41, b"a:b", b"\tq\t", b"n\rm", b""])
_IDS = st.sampled_from([b"557", b"558", b"0", b"0557", b"4294967295", b"4294967296", b"12", b"x", b""])
_BL = st.sampled_from([b"", b" ", b"\t", b"  \t"])


@st.composite
def line(draw):
    if draw(st.integers(0, 5)) == 0:
        return draw(st.binary(max_size=12))
    return (draw(_BL) + draw(_IDS) + draw(_BL) + draw(st.sampled_from([b":", b":", b";", b""])) + draw(_BL) +
            draw(_NAMES) + draw(_BL) + draw(st.sampled_from([b"", b"\r", b"\r\r"])))


@st.composite
def table(draw):
    lines = draw(st.lists(line(), max_size=6))
    t = b"\n".join(lines)
    return t + b"\n" if lines and draw(st.booleans()) else t


@st.composite
def type_inputs(draw):
    tables = draw(st.lists(table(), max_size=5))
    curs = draw(st.lists(st.tuples(st.one_of(st.none(), st.sampled_from([b"557", b"558\n", b"0", b"12", b"4294967295",
                                                                            b"557\n\n", b" 12", b"1" * 17])),
                                   st.sampled_from([None, READ, READ | CUR_ERR, 0])), max_size=12))
    return tables, vts(*[vt(c, f) for c, f in curs])


def dev(bdf, group, driver=b"nvidia", vendor=b"0x10de\n", flags=0, numa=0, device=b"0x2330\n"):
    return VC.rec(bdf, group, driver=driver, vendor=vendor, device=device, flags=flags, numa=numa)


@st.composite
def classify_inputs(draw):
    """(recs, keys): records of the three rules (and others), some in shared groups, with keys from a small pool."""
    n = draw(st.integers(0, 24))
    recs, keys = [], []
    pool = [b"", b"A", b"B", b"NVIDIA_H100-4C", b"A" * 40]
    for i in range(n):
        driver, vendor = draw(st.sampled_from([(b"nvidia", b"0x10de\n"), (b"vfio-pci", b"0x10de\n"),
                                               (b"vfio-pci", b"0x1002\n"), (b"nvme", b"0x144d\n")]))
        flags = draw(st.sampled_from([0, 0, 0, VC.DEVICE_ERR, VC.DRIVER_ERR, VC.IS_DIR, VC.BLOCKS, VC.NUMA]))
        device = draw(st.sampled_from([b"0x2330\n", b"0x2331\n", b"0x74a1\n"]))
        recs.append(dev(b"0000:%02x:00.%d" % (i // 4, i % 4), draw(st.integers(1, 8)), driver=driver, vendor=vendor,
                        flags=flags, numa=draw(st.integers(0, 3)), device=device))
        keys.append(key(draw(st.sampled_from(pool))))
    return np.array(recs, XO.DEVREC_DTYPE), np.array(keys, VGPUKEY_DTYPE)
