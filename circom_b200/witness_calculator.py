"""Host-side mirror of the reference's witness-calculator interface, over the C ABI.

Same surface as code_producers/src/wasm_elements/common/witness_calculator.js
(`builder(code, options)` -> `WitnessCalculator` with `calculateWitness`,
`calculateBinWitness`, `calculateWTNSBin`, :1,108,176,194,212) and the same input handling as
the C++ runtime (`qualify_input`, FNV-1a name hashes, size checks:
c_elements/common/main.cpp:190-286, calcwit.cpp:17-24,77-102) - plus batch variants, which
are the point of the GPU back end: one call computes the witnesses of many inputs.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, Iterable, List, Optional, Sequence, Union

import numpy as np

from . import native
from .circuit import CircuitDesc
from .native import CwError, CwStats, check, lib


def fnv_hash(s: str) -> int:
    """fnvHash (witness_calculator.js:369-383) / fnv1a (calcwit.cpp:17-24)."""
    h = 0xCBF29CE484222325
    for ch in s:
        h ^= ord(ch)
        h = (h * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h


def _flat(a) -> list:
    out = []

    def rec(x):
        if isinstance(x, (list, tuple, np.ndarray)):
            for y in x:
                rec(y)
        else:
            out.append(x)
    rec(a)
    return out


def qualify_input(prefix: str, inp, out: Dict[str, object]) -> None:
    """witness_calculator.js:292-321 / main.cpp:221-241: nested objects and arrays of objects
    (buses) become qualified names `a.b[i].c`."""
    if isinstance(inp, (list, tuple)):
        a = _flat(inp)
        if a:
            kinds = {isinstance(x, dict) for x in a}
            if len(kinds) > 1:
                raise ValueError("Types are not the same in the key %s" % prefix)
            if isinstance(a[0], dict):
                _qualify_list(prefix, inp, out)
            else:
                out[prefix] = inp
        else:
            out[prefix] = inp
    elif isinstance(inp, dict):
        for k, v in inp.items():
            qualify_input(k if prefix == "" else prefix + "." + k, v, out)
    else:
        out[prefix] = inp


def _qualify_list(prefix: str, inp, out) -> None:
    if isinstance(inp, (list, tuple)):
        for i, x in enumerate(inp):
            _qualify_list("%s[%d]" % (prefix, i), x, out)
    else:
        qualify_input(prefix, inp, out)


def parse_value(v, q: int) -> int:
    """json2FrElements (main.cpp:144-188): decimal / 0x / 0b / 0o strings, or integers; reduced mod q
    with a non-negative result (normalize, witness_calculator.js:363-367)."""
    if isinstance(v, str):
        s = v.strip()
        p = s[:2].lower()
        if p == "0x":
            n = int(s[2:], 16)
        elif p == "0b":
            n = int(s[2:], 2)
        elif p == "0o":
            n = int(s[2:], 8)
        else:
            if not s.isdigit():
                raise ValueError("Invalid number in JSON input: %s" % v)
            n = int(s, 10)
    elif isinstance(v, (bool, np.bool_)):
        n = int(v)
    elif isinstance(v, (int, np.integer)):
        n = int(v)
    else:
        raise ValueError("Invalid JSON type")
    return n % q


def ints_to_limbs(vals: Sequence[int]) -> np.ndarray:
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    m = 0xFFFFFFFFFFFFFFFF
    for i, v in enumerate(vals):
        out[i, 0] = v & m
        out[i, 1] = (v >> 64) & m
        out[i, 2] = (v >> 128) & m
        out[i, 3] = (v >> 192) & m
    return out


def limbs_to_ints(a: np.ndarray) -> List[int]:
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 4)
    return [int.from_bytes(row.tobytes(), "little") for row in a]


def aligned_empty(shape, dtype=np.uint64, align: int = 64, hugepages: Optional[bool] = None) -> np.ndarray:
    """numpy array whose data starts on an `align`-byte boundary: witness rows written into a 64-byte aligned buffer
    take full-cache-line streaming stores in the host-side expansion (numpy's own allocations are 16-byte aligned).
    hugepages (or CW_HUGEPAGES=1): align to 2 MB and advise the kernel to back the buffer with huge pages before its first
    touch.  Measured on the bench (24 GB row buffers, 16 expansion threads): 6.68 / 6.70 k witnesses/s with, 6.94 / 6.47 k
    without - no effect, the streaming stores are bandwidth-bound, so it stays opt-in."""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    if hugepages is None:
        hugepages = n >= (64 << 20) and os.environ.get("CW_HUGEPAGES", "0") == "1"
    if hugepages:
        align = max(align, 2 << 20)
    raw = np.empty(n + align, dtype=np.uint8)
    off = (-raw.ctypes.data) % align
    if hugepages:
        try:
            libc = ctypes.CDLL(None, use_errno=True)
            libc.madvise.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
            libc.madvise(ctypes.c_void_p(raw.ctypes.data + off), ctypes.c_size_t(n & ~((2 << 20) - 1)), 14)   # MADV_HUGEPAGE
        except (OSError, AttributeError):
            pass      # advice only
    return raw[off:off + n].view(dtype).reshape(shape)


class Circuit:
    """A lowered circuit (replaces Circom_Circuit + the compiled <name>.cpp)."""

    def __init__(self, src: Union[CircuitDesc, bytes, str], sanity_check: bool = True, host_only: bool = False,
                 o0: bool = False, flags: int = 0, compact: Optional[bool] = None, fuse: bool = False,
                 symbols: bool = False):
        """compact (default on; environment CW_COMPACT=0 turns it off): lower for the compact value store - bit runs in
        a per-instance bit plane, temporaries sharing slots (CW_FLAG_COMPACT) - instead of one 32-byte slot per value"""
        if compact is None:
            compact = os.environ.get("CW_COMPACT", "1") != "0" and not (flags & native.CW_FLAG_COMPACT)
        flags |= int(os.environ.get("CW_FLAGS_EXTRA", "0"))   # (experiments)
        if fuse:   # single-use values stay in registers of their reader's work item: pays for large batches only
            flags |= native.CW_FLAG_FUSE
        flags |= (0 if sanity_check else native.CW_FLAG_NO_ASSERTS) | (native.CW_FLAG_HOST_ONLY if host_only else 0) | \
            (native.CW_FLAG_O0 if o0 else 0) | (native.CW_FLAG_COMPACT if compact else 0)
        self.flags = flags
        self._h = ctypes.c_void_p()
        if isinstance(src, CircuitDesc):
            src = src.to_bytes(symbols=symbols)   # (symbols: signal / component names for write_sym)
        if isinstance(src, (bytes, bytearray)):
            buf = bytes(src)
            check(lib.cw_circuit_load_mem(buf, len(buf), flags, ctypes.byref(self._h)))
        else:
            check(lib.cw_circuit_load(str(src).encode(), flags, ctypes.byref(self._h)))
        self._init_from_handle()

    @classmethod
    def from_handle(cls, handle: ctypes.c_void_p, flags: int = 0) -> "Circuit":
        """wrap a cw_circuit* produced by the library (cw_circuit_deserialize / cw_circuit_broadcast); takes ownership"""
        c = cls.__new__(cls)
        c._h = handle
        c.flags = flags
        c._init_from_handle()
        return c

    @classmethod
    def deserialize(cls, blob: bytes) -> "Circuit":
        h = ctypes.c_void_p()
        check(lib.cw_circuit_deserialize(blob, len(blob), ctypes.byref(h)))
        return cls.from_handle(h)

    def serialize(self) -> bytes:
        """the LOWERED circuit as one blob (what rank 0 broadcasts; other ranks skip the lowering)"""
        n = ctypes.c_size_t()
        check(lib.cw_circuit_serialize(self._h, None, 0, ctypes.byref(n)))
        buf = (ctypes.c_uint8 * n.value)()
        check(lib.cw_circuit_serialize(self._h, buf, n.value, ctypes.byref(n)))
        return bytes(buf)

    def _init_from_handle(self):
        st = CwStats()
        check(lib.cw_circuit_stats(self._h, ctypes.byref(st)))
        self.stats = st.as_dict()
        pid = ctypes.c_int()
        q = (ctypes.c_uint64 * 4)()
        check(lib.cw_circuit_prime(self._h, ctypes.byref(pid), q))
        self.prime_id = pid.value
        self.prime = sum(int(q[i]) << (64 * i) for i in range(4))
        self.n_witness = self.stats["n_witness"]
        self.n_inputs = self.stats["n_inputs"]
        self.n_outputs = self.stats["n_outputs"]

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_circuit_destroy(h)

    def input_signal_size(self, name: str) -> int:
        size = ctypes.c_uint64()
        rc = lib.cw_get_input_signal_size(self._h, fnv_hash(name), ctypes.byref(size))
        if rc == native.CW_ENOTFOUND:
            return -1
        check(rc)
        return size.value

    def input_signal_id(self, name: str) -> int:
        sid = ctypes.c_uint64()
        check(lib.cw_get_input_signal_id(self._h, fnv_hash(name), ctypes.byref(sid)))
        return sid.value

    def tape(self):
        """(ops[n,4], level_start, witness_slot) copies of the lowered tape."""
        ops = np.zeros((self.stats["n_tape_ops"], 4), dtype=np.uint32)
        ls = np.zeros(self.stats["n_levels"] + 1, dtype=np.uint32)
        ws = np.zeros(self.n_witness, dtype=np.uint32)
        check(lib.cw_circuit_tape(self._h, ops.ctypes.data, ls.ctypes.data, ws.ctypes.data))
        return ops, ls, ws

    def tape_items(self) -> np.ndarray:
        """n_items+1 offsets: work item k = tape words [items[k], items[k+1]); level_start indexes work items"""
        it = np.zeros(self.stats["n_items"] + 1, dtype=np.uint32)
        check(lib.cw_circuit_tape_items(self._h, it.ctypes.data))
        return it

    def witness2signal(self) -> np.ndarray:
        out = np.zeros(self.n_witness, dtype=np.uint64)
        check(lib.cw_circuit_witness2signal(self._h, out.ctypes.data))
        return out

    def pack_info(self, entries: bool = True):
        """layout of the packed device->host records: ([words, plane words, extra-bit words, u64 entries, full
        entries], per witness entry (class << 30) | index)"""
        info = (ctypes.c_uint64 * 5)()
        ent = np.zeros(self.n_witness, dtype=np.uint32) if entries else None
        check(lib.cw_circuit_pack_info(self._h, info, ent.ctypes.data if entries else None))
        return [int(x) for x in info], ent

    def write_dat(self, path: str) -> None:
        check(lib.cw_circuit_write_dat(self._h, path.encode()))

    def functions(self) -> List[dict]:
        """the lowered functions: instructions and registers of a call frame (after the lowering's register allocation)"""
        n = ctypes.c_uint32()
        check(lib.cw_circuit_functions(self._h, ctypes.byref(n), None))
        info = (ctypes.c_uint32 * (4 * max(1, n.value)))()
        check(lib.cw_circuit_functions(self._h, ctypes.byref(n), info))
        return [{"n_instr": int(info[4 * i + 1]), "n_regs": int(info[4 * i + 2]), "n_params": int(info[4 * i + 3])}
                for i in range(n.value)]

    def format_log(self, witness) -> str:
        """what the circuit's log() calls print for one witness ([n_witness][4] uint64), as the reference calculator prints it"""
        w = np.ascontiguousarray(witness, dtype=np.uint64)
        assert w.size == self.n_witness * 4
        n = ctypes.c_size_t()
        check(lib.cw_circuit_format_log(self._h, w.ctypes.data, None, 0, ctypes.byref(n)))
        buf = ctypes.create_string_buffer(n.value + 1)
        check(lib.cw_circuit_format_log(self._h, w.ctypes.data, buf, n.value + 1, ctypes.byref(n)))
        return buf.value.decode()

    def assert_info(self, assert_no: int) -> str:
        """the reference's message for failed assert number `assert_no` (Batch.status() - 1): template name and, with the
        symbols section, the trace of components (c_code_generator.rs:461-468)"""
        n = ctypes.c_size_t()
        check(lib.cw_circuit_assert_info(self._h, assert_no, None, 0, ctypes.byref(n)))
        buf = ctypes.create_string_buffer(n.value + 1)
        check(lib.cw_circuit_assert_info(self._h, assert_no, buf, n.value + 1, ctypes.byref(n)))
        return buf.value.decode()

    def write_sym(self, path: str) -> None:
        """the compiler's `.sym` (`signal id,witness index or -1,node id,main.path.name` per signal); the description must
        carry the symbols section (Circuit(desc, symbols=True) / a producer that writes it)"""
        check(lib.cw_circuit_write_sym(self._h, path.encode()))

    def flatten_inputs(self, inp: dict) -> List[int]:
        """One instance's inputs in main-input signal order, with the reference's checks."""
        q = {}
        qualify_input("", inp, q)
        base = lib.cw_get_main_input_signal_start(self._h)
        vals: List[Optional[int]] = [None] * self.n_inputs
        count = 0
        for k, v in q.items():
            size = self.input_signal_size(k)
            if size < 0:
                raise ValueError("Signal %s not found\n" % k)
            arr = _flat(v)
            if len(arr) < size:
                raise ValueError("Not enough values for input signal %s\n" % k)
            if len(arr) > size:
                raise ValueError("Too many values for input signal %s\n" % k)
            sid = self.input_signal_id(k)
            if sid < base or sid - base + size > self.n_inputs:
                raise ValueError("Signal %s lies outside the main inputs\n" % k)
            for i, x in enumerate(arr):
                if vals[sid - base + i] is not None:
                    raise ValueError("Signal assigned twice: %d" % (sid + i))
                vals[sid - base + i] = parse_value(x, self.prime)
                count += 1
        if count < self.n_inputs:
            raise ValueError("Not all inputs have been set. Only %d out of %d" % (count, self.n_inputs))
        return vals  # type: ignore


class Batch:
    """Circom_CalcWit for `batch` independent inputs on one GPU."""

    def __init__(self, circuit: Circuit, batch: int, device: int = 0):
        self.circuit = circuit
        self.batch = batch
        self._h = ctypes.c_void_p()
        check(lib.cw_batch_create(circuit._h, batch, device, ctypes.byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_batch_destroy(h)

    def set_input(self, instance: int, name: str, idx: int, value: int) -> None:
        limbs = (ctypes.c_uint64 * 4)(*[(value >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)])
        check(lib.cw_batch_set_input(self._h, instance, fnv_hash(name), idx, limbs))

    def remaining_inputs(self, instance: int) -> int:
        r = ctypes.c_uint32()
        check(lib.cw_batch_remaining_inputs(self._h, instance, ctypes.byref(r)))
        return r.value

    def set_inputs(self, arr, device_ptr: Optional[int] = None) -> None:
        """arr: uint64 [batch][n_inputs][4] canonical (numpy, host) - or a raw device pointer."""
        if device_ptr is not None:
            check(lib.cw_batch_set_inputs(self._h, ctypes.c_void_p(device_ptr), 1))
            return
        a = np.ascontiguousarray(arr, dtype=np.uint64)
        assert a.size == self.batch * self.circuit.n_inputs * 4, "bad input array shape"
        self._keep = a
        check(lib.cw_batch_set_inputs(self._h, a.ctypes.data, 0))

    def run(self, sync: bool = True) -> None:
        check(lib.cw_batch_run(self._h))
        if sync:
            check(lib.cw_batch_sync(self._h))

    def sync(self) -> None:
        check(lib.cw_batch_sync(self._h))

    def status(self) -> np.ndarray:
        st = np.zeros(self.batch, dtype=np.int32)
        check(lib.cw_batch_status(self._h, st.ctypes.data))
        return st

    def witness(self, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = aligned_empty((self.batch, self.circuit.n_witness, 4))
        check(lib.cw_batch_get_witness(self._h, out.ctypes.data))
        return out

    def witness_async(self, out: np.ndarray) -> None:
        """start the transfer on a helper thread (other batches may run meanwhile); finish with witness_wait()"""
        self._async_out = out
        check(lib.cw_batch_get_witness_async(self._h, out.ctypes.data))

    def witness_wait(self) -> None:
        check(lib.cw_batch_get_witness_wait(self._h))

    def witness_packed(self) -> np.ndarray:
        """uint32 [batch][words]: the packed records (see Circuit.pack_info)"""
        info, _ = self.circuit.pack_info(entries=False)
        out = np.empty((self.batch, info[0]), dtype=np.uint32)
        check(lib.cw_batch_get_witness_packed(self._h, out.ctypes.data))
        return out

    def layout(self):
        """(log2 instances per tile, threads per CTA, bytes of value store per instance)"""
        bt, th, by = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint64()
        check(lib.cw_batch_layout(self._h, ctypes.byref(bt), ctypes.byref(th), ctypes.byref(by)))
        return bt.value, th.value, by.value

    def tape_build(self):
        """the interpreter build run() launches: (prime or -1, calls, bit plane, compile-time log2 tile size or -1, fused)"""
        k = (ctypes.c_int32 * 5)()
        check(lib.cw_batch_tape_build(self._h, k))
        return k[0], bool(k[1]), bool(k[2]), k[3], bool(k[4])

    def expand_witness(self, first: int, count: int, device_ptr: int) -> None:
        check(lib.cw_batch_expand_witness(self._h, first, count, ctypes.c_void_p(device_ptr)))

    def last_d2h_bytes(self) -> int:
        return int(lib.cw_batch_last_d2h_bytes(self._h))

    def witness_device_ptr(self) -> int:
        p = ctypes.c_void_p()
        check(lib.cw_batch_witness_device(self._h, ctypes.byref(p)))
        return p.value

    def witness_strided(self):
        """(device pointer, stride in 32-byte elements): the witness rows where the tape wrote them"""
        p, st = ctypes.c_void_p(), ctypes.c_uint64()
        check(lib.cw_batch_witness_strided(self._h, ctypes.byref(p), ctypes.byref(st)))
        return p.value, st.value

    def stream(self) -> int:
        return lib.cw_batch_stream(self._h) or 0

    def last_ms(self):
        a, b = ctypes.c_float(), ctypes.c_float()
        check(lib.cw_batch_last_ms(self._h, ctypes.byref(a), ctypes.byref(b)))
        return a.value, b.value

    def wtns_bytes(self, instance: int) -> bytes:
        n = ctypes.c_size_t()
        check(lib.cw_batch_wtns_bytes(self._h, instance, None, 0, ctypes.byref(n)))
        buf = (ctypes.c_uint8 * n.value)()
        check(lib.cw_batch_wtns_bytes(self._h, instance, buf, n.value, ctypes.byref(n)))
        return bytes(buf)

    def log(self, instance: int) -> str:
        """what the circuit's log() calls print for this instance (cw_batch_log)"""
        n = ctypes.c_size_t()
        check(lib.cw_batch_log(self._h, instance, None, 0, ctypes.byref(n)))
        buf = ctypes.create_string_buffer(n.value + 1)
        check(lib.cw_batch_log(self._h, instance, buf, n.value + 1, ctypes.byref(n)))
        return buf.value.decode()

    def write_wtns(self, instance: int, path: str) -> None:
        check(lib.cw_batch_write_wtns(self._h, instance, path.encode()))


class R1cs:
    def __init__(self, src: Union[Circuit, str]):
        self._h = ctypes.c_void_p()
        if isinstance(src, Circuit):
            check(lib.cw_r1cs_from_circuit(src._h, ctypes.byref(self._h)))
        else:
            check(lib.cw_r1cs_load(str(src).encode(), ctypes.byref(self._h)))
        nw, nc, nnz, pid = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_int()
        check(lib.cw_r1cs_info(self._h, ctypes.byref(nw), ctypes.byref(nc), ctypes.byref(nnz), ctypes.byref(pid)))
        self.n_wires, self.n_constraints, self.nnz, self.prime_id = nw.value, nc.value, nnz.value, pid.value

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_r1cs_destroy(h)

    def check_batch(self, b: "Batch", device: int = 0):
        """check the witnesses of a Batch where the tape left them (no copy, any layout)"""
        ms = ctypes.c_float()
        fb = np.zeros(b.batch, dtype=np.int64)
        check(lib.cw_r1cs_check_batch(self._h, b._h, fb.ctypes.data, ctypes.byref(ms)))
        return fb, ms.value

    def compiled_info(self, b: Optional["Batch"] = None, device: int = 0) -> dict:
        """rows by the kernel that decides them, for the value layout of batch b (None: dense witness rows)"""
        info = (ctypes.c_uint64 * 4)()
        check(lib.cw_r1cs_compiled_info(self._h, b._h if b is not None else None, device, info))
        return {"general_rows": info[0], "integer_rows": info[1], "boolean_rows": info[2], "terms": info[3]}

    def eval_batch(self, b: "Batch", first: int, count: int, a_ptr: int, b_ptr: int, c_ptr: int) -> None:
        """A.w, B.w, C.w of instances [first, first+count) into device arrays [count][n_constraints][4] uint64"""
        check(lib.cw_r1cs_eval_batch(self._h, b._h, first, count, ctypes.c_void_p(a_ptr), ctypes.c_void_p(b_ptr),
                                     ctypes.c_void_p(c_ptr)))

    def qap_info(self):
        """(log2 n, nPublic): the Groth16 evaluation domain of this constraint system (include/circom_b200.h)"""
        k, npub = ctypes.c_uint32(), ctypes.c_uint32()
        check(lib.cw_r1cs_qap_info(self._h, ctypes.byref(k), ctypes.byref(npub)))
        return k.value, npub.value

    def quotient_batch(self, b: "Batch", first: int, count: int, h_ptr: int, scratch_ptr: int) -> None:
        """h = a'b' - c' of instances [first, first+count) into device array [count][n][4] uint64; scratch: 2*count*n*32
        bytes of device memory.  Asynchronous on the batch stream (b.sync())."""
        check(lib.cw_r1cs_quotient_batch(self._h, b._h, first, count, ctypes.c_void_p(h_ptr), ctypes.c_void_p(scratch_ptr)))

    def quotient(self, device_ptr: int, count: int, stride: Optional[int], h_ptr: int, scratch_ptr: int,
                 device: int = 0) -> None:
        """the same for `count` dense witness rows on the device, `stride` 32-byte elements apart (None: n_wires)"""
        check(lib.cw_r1cs_quotient_strided(self._h, ctypes.c_void_p(device_ptr), stride or self.n_wires, count, device,
                                           ctypes.c_void_p(h_ptr), ctypes.c_void_p(scratch_ptr)))

    def write(self, path: str, n_pub_out: Optional[int] = None, n_pub_in: Optional[int] = None,
              n_prv_in: Optional[int] = None) -> None:
        """None keeps the count the circuit / the loaded file carries (the header feeds snarkjs' public-signal count)"""
        keep = 0xFFFFFFFF
        check(lib.cw_r1cs_write(self._h, path.encode(), keep if n_pub_out is None else n_pub_out,
                                keep if n_pub_in is None else n_pub_in, keep if n_prv_in is None else n_prv_in))

    def check(self, witness, batch: Optional[int] = None, device: int = 0, device_ptr: Optional[int] = None,
              stride: Optional[int] = None):
        """A.w o B.w == C.w for each instance.  Returns (first_bad[batch] int64, -1 = satisfied; kernel ms).
        `stride` (32-byte elements between witness rows) lets the check read a Batch's slot store in place."""
        ms = ctypes.c_float()
        if device_ptr is not None:
            assert batch is not None
            fb = np.zeros(batch, dtype=np.int64)
            check(lib.cw_r1cs_check_strided(self._h, ctypes.c_void_p(device_ptr), stride or self.n_wires, 1, batch, device,
                                            fb.ctypes.data, ctypes.byref(ms)))
            return fb, ms.value
        w = np.ascontiguousarray(witness, dtype=np.uint64)
        batch = w.size // (self.n_wires * 4)
        fb = np.zeros(batch, dtype=np.int64)
        check(lib.cw_r1cs_check(self._h, w.ctypes.data, 0, batch, device, fb.ctypes.data, ctypes.byref(ms)))
        return fb, ms.value


def ntt_batch(prime_id: int, log2_n: int, count: int, data_ptr: int, mode: int, device: int = 0) -> None:
    """in-place transforms of `count` device vectors [count][2^log2_n][4] uint64 (mode: CW_NTT_FORWARD / INVERSE / COSET)"""
    check(lib.cw_fr_ntt_batch(prime_id, log2_n, count, ctypes.c_void_p(data_ptr), mode, device))


class G1Bases:
    """BN254 G1 points on the device for multi-scalar multiplications (cw_g1_bases_*, include/circom_b200.h).
    points: numpy uint64 [n][2][4] canonical affine, or a list of (x, y) ints; (0, 0) or None is the point at infinity."""

    def __init__(self, points, device: int = 0, prime_id: int = 0):   # (the scalar field: bn128 is the only one)
        if isinstance(points, np.ndarray):
            arr = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 2, 4)
        else:
            arr = np.zeros((len(points), 2, 4), dtype=np.uint64)
            for i, p in enumerate(points):
                for j, v in enumerate((0, 0) if p is None else p):
                    arr[i, j] = [(v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)]
        self.n = arr.shape[0]
        self.device = device
        self._h = ctypes.c_void_p()
        check(lib.cw_g1_bases_create(prime_id, arr.ctypes.data, self.n, device, ctypes.byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_g1_bases_destroy(h)

    def scratch_bytes(self, count: int) -> int:
        b = ctypes.c_uint64()
        check(lib.cw_g1_msm_scratch_bytes(self._h, count, ctypes.byref(b)))
        return b.value

    def msm(self, scalars_ptr: int, stride: int, count: int, out_ptr: int, scratch_ptr: int, stream=None) -> None:
        """out[c] = sum_i s_{c,i} P_i into device [count][2][4] uint64; scalars: device [count][stride][4] uint64.
        Asynchronous on `stream` (a Batch.stream() value; None = the legacy default stream)."""
        check(lib.cw_g1_msm_batch(self._h, ctypes.c_void_p(scalars_ptr), stride, count, ctypes.c_void_p(out_ptr),
                                  ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream or None)))

    def msm_host(self, scalars) -> List[Optional[tuple]]:
        """the MSMs of host scalars ([count][n] ints, or numpy uint64 [count][n][4]): [(x, y) or None per vector]"""
        import torch
        if isinstance(scalars, np.ndarray):
            arr = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.n, 4)
        else:
            arr = np.array([[[(s >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)] for s in row] for row in scalars],
                           dtype=np.uint64).reshape(-1, self.n, 4)
        count = arr.shape[0]
        dev = torch.device("cuda", self.device)
        s = torch.from_numpy(arr.view(np.int64)).to(dev)
        out = torch.zeros((count, 2, 4), dtype=torch.int64, device=dev)
        scratch = torch.empty(self.scratch_bytes(count), dtype=torch.uint8, device=dev)
        self.msm(s.data_ptr(), self.n, count, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize(dev)
        v = limbs_to_ints(out.cpu().numpy().view(np.uint64))
        return [None if (x, y) == (0, 0) else (x, y) for x, y in zip(v[0::2], v[1::2])]


class G2Bases:
    """BN254 G2 points (on the twist over Fq2) on the device for multi-scalar multiplications (cw_g2_bases_*,
    include/circom_b200.h).  points: numpy uint64 [n][2][2][4] canonical affine (x.c0, x.c1, y.c0, y.c1), or a list of
    ((x0, x1), (y0, y1)) ints; all zeros or None is the point at infinity.  Points are checked to lie on the twist, not
    to lie in the order-r subgroup."""

    def __init__(self, points, device: int = 0, prime_id: int = 0):   # (the scalar field: bn128 is the only one)
        if isinstance(points, np.ndarray):
            arr = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 2, 2, 4)
        else:
            arr = np.zeros((len(points), 2, 2, 4), dtype=np.uint64)
            for i, p in enumerate(points):
                for j, e in enumerate(((0, 0), (0, 0)) if p is None else p):
                    for k, v in enumerate(e):
                        arr[i, j, k] = [(v >> (64 * m)) & 0xFFFFFFFFFFFFFFFF for m in range(4)]
        self.n = arr.shape[0]
        self.device = device
        self._h = ctypes.c_void_p()
        check(lib.cw_g2_bases_create(prime_id, arr.ctypes.data, self.n, device, ctypes.byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_g2_bases_destroy(h)

    def scratch_bytes(self, count: int) -> int:
        b = ctypes.c_uint64()
        check(lib.cw_g2_msm_scratch_bytes(self._h, count, ctypes.byref(b)))
        return b.value

    def msm(self, scalars_ptr: int, stride: int, count: int, out_ptr: int, scratch_ptr: int, stream=None) -> None:
        """out[c] = sum_i s_{c,i} Q_i into device [count][2][2][4] uint64; scalars: device [count][stride][4] uint64.
        Asynchronous on `stream` (a Batch.stream() value; None = the legacy default stream)."""
        check(lib.cw_g2_msm_batch(self._h, ctypes.c_void_p(scalars_ptr), stride, count, ctypes.c_void_p(out_ptr),
                                  ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream or None)))

    def msm_host(self, scalars) -> List[Optional[tuple]]:
        """the MSMs of host scalars ([count][n] ints, or numpy uint64 [count][n][4]): [((x0, x1), (y0, y1)) or None]"""
        import torch
        if isinstance(scalars, np.ndarray):
            arr = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.n, 4)
        else:
            arr = np.array([[[(s >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)] for s in row] for row in scalars],
                           dtype=np.uint64).reshape(-1, self.n, 4)
        count = arr.shape[0]
        dev = torch.device("cuda", self.device)
        s = torch.from_numpy(arr.view(np.int64)).to(dev)
        out = torch.zeros((count, 2, 2, 4), dtype=torch.int64, device=dev)
        scratch = torch.empty(self.scratch_bytes(count), dtype=torch.uint8, device=dev)
        self.msm(s.data_ptr(), self.n, count, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize(dev)
        v = limbs_to_ints(out.cpu().numpy().view(np.uint64))
        return [None if not any(v[4 * i:4 * i + 4]) else ((v[4 * i], v[4 * i + 1]), (v[4 * i + 2], v[4 * i + 3]))
                for i in range(count)]


class Bls12381G1Bases:
    """BLS12-381 G1 points on the device for multi-scalar multiplications (cw_bls12381_g1_bases_*, include/circom_b200.h).
    points: numpy uint64 [n][2][6] canonical affine (381-bit coordinates, 6 limbs each), or a list of (x, y) ints; (0, 0)
    or None is the point at infinity.  Points are checked to lie on y^2 = x^3 + 4, not to lie in the order-r subgroup.
    Scalars are [count][n][4] uint64, as for G1Bases (BLS12-381's r has 255 bits)."""

    def __init__(self, points, device: int = 0):
        if isinstance(points, np.ndarray):
            arr = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 2, 6)
        else:
            arr = np.zeros((len(points), 2, 6), dtype=np.uint64)
            for i, p in enumerate(points):
                for j, v in enumerate((0, 0) if p is None else p):
                    arr[i, j] = [(v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(6)]
        self.n = arr.shape[0]
        self.device = device
        self._h = ctypes.c_void_p()
        check(lib.cw_bls12381_g1_bases_create(arr.ctypes.data, self.n, device, ctypes.byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_bls12381_g1_bases_destroy(h)

    def scratch_bytes(self, count: int) -> int:
        b = ctypes.c_uint64()
        check(lib.cw_bls12381_g1_msm_scratch_bytes(self._h, count, ctypes.byref(b)))
        return b.value

    def msm(self, scalars_ptr: int, stride: int, count: int, out_ptr: int, scratch_ptr: int, stream=None) -> None:
        """out[c] = sum_i s_{c,i} P_i into device [count][2][6] uint64; scalars: device [count][stride][4] uint64.
        Asynchronous on `stream` (a Batch.stream() value; None = the legacy default stream)."""
        check(lib.cw_bls12381_g1_msm_batch(self._h, ctypes.c_void_p(scalars_ptr), stride, count, ctypes.c_void_p(out_ptr),
                                           ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream or None)))

    @staticmethod
    def decode(out: np.ndarray) -> List[Optional[tuple]]:
        """[count][2][6] uint64 results -> [(x, y) or None per vector]"""
        a = np.ascontiguousarray(out, dtype=np.uint64).reshape(-1, 6)
        v = [sum(int(r[k]) << (64 * k) for k in range(6)) for r in a]
        return [None if (x, y) == (0, 0) else (x, y) for x, y in zip(v[0::2], v[1::2])]

    def msm_host(self, scalars) -> List[Optional[tuple]]:
        """the MSMs of host scalars ([count][n] ints, or numpy uint64 [count][n][4]): [(x, y) or None per vector]"""
        import torch
        if isinstance(scalars, np.ndarray):
            arr = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.n, 4)
        else:
            arr = np.array([[[(s >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)] for s in row] for row in scalars],
                           dtype=np.uint64).reshape(-1, self.n, 4)
        count = arr.shape[0]
        dev = torch.device("cuda", self.device)
        s = torch.from_numpy(arr.view(np.int64)).to(dev)
        out = torch.zeros((count, 2, 6), dtype=torch.int64, device=dev)
        scratch = torch.empty(self.scratch_bytes(count), dtype=torch.uint8, device=dev)
        self.msm(s.data_ptr(), self.n, count, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize(dev)
        return self.decode(out.cpu().numpy().view(np.uint64))


class Bls12381G2Bases:
    """BLS12-381 G2 points (on the twist y^2 = x^3 + 4 (1 + u) over Fq2) on the device for multi-scalar multiplications
    (cw_bls12381_g2_bases_*, include/circom_b200.h).  points: numpy uint64 [n][2][2][6] canonical affine (x.c0, x.c1, y.c0,
    y.c1, 6 limbs each), or a list of ((x0, x1), (y0, y1)) ints; all zeros or None is the point at infinity.  Points are
    checked to lie on the twist, not to lie in the order-r subgroup.  Scalars are [count][n][4] uint64, as for G2Bases."""

    def __init__(self, points, device: int = 0):
        if isinstance(points, np.ndarray):
            arr = np.ascontiguousarray(points, dtype=np.uint64).reshape(-1, 2, 2, 6)
        else:
            arr = np.zeros((len(points), 2, 2, 6), dtype=np.uint64)
            for i, p in enumerate(points):
                for j, e in enumerate(((0, 0), (0, 0)) if p is None else p):
                    for k, v in enumerate(e):
                        arr[i, j, k] = [(v >> (64 * m)) & 0xFFFFFFFFFFFFFFFF for m in range(6)]
        self.n = arr.shape[0]
        self.device = device
        self._h = ctypes.c_void_p()
        check(lib.cw_bls12381_g2_bases_create(arr.ctypes.data, self.n, device, ctypes.byref(self._h)))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_bls12381_g2_bases_destroy(h)

    def scratch_bytes(self, count: int) -> int:
        b = ctypes.c_uint64()
        check(lib.cw_bls12381_g2_msm_scratch_bytes(self._h, count, ctypes.byref(b)))
        return b.value

    def msm(self, scalars_ptr: int, stride: int, count: int, out_ptr: int, scratch_ptr: int, stream=None) -> None:
        """out[c] = sum_i s_{c,i} Q_i into device [count][2][2][6] uint64; scalars: device [count][stride][4] uint64.
        Asynchronous on `stream` (a Batch.stream() value; None = the legacy default stream)."""
        check(lib.cw_bls12381_g2_msm_batch(self._h, ctypes.c_void_p(scalars_ptr), stride, count, ctypes.c_void_p(out_ptr),
                                           ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream or None)))

    @staticmethod
    def decode(out: np.ndarray) -> List[Optional[tuple]]:
        """[count][2][2][6] uint64 results -> [((x0, x1), (y0, y1)) or None per vector]"""
        a = np.ascontiguousarray(out, dtype=np.uint64).reshape(-1, 6)
        v = [sum(int(r[k]) << (64 * k) for k in range(6)) for r in a]
        return [None if not any(v[i:i + 4]) else ((v[i], v[i + 1]), (v[i + 2], v[i + 3])) for i in range(0, len(v), 4)]

    def msm_host(self, scalars) -> List[Optional[tuple]]:
        """the MSMs of host scalars ([count][n] ints, or numpy uint64 [count][n][4]): [((x0, x1), (y0, y1)) or None]"""
        import torch
        if isinstance(scalars, np.ndarray):
            arr = np.ascontiguousarray(scalars, dtype=np.uint64).reshape(-1, self.n, 4)
        else:
            arr = np.array([[[(s >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(4)] for s in row] for row in scalars],
                           dtype=np.uint64).reshape(-1, self.n, 4)
        count = arr.shape[0]
        dev = torch.device("cuda", self.device)
        s = torch.from_numpy(arr.view(np.int64)).to(dev)
        out = torch.zeros((count, 2, 2, 6), dtype=torch.int64, device=dev)
        scratch = torch.empty(self.scratch_bytes(count), dtype=torch.uint8, device=dev)
        self.msm(s.data_ptr(), self.n, count, out.data_ptr(), scratch.data_ptr())
        torch.cuda.synchronize(dev)
        return self.decode(out.cpu().numpy().view(np.uint64))


def _proof_from_limbs(v: Sequence[int]):
    """one proof's 8 canonical coordinates -> (A, B, C): A, C = (x, y), B = ((x0, x1), (y0, y1)); None = infinity"""
    A = None if not any(v[0:2]) else (v[0], v[1])
    B = None if not any(v[2:6]) else ((v[2], v[3]), (v[4], v[5]))
    C = None if not any(v[6:8]) else (v[6], v[7])
    return A, B, C


def _rs_array(rs, count: int):
    """(r, s) per proof as a [count][2][4] uint64 array, or None (the library draws them)"""
    if rs is None:
        return None
    if isinstance(rs, np.ndarray):
        return np.ascontiguousarray(rs, dtype=np.uint64).reshape(count, 2, 4)
    assert len(rs) == count, "one (r, s) pair per proof"
    return ints_to_limbs([x for pair in rs for x in pair]).reshape(count, 2, 4)


class Groth16Key:
    """A BN254 Groth16 proving key on the device (cw_groth16_key_*, include/circom_b200.h), read from the bytes of a
    snarkjs .zkey - or from its path - and checked against the R1CS `r1cs` (an R1cs).  Proofs are [32] uint64 rows:
    A (x, y) | B (x.c0, x.c1, y.c0, y.c1) | C (x, y), canonical, zeros = infinity.  rs: (r, s) per proof - ints, or
    uint64 [count][2][4] - or None for blinding drawn by the library (what zero knowledge needs)."""

    def __init__(self, zkey: Union[bytes, str, os.PathLike], r1cs: "R1cs", device: int = 0):
        if not isinstance(zkey, (bytes, bytearray, memoryview)):
            with open(zkey, "rb") as f:
                zkey = f.read()
        data = bytes(zkey)
        self.device = device
        self.r1cs = r1cs
        self._h = ctypes.c_void_p()
        check(lib.cw_groth16_key_create(data, len(data), r1cs._h, device, ctypes.byref(self._h)))
        info = (ctypes.c_uint64 * 4)()
        check(lib.cw_groth16_key_info(self._h, info))
        self.info = {"n_vars": info[0], "n_public": info[1], "log2_domain": info[2], "n_coefs": info[3]}
        self.n_vars, self.n_public = info[0], info[1]

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            lib.cw_groth16_key_destroy(h)

    def ic(self) -> List[Optional[tuple]]:
        """the verifier's IC points (nPublic + 1 of them), affine (x, y) or None"""
        out = np.zeros((self.n_public + 1, 2, 4), dtype=np.uint64)
        check(lib.cw_groth16_key_ic(self._h, out.ctypes.data))
        v = limbs_to_ints(out)
        return [None if (x, y) == (0, 0) else (x, y) for x, y in zip(v[0::2], v[1::2])]

    def scratch_bytes(self, count: int) -> int:
        b = ctypes.c_uint64()
        check(lib.cw_groth16_scratch_bytes(self._h, count, ctypes.byref(b)))
        return b.value

    def prove_batch(self, batch: "Batch", first: int, count: int, proofs_ptr: int, scratch_ptr: int, rs=None) -> None:
        """proofs of instances [first, first + count) of a batch that has run into device [count][32] uint64;
        asynchronous on the batch stream.  Instances whose witness violates the R1CS give proofs that do not verify."""
        a = _rs_array(rs, count)
        check(lib.cw_groth16_prove_batch(self._h, self.r1cs._h, batch._h, first, count, None if a is None else a.ctypes.data,
                                         ctypes.c_void_p(proofs_ptr), ctypes.c_void_p(scratch_ptr)))

    def last_ms(self) -> dict:
        """device ms of the stages of the last prove call (waits for it): expansion, quotient, H, A, B1, B2, C, assembly"""
        ms = (ctypes.c_float * 8)()
        check(lib.cw_groth16_last_ms(self._h, ms))
        return dict(zip(("expansion", "quotient", "H", "A", "B1", "B2", "C", "assembly"), (float(x) for x in ms)))

    def prove(self, witness_ptr: int, stride: Optional[int], count: int, proofs_ptr: int, scratch_ptr: int, rs=None) -> None:
        """proofs of `count` dense witness rows on the device, `stride` 32-byte elements apart (None: nVars); returns
        when the proofs are written"""
        a = _rs_array(rs, count)
        check(lib.cw_groth16_prove_strided(self._h, self.r1cs._h, ctypes.c_void_p(witness_ptr), stride or self.n_vars, count,
                                           None if a is None else a.ctypes.data, ctypes.c_void_p(proofs_ptr),
                                           ctypes.c_void_p(scratch_ptr)))

    def _chunk(self, count: int, max_scratch: Optional[int]) -> int:
        import torch
        budget = max_scratch if max_scratch is not None else torch.cuda.mem_get_info(self.device)[0] // 2
        c = count
        while c > 1 and self.scratch_bytes(c) > budget:
            c = (c + 1) // 2
        return c

    def prove_host(self, source, rs=None, first: int = 0, count: Optional[int] = None,
                   max_scratch: Optional[int] = None) -> list:
        """proofs as Python ints, [(A, B, C)] (see _proof_from_limbs), in chunks whose scratch fits max_scratch bytes
        (None: half the free device memory).  source: a Batch that has run - instances [first, first + count), refused
        if any of them has a non-zero status - or host witness rows (uint64 [count][nVars][4], or lists of ints)."""
        import torch
        dev = torch.device("cuda", self.device)
        if isinstance(source, Batch):
            count = source.batch - first if count is None else count
            st = source.status()[first:first + count]
            if (st != 0).any():
                bad = int(np.nonzero(st)[0][0])
                raise CwError(native.CW_ESTATE, "instance %d has status %d: its witness is not valid" % (first + bad, st[bad]))
            rows = None
        else:
            rows = source if isinstance(source, np.ndarray) else ints_to_limbs([x for row in source for x in row])
            rows = np.ascontiguousarray(rows, dtype=np.uint64).reshape(-1, self.n_vars, 4)
            count = rows.shape[0]
        a = _rs_array(rs, count)
        chunk = self._chunk(count, max_scratch)
        out = []
        scratch = torch.empty(self.scratch_bytes(chunk), dtype=torch.uint8, device=dev)
        for i0 in range(0, count, chunk):
            cn = min(chunk, count - i0)
            proofs = torch.empty((cn, 32), dtype=torch.int64, device=dev)
            part = None if a is None else a[i0:i0 + cn]
            # (torch's allocations are ordered on its current stream; the batch stream is another one)
            torch.cuda.current_stream(dev).synchronize()
            if rows is None:
                self.prove_batch(source, first + i0, cn, proofs.data_ptr(), scratch.data_ptr(), part)
                source.sync()
            else:
                w = torch.from_numpy(rows[i0:i0 + cn].view(np.int64)).to(dev)
                self.prove(w.data_ptr(), self.n_vars, cn, proofs.data_ptr(), scratch.data_ptr(), part)
            v = limbs_to_ints(proofs.cpu().numpy().view(np.uint64))
            out += [_proof_from_limbs(v[8 * i:8 * i + 8]) for i in range(cn)]
        return out

    @staticmethod
    def proof_json(proof) -> str:
        """snarkjs' proof.json text of one proof: a (A, B, C) tuple as prove_host returns, or its [32] uint64 row"""
        if isinstance(proof, np.ndarray):
            row = np.ascontiguousarray(proof, dtype=np.uint64).reshape(32)
        else:
            A, B, C = proof
            row = ints_to_limbs(list(A or (0, 0)) + ([0] * 4 if B is None else [B[0][0], B[0][1], B[1][0], B[1][1]])
                                + list(C or (0, 0))).reshape(32)
        return _text(lambda buf, cap, ln: lib.cw_groth16_proof_json(row.ctypes.data, buf, cap, ln))

    @staticmethod
    def public_json(signals: Sequence[int]) -> str:
        """snarkjs' public.json text of the public signals w_1..w_nPublic"""
        arr = ints_to_limbs(list(signals)) if len(signals) else np.zeros((1, 4), dtype=np.uint64)
        return _text(lambda buf, cap, ln: lib.cw_groth16_public_json(arr.ctypes.data, len(signals), buf, cap, ln))


def _text(call) -> str:
    n = ctypes.c_size_t()
    check(call(None, 0, ctypes.byref(n)))
    buf = ctypes.create_string_buffer(n.value + 1)
    check(call(buf, n.value + 1, ctypes.byref(n)))
    return buf.value.decode()


class WitnessCalculator:
    """`builder(code, options)` of witness_calculator.js:1-106, for a circuit description."""

    def __init__(self, circuit: Union[Circuit, CircuitDesc, bytes, str], sanity_check: bool = True, device: int = 0,
                 compact: Optional[bool] = None):
        self.circuit = circuit if isinstance(circuit, Circuit) else Circuit(circuit, sanity_check=sanity_check, compact=compact)
        # witness_calculator.js:108-131: `init((this.sanityCheck || sanityCheck) ? 1 : 0)` - a calculator built without the
        # `===` asserts still runs them for a call that asks for them (a second lowering of the same description, made on demand)
        self._sanity = sanity_check
        self._src = None if isinstance(circuit, Circuit) else (circuit, compact)
        self._strict: Optional[Circuit] = None
        self.device = device
        self.prime = self.circuit.prime
        self.witnessSize = self.circuit.n_witness
        self.n32 = 2 * ((self.prime.bit_length() + 63) // 64)   # getFieldNumLen32 (wasm_code_generator.rs:655-674): 8; goldilocks 2
        self._batches: Dict[int, Batch] = {}

    def circom_version(self) -> int:
        return 2

    def _batch(self, n: int) -> Batch:
        b = self._batches.get(n)
        if b is None:
            b = Batch(self.circuit, n, self.device)
            self._batches = {n: b}  # keep one
        return b

    def _run(self, inputs: Sequence[dict], sanityCheck: bool = False) -> Batch:
        c = self.circuit
        if sanityCheck and not self._sanity and self._src is not None:
            if self._strict is None:
                self._strict = Circuit(self._src[0], sanity_check=True, compact=self._src[1])
            c = self._strict
        flat: List[int] = []
        for inp in inputs:
            flat.extend(c.flatten_inputs(inp))
        b = self._batch(len(inputs)) if c is self.circuit else Batch(c, len(inputs), self.device)
        b.set_inputs(ints_to_limbs(flat).reshape(len(inputs), c.n_inputs, 4))
        b.run()
        st = b.status()
        bad = np.nonzero(st)[0]
        if bad.size:
            i = int(bad[0])
            if st[i] < 0:
                raise RuntimeError("Error: division by zero in instance %d" % i)
            try:
                where = " " + c.assert_info(int(st[i]) - 1)
            except Exception:
                where = ""
            raise RuntimeError("Error: Assert Failed. (assert #%d, instance %d)%s" % (int(st[i]) - 1, i, where))
        return b

    # --- the reference surface (single input) ------------------------------------------------------
    def calculateWitness(self, input: dict, sanityCheck: bool = False) -> List[int]:
        return limbs_to_ints(self._run([input], sanityCheck).witness()[0])

    def calculateBinWitness(self, input: dict, sanityCheck: bool = False) -> bytes:
        """witnessSize x n32 32-bit words (witness_calculator.js:194-210)"""
        w = self._run([input], sanityCheck).witness()[0]
        return np.ascontiguousarray(w[:, :self.n32 // 2]).tobytes()

    def calculateWTNSBin(self, input: dict, sanityCheck: bool = False) -> bytes:
        return self._run([input], sanityCheck).wtns_bytes(0)

    # --- batch variants -----------------------------------------------------------------------------
    def calculate_witness_batch(self, inputs: Sequence[dict]) -> np.ndarray:
        """uint64 [batch][witnessSize][4], canonical little-endian limbs."""
        return self._run(inputs).witness()

    def calculate_wtns_batch(self, inputs: Sequence[dict]) -> List[bytes]:
        b = self._run(inputs)
        return [b.wtns_bytes(i) for i in range(len(inputs))]


def builder(code: Union[CircuitDesc, bytes, str], options: Optional[dict] = None) -> WitnessCalculator:
    options = options or {}
    return WitnessCalculator(code, sanity_check=options.get("sanityCheck", True), device=options.get("device", 0),
                             compact=options.get("compact"))
