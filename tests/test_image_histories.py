"""Seeded random histories of a sleeping image's operations against an executable model of their contract (include/fma_engine.h:
fma_image_move, fma_image_verify, fma_image_prefetch, and the sleeps, wakes, frees and allocations around them).

Each history allocates 4-9 segments of 1-4 pages (tags weights / adapters / kv_cache; bf16 weights that code, noise that stays raw
and pages with exactly 2048 exceptions, every page stamped with its own id: tests/pagegen.py) and runs 24 steps: sleeps
in every tier (plain and PACKED images in turn, INCREMENTAL, a resident share), moves to any tier, prefetches with any budget,
verifies, one flipped bit in the store or the image file, frees and allocations while asleep, tag-selective / retried / full /
KEEP_BACKUP wakes, file_store and host_release.  The model predicts every outcome before the step runs, refusals included, and
after every step the engine's segments, statistics, page table and stored pages must be what the model says.  On the host-simulated
engine a step may also make the next driver call fail (tests/cpp/hostsim/hostsim_cuda.cpp) and the failure must leave what the
header says.  The -m gpu tests run on an H100; test_image_histories_against_the_host_simulated_engine reruns them on CPU.
A failure names the seed and prints the history up to the failing step."""
import collections
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.pagegen import stamp
from tests.test_image_verify import _flip_file, _snapshot
from tests.test_resident_share import _resident_split, _same_stored_page

PAGE = 2 << 20
HDR = (3 << 19) + (12 << 10)               # a coded page's header (csrc/fma_codec.h kHdrOff): magic, exception count
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "cpp", "hostsim")
gpu = pytest.mark.gpu
HOSTSIM = os.environ.get("FMA_HOSTSIM") == "1"
SEEDS = list(range(1, 1 + int(os.environ.get("FMA_TEST_SEEDS", "12"))))
TAGS = ["weights", "adapters", "kv_cache"]
KINDS = ["weights", "noise", "exc2048"]     # pool pages: coded, raw, coded at the exception capacity
STEPS = 24                                  # random steps, the scenarios every history runs once among them


def _L():
    from fma_b200 import _lib as L

    return L


def _n_gpus():
    if HOSTSIM:
        return int(os.environ.get("HOSTSIM_DEVICES", "2"))
    import torch

    return torch.cuda.device_count()


def _pool(oracle):
    rng = np.random.default_rng(2048)
    n = PAGE // 2
    exc = np.full(n, 0x3F80, np.uint16)
    exc[rng.choice(n, 2048, replace=False)] = 0x0080 | 0x0055
    pool = [oracle.bf16_weights(n, 17).view(np.uint8), rng.integers(0, 256, PAGE, dtype=np.uint8), exc.view(np.uint8)]
    assert [oracle.pack_page(p).size for p in pool] == [_L().FMA_PACKED_PAGE_BYTES, PAGE, _L().FMA_PACKED_PAGE_BYTES]
    return pool


class Refused(Exception):
    """What the model says a call returns instead of succeeding"""

    def __init__(self, code):
        self.code = code


class Seg:
    def __init__(self, uid, tag, kinds, va, pages):
        self.uid, self.tag, self.kinds, self.va, self.pages = uid, tag, kinds, va, pages
        self.bytes = len(pages) * PAGE
        self.mapped, self.backup, self.tier, self.off = True, False, None, None
        self.digest = False                 # the sleep recorded a K3 digest
        self.res = False                    # in the resident share
        self.pf = None                      # offset in the prefetch buffer
        self.store_bad = self.pf_bad = False
        self.known = True                   # its bytes are defined (a discarded segment's are not, until rewritten)
        self._stored = {}

    def data(self):
        return b"".join(p.tobytes() for p in self.pages)

    def stored(self, oracle, j):
        if j not in self._stored:
            self._stored[j] = oracle.pack_page(self.pages[j])
        return self._stored[j]


class Model:
    """One engine's segments and its sleeping image, as include/fma_engine.h describes them."""

    def __init__(self):
        self.segs = []                      # live segments in engine index order
        self.tag_rank = {}                  # arenas: one per tag, in the order tags were first allocated
        self.tier = None                    # the image's tier (None: no image yet)
        self.st_tier = 0                    # fma_stats_t.tier
        self.packed, self.res_packed = False, False
        self.pages = []                     # stored size of every image page of the store's part (image order)
        self.res_pages = []
        self.store_bytes = self.res_bytes = self.pf_bytes = self.offloaded = 0
        self.image_file = None              # the file the image sleeps in
        self.path = None                    # fma_file_store
        self.park = None                    # ("local" | "peer", bytes)
        self.exact_mapped = True            # no wake since the last sleep: hbm_mapped_bytes is the allocations made since
        self.kept_forms = set()             # INCREMENTAL: forms a kept image may have

    def index(self, s):
        return self.segs.index(s)

    def asleep(self):
        return [s for s in self.segs if s.backup and not s.mapped]

    def backup_mapped(self):
        return any(s.backup and s.mapped for s in self.segs)

    def is_sleeping(self):
        return any(not s.mapped for s in self.segs)

    def order(self, segs):
        return sorted(segs, key=lambda s: (self.tag_rank[s.tag], s.va))

    def seg_stored(self, s):
        if s.res:
            return sum(self.res_pages[s.off // PAGE + j] for j in range(len(s.pages)))
        return sum(self.pages[s.off // PAGE + j] for j in range(len(s.pages)))

    def resident(self):
        return self.res_bytes > 0

    def mapped_bytes(self):
        return sum(s.bytes for s in self.segs if s.mapped)


def _tier_name(t):
    return {0: "host", 1: "peer", 2: "local", 3: "file"}.get(t, str(t))


class History:
    def __init__(self, engine, oracle, seed, tmp_path):
        self.e, self.o, self.seed, self.tmp = engine, oracle, seed, tmp_path
        self.rng = np.random.default_rng(seed)
        self.m = Model()
        self.pool = _pool(oracle)
        self.log = []
        self.counts = collections.Counter()
        self.next_uid = 0
        self.n_sleeps = 0
        self.forced = None
        self.peer = _n_gpus() >= 2

    # ---- helpers ----------------------------------------------------------------------------------------------------
    def note(self, text):
        self.log.append(text)

    def fail_msg(self):
        return f"seed {self.seed}, history so far:\n  " + "\n  ".join(f"{k}: {t}" for k, t in enumerate(self.log))

    def expect(self, cond, what):
        assert cond, f"{what}\n{self.fail_msg()}"

    def call(self, fn, refusal=None, count_as=None, injected=False):
        """Run fn; refusal is the code the model predicts (None: success).  A refusal must leave _snapshot as it was.  With an
        injected failure armed, a failure goes to the caller."""
        L = _L()
        before = _snapshot(self.e) if refusal is not None else None
        try:
            out = fn()
        except L.FmaError as ex:
            if refusal is None and injected:
                raise
            self.expect(refusal is not None and ex.code == refusal, f"refused with {ex} where the model said {refusal}")
            self.expect(_snapshot(self.e) == before, "a refusal changed the engine")
            self.counts["refusal"] += 1
            if count_as:
                self.counts[f"refusal:{count_as}"] += 1
            return Refused(ex.code)
        self.expect(refusal is None, f"succeeded where the model said {refusal}")
        return out

    def alloc(self, tag=None):
        tag = tag or TAGS[int(self.rng.integers(0, 3))]
        kinds = [int(k) for k in self.rng.integers(0, 3, int(self.rng.integers(1, 5)))]
        uid = self.next_uid
        self.next_uid += 1
        pages = [stamp(self.pool[k], self.seed, 8 * uid + j) for j, k in enumerate(kinds)]
        va = self.e.alloc(len(pages) * PAGE, tag)
        self.m.tag_rank.setdefault(tag, len(self.m.tag_rank))
        s = Seg(uid, tag, kinds, va, pages)
        self.m.segs.append(s)
        self.e.write(self.m.index(s), s.data())
        return s

    # ---- invariants after every step ------------------------------------------------------------------------------------
    def check(self):
        L, e, m = _L(), self.e, self.m
        info = e.segments()
        self.expect([s.va for s in info] == [s.va for s in m.segs], "segment VAs moved")
        for i, (s, g) in enumerate(zip(m.segs, info)):
            self.expect((g.mapped, g.has_backup) == (s.mapped, s.backup), f"segment {i}: mapped/backup {(g.mapped, g.has_backup)} != {(s.mapped, s.backup)}")
            if s.backup:
                self.expect(g.tier == s.tier and g.packed_offset == s.off, f"segment {i}: tier/offset {(g.tier, g.packed_offset)} != {(s.tier, s.off)}")
        st = e.stats()
        want = {"tier": m.st_tier, "image_packed": int(m.packed), "image_store_bytes": m.store_bytes, "prefetched_bytes": m.pf_bytes,
                "resident_bytes": m.res_bytes, "sleep_bytes_offloaded": m.offloaded, "parked_bytes": m.park[1] if m.park else 0}
        got = {k: st[k] for k in want}
        self.expect(got == want, f"stats {got} != model {want}")
        self.expect(e.is_sleeping() == m.is_sleeping(), "is_sleeping")
        if m.exact_mapped:
            self.expect(st["hbm_mapped_bytes"] == m.mapped_bytes(), f"hbm_mapped_bytes {st['hbm_mapped_bytes']} != {m.mapped_bytes()}")
        else:
            self.expect(st["hbm_mapped_bytes"] >= m.mapped_bytes(), "hbm_mapped_bytes below the mapped segments")
        for i, s in enumerate(m.segs):                       # mapped bytes come back exactly
            if s.mapped and s.known:
                self.expect(e.read(i, s.bytes) == s.data(), f"segment {i} (uid {s.uid}) holds other bytes")
        if m.asleep():
            off, nb = e.image_pages()
            want_nb = m.pages + m.res_pages
            self.expect(nb == want_nb, f"image_pages sizes {nb} != {want_nb}")
            host = [sum(m.pages[:k]) for k in range(len(m.pages))] if m.packed else [k * PAGE for k in range(len(m.pages))]
            res = [sum(m.res_pages[:k]) for k in range(len(m.res_pages))] if m.res_packed else [k * PAGE for k in range(len(m.res_pages))]
            self.expect(off == host + res, "image_pages offsets")
            spans = sorted((s.res, s.off, s.off + s.bytes) for s in m.segs if s.backup)
            for a, b in zip(spans, spans[1:]):               # live segments do not overlap and lie inside their part
                self.expect(a[0] != b[0] or a[2] <= b[1], f"image offsets overlap: {a} {b}")
            for r, lo, hi in spans:
                self.expect(hi <= (len(m.res_pages) if r else len(m.pages)) * PAGE, "a segment lies outside the image")

    def check_store(self):
        """Every stored page of the store's part, where it lies, against the oracle's stored form (after a sleep or a move into the
        host or file tier)."""
        L, e, m = _L(), self.e, self.m
        if not m.pages:                                      # (all of it in a resident share: no store)
            return
        if m.tier == L.FMA_TIER_HOST:
            base, n = e.host_store_view()
            self.expect(n == m.store_bytes, f"host store view {n} != {m.store_bytes}")
            img = np.ctypeslib.as_array((C.c_uint8 * n).from_address(base)) if n else np.empty(0, np.uint8)
        elif m.tier == L.FMA_TIER_FILE:
            img = np.fromfile(m.image_file, dtype=np.uint8)
            self.expect(img.size == m.store_bytes + (2 << 20), "image file size")
        else:
            return
        offs = [sum(m.pages[:k]) for k in range(len(m.pages))]
        for s in m.segs:
            if not s.backup or s.res:
                continue
            for j in range(len(s.pages)):
                q = s.off // PAGE + j
                got = img[offs[q]:offs[q] + m.pages[q]]
                want = s.stored(self.o, j) if m.packed else s.pages[j]
                self.expect(_same_stored_page(got, want), f"stored page {j} of uid {s.uid} differs from the oracle's")

    # ---- steps ------------------------------------------------------------------------------------------------------------
    def step_sleep(self):
        L, e, m, rng = _L(), self.e, self.m, self.rng
        tags = [t for t in TAGS if rng.random() < 0.6] or ["weights"]
        choices = ["host", "local", "file", "host_resident"] + (["peer"] if self.peer else [])
        where = choices[int(rng.integers(0, len(choices)))]
        if where == "peer" and any(s.backup and s.tier in (L.FMA_TIER_PEER, L.FMA_TIER_LOCAL) for s in m.segs):
            where = "host"                                   # (a parking buffer that holds an image cannot be replaced)
        tier = {"host": 0, "host_resident": 0, "local": 2, "file": 3, "peer": 1}[where]
        pack = self.n_sleeps % 2                              # plain and PACKED images in turn
        mode = [L.FMA_MODE_AUTO, L.FMA_MODE_STAGED, L.FMA_MODE_DIRECT, L.FMA_MODE_KERNEL][int(rng.choice(4, p=[0.5, 0.2, 0.15, 0.15]))]
        inc = int(rng.random() < 0.3) if where != "host_resident" else 0
        flags = L.FMA_FLAG_VERIFY if rng.random() < 0.7 else 0
        cap = int(rng.integers(1, 12)) * PAGE + int(rng.integers(0, PAGE)) if where == "host_resident" else 0
        self.note(f"sleep tags={tags} tier={where} pack={pack} mode={mode} incremental={inc} verify={bool(flags)} resident_bytes={cap}")
        e.set_option("pack", pack)
        e.set_option("mode", mode)
        e.set_option("incremental", inc)
        e.set_option("resident_bytes", cap)
        if where == "file":
            m.path = str(self.tmp / f"img{int(rng.integers(0, 2))}.fmaimg")
            e.file_store(m.path)
        W_all = sum(s.bytes for s in m.segs if s.tag in tags)
        if where == "peer":
            self.peer_reserve(W_all)
        if m.is_sleeping() or not m.segs:                     # asleep already: a harmless no-op
            e.sleep(tags, tier=tier, flags=flags)
            self.counts["sleep:noop"] += 1
            return
        self.n_sleeps += 1
        e.sleep(tags, tier=tier, flags=flags)
        # the model's sleep
        m.pf_bytes = 0
        for s in m.segs:
            s.pf, s.res, s.backup, s.off, s.tier, s.digest = None, False, False, None, None, False
            s.store_bad = s.pf_bad = False
            s.mapped = False
            if s.tag not in tags:
                s.known = False                              # discarded
        off = [s for s in m.order(m.segs) if s.tag in tags]
        W = sum(s.bytes for s in off)
        resolved = 2 if tier == 3 else (2 if tier == 0 else 3) if mode == L.FMA_MODE_AUTO else (3 if tier != 0 and mode == L.FMA_MODE_STAGED else mode)
        coded = bool(pack) and (tier == 3 or (tier == 0 and resolved == L.FMA_MODE_STAGED) or (tier in (1, 2) and resolved == L.FMA_MODE_KERNEL))
        sizes = {s.uid: [s.stored(self.o, j).size for j in range(len(s.pages))] for s in off}
        packed_total = sum(sum(v) for v in sizes.values())
        packed = coded and W > 0 and packed_total * 100 <= W * 95
        st = e.stats()
        if inc and (st["image_packed"] != packed) and W:
            # INCREMENTAL: a clean or partial sleep keeps the form of the image the store kept
            self.expect(st["image_packed"] in m.kept_forms, f"INCREMENTAL sleep took form {st['image_packed']}, kept forms {m.kept_forms}")
            packed = bool(st["image_packed"])
        keep = [False] * len(off)
        if where == "host_resident" and W:
            keep = _resident_split([sum(sizes[s.uid]) if packed else s.bytes for s in off], cap)
        host_part = [s for s, k in zip(off, keep) if not k]
        res_part = [s for s, k in zip(off, keep) if k]
        m.tier = m.st_tier = tier
        m.packed = packed and bool(host_part)
        m.res_packed = packed
        m.pages, m.res_pages = [], []
        for part, pages, seg_tier in ((host_part, m.pages, tier), (res_part, m.res_pages, L.FMA_TIER_LOCAL)):
            at = 0
            for s in part:
                s.backup, s.tier, s.off, s.res = True, seg_tier, at, part is res_part
                s.digest = bool(flags) or bool(inc)
                s.known = True
                at += s.bytes
                pages += sizes[s.uid] if (packed if part is res_part else m.packed) else [PAGE] * len(s.pages)
        m.store_bytes = sum(m.pages)
        m.res_bytes = sum(m.res_pages)
        m.offloaded = W
        if tier == 3:
            m.image_file = m.path
        if tier == 2 and W:
            need = -(-max(m.store_bytes, PAGE) // PAGE) * PAGE
            if not (m.park and m.park[0] == "local" and m.park[1] >= need):
                m.park = ("local", need)
        m.exact_mapped = True
        m.kept_forms = {int(m.packed)} if inc else set()
        self.counts[f"sleep:{where}"] += 1
        self.counts["form:packed" if m.packed else "form:plain"] += 1
        if host_part and tier == 0 and not res_part:
            self.expect([s.uid for s in sorted(host_part, key=lambda s: s.off)] == [s.uid for s in host_part], "image order")
        self.check()
        self.check_store()

    def peer_reserve(self, nbytes):
        """a parking buffer on the second GPU; one there that is large enough stays"""
        need = -(-max(nbytes, PAGE) // PAGE) * PAGE
        self.e.peer_reserve(1, need)
        if not (self.m.park and self.m.park[0] == "peer" and self.m.park[1] >= need):
            self.m.park = ("peer", need)

    def move_refusal(self, to):
        L, m = _L(), self.m
        park = (L.FMA_TIER_PEER, L.FMA_TIER_LOCAL)
        if to not in (0, 1, 2, 3):
            return L.FMA_EINVAL
        if not m.asleep():
            return L.FMA_ESTATE
        if m.backup_mapped():
            return L.FMA_ESTATE
        if any(s.res for s in m.asleep()):
            return L.FMA_ESTATE
        if to == m.tier or (m.tier in park and to in park):
            return L.FMA_EINVAL
        if to == L.FMA_TIER_FILE and not m.path:
            return L.FMA_ESTATE
        if to == L.FMA_TIER_PEER and not (m.park and m.park[0] == "peer" and m.park[1] >= m.store_bytes):
            return L.FMA_ESTATE
        return None

    def step_move(self, to=None, allow_inject=True):
        L, e, m, rng = _L(), self.e, self.m, self.rng
        choices = [0, 2, 3, 7] + ([1] if self.peer else [])
        if to is None:
            to = int(choices[int(rng.integers(0, len(choices)))])
        if m.pf_bytes and rng.random() < 0.25:               # a move into HBM drops the prefetched copy
            to = 1 if self.peer and rng.random() < 0.5 else 2
        if to == 1 and not (m.park and m.park[0] == "peer") and rng.random() < 0.7 and \
                not any(s.backup and s.tier in (1, 2) for s in m.segs):
            self.peer_reserve(m.store_bytes)
        refusal = self.move_refusal(to)
        inject = self.inject("move") if refusal is None and allow_inject else None
        self.note(f"move to {_tier_name(to)} (model: {'ok' if refusal is None else refusal}{', inject ' + inject if inject else ''})")
        before = _snapshot(e)
        try:
            r = self.call(lambda: e.move_image(to), refusal, "move", bool(inject))
        except _L().FmaError as ex:
            self.injected_failure("move", ex, before)
            return
        finally:
            self.disarm()
        self.counts["move"] += 1
        if isinstance(r, Refused):
            return
        if inject:
            self.counts["inject_missed"] += 1
        m.tier = m.st_tier = to
        for s in m.asleep():
            s.tier = to
        if to == L.FMA_TIER_FILE:
            m.image_file = m.path
            m.kept_forms = set()
        if to in (1, 2):
            self.counts["move:drops_prefetch"] += bool(m.pf_bytes)
            for s in m.segs:
                s.pf, s.pf_bad = None, False
            m.pf_bytes = 0
        if to == 2:
            need = -(-max(m.store_bytes, PAGE) // PAGE) * PAGE
            if not (m.park and m.park[0] == "local" and m.park[1] >= need):
                m.park = ("local", need)
        m.kept_forms = set()                                 # the shadows stayed in the store the image left
        self.counts[f"move:{_tier_name(to)}"] += 1
        self.check()
        self.check_store()

    def prefetch_refusal(self, nbytes):
        L, m = _L(), self.m
        if nbytes == 0:
            return None
        if m.backup_mapped() or not m.asleep() or m.resident():
            return L.FMA_ESTATE
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE):
            return L.FMA_EINVAL
        return None

    def prefetch_model(self, nbytes):
        m = self.m
        for s in m.segs:
            s.pf, s.pf_bad = None, False
        m.pf_bytes = 0
        if not nbytes:
            return []
        order = sorted(m.asleep(), key=lambda s: s.off)
        stored = [m.seg_stored(s) for s in order]
        keep = _resident_split(stored, nbytes)
        at = 0
        taken = []
        for s, k, n in zip(order, keep, stored):
            if k:
                s.pf, s.pf_bad = at, s.store_bad           # damage in the store is carried into the copy
                at += s.bytes
                m.pf_bytes += n
                taken.append(s)
        return taken

    def step_prefetch(self, nbytes=None, allow_inject=True, armed=None):
        L, e, m, rng = _L(), self.e, self.m, self.rng
        if nbytes is None:
            S = m.store_bytes
            nbytes = int(rng.choice([0, int(rng.integers(0, S // PAGE + 1)) * PAGE, int(rng.integers(0, S + 1)), S + int(rng.integers(1, 4 * PAGE)),
                                     int(rng.integers(1, 4)) * PAGE + int(rng.integers(1, PAGE))]))
        refusal = self.prefetch_refusal(nbytes)
        inject = armed or (self.inject("prefetch") if refusal is None and nbytes and allow_inject and self.prefetch_takes(nbytes) else None)
        self.note(f"prefetch {nbytes} (model: {'ok' if refusal is None else refusal}{', inject ' + inject if inject else ''})")
        before = _snapshot(e)
        try:
            r = self.call(lambda: e.prefetch_image(nbytes), refusal, "prefetch", bool(inject))
        except _L().FmaError as ex:
            self.injected_failure("prefetch", ex, before)
            return
        finally:
            self.disarm()
        self.counts["prefetch"] += 1
        if isinstance(r, Refused):
            return
        if inject:
            self.counts["inject_missed"] += 1
        self.prefetch_model(nbytes)
        self.check()

    def prefetch_takes(self, nbytes):
        order = sorted(self.m.asleep(), key=lambda s: s.off)
        return any(_resident_split([self.m.seg_stored(s) for s in order], nbytes))

    def verify_refusal(self):
        L, m = _L(), self.m
        if m.backup_mapped() or not m.asleep() or any(not s.digest for s in m.asleep()):
            return L.FMA_ESTATE
        return None

    def expected_bad(self):
        return sorted(i for i, s in enumerate(self.m.segs) if s.backup and not s.mapped and (s.store_bad or (s.pf is not None and s.pf_bad)))

    def step_verify(self, allow_inject=True):
        L, e = _L(), self.e
        refusal = self.verify_refusal()
        inject = self.inject("verify") if refusal is None and allow_inject else None
        self.note(f"verify (model: {self.expected_bad() if refusal is None else refusal}{', inject ' + inject if inject else ''})")
        before = _snapshot(e)
        try:
            bad = self.call(e.verify_image, refusal, "verify", bool(inject))
        except _L().FmaError as ex:
            self.injected_failure("verify", ex, before)
            return None
        finally:
            self.disarm()
        self.counts["verify"] += 1
        if isinstance(bad, Refused):
            return bad
        self.expect(_snapshot(e) == before, "verify changed the engine")
        self.expect(bad == self.expected_bad(), f"verify reported {bad}, the model {self.expected_bad()}")
        self.counts["verify:bad_twice"] += any(s.store_bad and s.pf is not None and s.pf_bad for s in self.m.segs)
        if inject:
            self.counts["inject_missed"] += 1
        return bad

    # damage: one flipped bit of one stored page that the test can reach (host store, image file)
    def damage_target(self, want_pf=None):
        L, m, rng = _L(), self.m, self.rng
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or self.verify_refusal() is not None:
            return None
        cands = [s for s in m.asleep() if not s.res and (want_pf is None or (s.pf is not None) == want_pf)]
        if not cands:
            return None
        s = cands[int(rng.integers(0, len(cands)))]
        j = int(rng.integers(0, len(s.pages)))
        q = s.off // PAGE + j
        off = sum(m.pages[:q]) if m.packed else q * PAGE
        coded = m.packed and m.pages[q] != PAGE
        at = off + (HDR if coded and rng.random() < 0.3 else m.pages[q] // 3)
        kind = ("header" if at - off == HDR else "coded") if coded else ("raw" if m.packed else "plain")
        if m.tier == L.FMA_TIER_HOST:
            base, _ = self.e.host_store_view()
            addr = base + at

            def flip():
                b = (C.c_uint8 * 1).from_address(addr)
                b[0] ^= 0x04
        else:
            path = m.image_file

            def flip():
                _flip_file(path, at)
        return s, kind, flip

    def step_damage(self, variant=None):
        m, rng = self.m, self.rng
        t = self.damage_target()
        if t is None:
            self.note("damage: nothing reachable")
            return self.step_verify()
        s, kind, flip = t
        variant = variant or ("carry" if (rng.random() < 0.6 and not m.resident()) else "plain")
        self.note(f"damage uid {s.uid} ({kind} page, {_tier_name(m.tier)}), {variant}")
        self.counts[f"damage:{kind}"] += 1
        flip()
        s.store_bad = True
        self.step_verify(allow_inject=False)
        if variant == "carry":                              # a prefetch taken now carries the damage into HBM
            self.step_prefetch(m.store_bytes + PAGE if rng.random() < 0.7 or self.forced == "carry" else None, allow_inject=False)
            self.step_verify(allow_inject=False)            # bad in the store and in its copy: reported once
            flip()
            s.store_bad = False
            self.note(f"repair uid {s.uid}")
            self.step_verify(allow_inject=False)
            if any(x.pf_bad for x in m.segs):               # drop or re-take the copy before anything wakes from it
                self.step_prefetch(0 if rng.random() < 0.5 else m.store_bytes + PAGE, allow_inject=False)
                self.expect(not any(x.pf_bad for x in m.segs), "a re-taken prefetch still carries the damage")
                self.step_verify(allow_inject=False)
        else:
            flip()
            s.store_bad = False
            self.note(f"repair uid {s.uid}")
            self.step_verify(allow_inject=False)
        self.counts["damage"] += 1

    def step_damage_prefetched_then_wake(self):
        """The store of a prefetched segment damaged, then a VERIFY wake: the wake reads the HBM copy, so it succeeds and the
        bytes are right."""
        L, m = _L(), self.m
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or self.verify_refusal() is not None or m.resident() or not m.asleep():
            return False
        if not any(s.pf is not None for s in m.asleep()):
            self.step_prefetch(m.store_bytes + PAGE, allow_inject=False)
        t = self.damage_target(want_pf=True)
        if t is None:
            return False
        s, kind, flip = t
        self.note(f"damage uid {s.uid} ({kind} page, {_tier_name(m.tier)}) while prefetched, then a VERIFY wake")
        flip()
        s.store_bad = True
        self.step_verify(allow_inject=False)
        self.step_wake(tags=None, flags=L.FMA_FLAG_VERIFY, allow_inject=False)
        flip()                                               # (the store outlives the wake)
        s.store_bad = False
        self.note(f"repair uid {s.uid}")
        self.counts["damage:prefetched_wake"] += 1
        return True

    def forced_carry(self):
        """One flipped bit carried into a prefetch of everything: bad in the store and in its copy, it is reported once."""
        L, m = _L(), self.m
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or m.resident() or self.damage_target() is None:
            return False
        self.step_damage("carry")
        return True

    def forced_move_into_hbm(self):
        """A move into a parking buffer while part of the image is prefetched: the copy goes."""
        L, m = _L(), self.m
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or m.resident() or m.backup_mapped() or not m.asleep():
            return False
        if not m.pf_bytes:
            self.step_prefetch(m.store_bytes + PAGE, allow_inject=False)
        self.step_move(1 if self.peer and self.rng.random() < 0.5 else 2, allow_inject=False)
        return True

    def forced_hole_then_prefetch(self):
        """A segment in the middle of the image freed, then a prefetch of everything: the copy skips the hole the segment left."""
        L, m = _L(), self.m
        order = sorted(m.asleep(), key=lambda s: s.off)
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or m.resident() or m.backup_mapped() or len(order) < 3 or len(m.segs) <= 3:
            return False
        gone = order[len(order) // 2]
        self.note(f"free uid {gone.uid} (asleep, in the middle of the image)")
        self.e.free(gone.va)
        m.segs.remove(gone)
        self.counts["free:asleep"] += 1
        self.check()
        self.step_prefetch(m.store_bytes + PAGE, allow_inject=False)
        if self.verify_refusal() is None:
            self.step_verify(allow_inject=False)
        else:
            self.step_wake(tags=None, flags=0, allow_inject=False)
        return True

    def forced_failed_prefetch(self):
        """A prefetch whose buffer cannot be had (host simulation): no buffer, and nothing refers to one; then a check and a wake."""
        L, m = _L(), self.m
        if not HOSTSIM:
            return True
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or m.resident() or m.backup_mapped() or not m.asleep():
            return False
        C.CDLL(os.environ["FMA_B200_LIB"]).hostsim_fail_create_after(C.c_long(0))
        self.step_prefetch(m.store_bytes + PAGE, armed="cuMemCreate")
        self.step_verify(allow_inject=False)
        self.step_wake(tags=None, flags=L.FMA_FLAG_VERIFY, allow_inject=False)
        return True

    def forced_prefetch_then_partial_wake(self):
        return self.step_prefetch_then_partial_wake()

    def step_prefetch_then_partial_wake(self):
        """A prefetch, then a wake of a tag whose segments hold none of it: the copy stays for the segments that still sleep."""
        L, m = _L(), self.m
        if m.tier not in (L.FMA_TIER_HOST, L.FMA_TIER_FILE) or m.backup_mapped() or m.resident() or not m.asleep():
            return False
        if not m.pf_bytes:
            self.step_prefetch(int(self.rng.integers(1, max(2, m.store_bytes // PAGE))) * PAGE, allow_inject=False)
        held = {s.tag for s in m.asleep() if s.pf is not None}
        other = [t for t in TAGS if t not in held and any(s.tag == t and not s.mapped for s in m.segs)]
        if not held or not other:
            return False
        self.step_wake(tags=other, flags=0, allow_inject=False)
        self.expect(m.pf_bytes > 0, "the model dropped a prefetch whose segments still sleep")
        self.counts["wake:beside_prefetch"] += 1
        return True

    def step_wake(self, tags="random", flags=None, allow_inject=True):
        L, e, m, rng = _L(), self.e, self.m, self.rng
        if tags == "random":
            tags = None if rng.random() < 0.4 else [t for t in TAGS if rng.random() < 0.5] or ["kv_cache"]
        if flags is None:
            flags = (L.FMA_FLAG_VERIFY if rng.random() < 0.5 else 0) | (L.FMA_FLAG_KEEP_BACKUP if rng.random() < 0.15 else 0)
        targets = [s for s in m.segs if not s.mapped and (tags is None or s.tag in tags)]
        inject = self.inject("wake") if targets and allow_inject else None
        self.note(f"wake tags={tags} verify={bool(flags & 1)} keep_backup={bool(flags & 2)} ({len(targets)} segments{', inject ' + inject if inject else ''})")
        woke = False
        if inject:
            pf_before = e.stats()["prefetched_bytes"]
            try:
                e.wake(tags, flags=flags)
                self.counts["inject_missed"] += 1
                woke = True
            except L.FmaError as ex:                         # rolled back, the prefetch kept for the retry
                self.note(f"  the wake failed as injected ({ex.message[:60]}); retried")
                self.counts["inject:wake"] += 1
                self.expect(e.stats()["prefetched_bytes"] == pf_before and e.is_sleeping(), "a failed wake dropped the prefetch")
                info = e.segments()
                self.expect(all(not info[m.index(s)].mapped and info[m.index(s)].has_backup == s.backup for s in targets), "a failed wake was not rolled back")
            finally:
                self.disarm()
        if not woke:
            try:
                e.wake(tags, flags=flags)
            except L.FmaError as ex:
                self.expect(False, f"the wake failed: {ex}")
        self.counts["wake"] += 1
        self.counts["wake:" + ("full" if tags is None else "tags") + (":keep" if flags & 2 else "")] += 1
        if not targets:
            self.counts["wake:noop"] += 1
            self.check()
            return
        for s in targets:
            s.mapped = True
            if not s.backup:
                s.known = False                              # discarded: mapped again, contents undefined
        m.exact_mapped = False
        m.st_tier = m.tier
        if m.pf_bytes and (flags & 2 or not any(s.pf is not None and not s.mapped for s in m.segs)):
            self.release_pf()
        if m.res_bytes and not flags & 2 and not any(s.res and not s.mapped for s in m.segs):
            m.res_bytes, m.res_pages = 0, []
        if not flags & 2:
            for s in targets:
                if s.backup:
                    s.backup, s.off, s.tier, s.pf, s.res = False, None, None, None, False
            if m.tier is not None:
                m.kept_forms = {int(m.packed)}
        self.check()
        for s in m.segs:                                     # discarded segments get their bytes again
            if s.mapped and not s.known:
                s.known = True
                self.e.write(m.index(s), s.data())

    def release_pf(self):
        for s in self.m.segs:
            s.pf, s.pf_bad = None, False
        self.m.pf_bytes = 0

    def step_free(self):
        m, rng = self.m, self.rng
        if len(m.segs) <= 3:
            return self.step_alloc()
        asleep = [s for s in m.segs if not s.mapped]
        pool = asleep if asleep and rng.random() < 0.8 else m.segs
        s = pool[int(rng.integers(0, len(pool)))]
        self.note(f"free uid {s.uid} ({'prefetched' if s.pf is not None else 'asleep' if not s.mapped else 'mapped'})")
        self.e.free(s.va)
        m.segs.remove(s)
        self.counts["free:asleep" if not s.mapped else "free:mapped"] += 1
        self.counts["free"] += 1
        self.check()

    def step_alloc(self):
        s = self.alloc()
        self.note(f"alloc uid {s.uid} {s.tag} {len(s.pages)} pages (asleep: {self.m.is_sleeping()})")
        self.counts["alloc"] += 1
        self.check()

    def step_file_store(self):
        path = None if self.rng.random() < 0.3 else str(self.tmp / f"img{int(self.rng.integers(0, 3))}.fmaimg")
        self.note(f"file_store {path}")
        self.e.file_store(path)
        self.m.path = path
        self.counts["file_store"] += 1
        self.check()

    def step_host_release(self):
        L, m = _L(), self.m
        refusal = L.FMA_ESTATE if any(s.backup and s.tier == L.FMA_TIER_HOST for s in m.segs) else None
        self.note(f"host_release (model: {'ok' if refusal is None else refusal})")
        r = self.call(self.e.host_release, refusal, "host_release")
        if not isinstance(r, Refused):
            m.kept_forms = set() if m.tier == L.FMA_TIER_HOST else m.kept_forms
        self.counts["host_release"] += 1
        self.check()

    # ---- failure injection (host simulation only) ----------------------------------------------------------------------
    def inject(self, op):
        if not HOSTSIM or self.rng.random() >= 0.3:
            return None
        L, m = _L(), self.m
        sim = C.CDLL(os.environ["FMA_B200_LIB"])
        if op == "verify":
            sim.hostsim_fail_call_after(b"cudaMemsetAsync", C.c_long(0))
            return "cudaMemsetAsync"
        if op == "wake":
            n = int(self.rng.integers(0, 2))
            sim.hostsim_fail_call_after(b"cuMemMap", C.c_long(n))
            return f"cuMemMap#{n}"
        if self.rng.random() < 0.5:
            sim.hostsim_fail_create_after(C.c_long(0))
            return "cuMemCreate"
        sim.hostsim_fail_memcpy_after(C.c_long(0))
        return "memcpy"

    def disarm(self):
        if HOSTSIM:
            sim = C.CDLL(os.environ["FMA_B200_LIB"])
            sim.hostsim_fail_create_after(C.c_long(-1))
            sim.hostsim_fail_memcpy_after(C.c_long(-1))
            for name in (b"cuMemMap", b"cudaMemsetAsync"):
                sim.hostsim_fail_call_after(name, C.c_long(-1))

    def injected_failure(self, op, ex, before):
        """A move, prefetch or verify that failed leaves the image, its tier and every statistic as they were; a failed prefetch
        leaves no buffer (the old one went first)."""
        L = _L()
        self.expect(HOSTSIM, f"{op} failed without an injected failure: {ex}")
        self.expect(ex.code in (L.FMA_ENOMEM, L.FMA_ECUDA, L.FMA_EIO), f"{op} failed with {ex}")
        self.note(f"  {op} failed as injected: {ex.message[:80]}")
        self.counts[f"inject:{op}"] += 1
        if op == "prefetch":
            self.release_pf()
        after = _snapshot(self.e)
        self.expect(after == before, f"a failed {op} changed the engine: {before[0]} -> {after[0]}")
        self.check()

    # ---- the history -------------------------------------------------------------------------------------------------------
    def run(self):
        L, e, rng = _L(), self.e, self.rng
        e.set_option("chunk_bytes", 8 << 20)
        e.set_option("load_chunk_bytes", 4 << 20)
        e.set_option("load_slots", 3)
        for k in range(int(rng.integers(4, 10))):
            self.alloc(TAGS[k] if k < 3 else None)
        self.note(f"{len(self.m.segs)} segments: " + ", ".join(f"uid {s.uid} {s.tag} {[KINDS[k] for k in s.kinds]}" for s in self.m.segs))
        self.check()
        # scenarios every history tries once, each from a random step on, in a random order
        todo = {name: int(rng.integers(1, STEPS - 2)) for name in ("carry", "damage_prefetched_then_wake", "prefetch_then_partial_wake", "move_into_hbm",
                                                                  "hole_then_prefetch", "failed_prefetch")}
        self.forced = None
        for k in range(STEPS):
            due = [n for n, at in todo.items() if at <= k]
            if not self.m.is_sleeping():
                kind = "sleep" if rng.random() < 0.8 else str(rng.choice(["alloc", "free", "file_store", "host_release", "verify", "move", "prefetch"]))
            elif due:
                self.forced = due[int(rng.integers(0, len(due)))]
                fn = {"damage_prefetched_then_wake": self.step_damage_prefetched_then_wake}.get(self.forced) or getattr(self, "forced_" + self.forced)
                if fn():
                    del todo[self.forced]
                    self.counts["forced:" + self.forced] += 1
                    self.forced = None
                    continue
                self.forced = None
                todo[due[0]] = k + 1 + int(rng.integers(0, 3))   # not possible now: later
            if self.m.is_sleeping():
                kind = str(rng.choice(["move", "prefetch", "verify", "damage", "free", "alloc", "wake", "wake", "file_store", "host_release", "sleep"],
                                      p=[0.24, 0.15, 0.08, 0.11, 0.05, 0.03, 0.22, 0, 0.04, 0.04, 0.04]))
            getattr(self, "step_" + kind)()
        if self.m.is_sleeping():
            if any(s.store_bad or s.pf_bad for s in self.m.segs):
                raise AssertionError("damage left behind\n" + self.fail_msg())
            self.step_wake(tags=None, flags=L.FMA_FLAG_VERIFY, allow_inject=False)
        self.check()
        return self.counts


def _open_fds(tmp):
    out = []
    for fd in os.listdir("/proc/self/fd"):
        try:
            if os.readlink(f"/proc/self/fd/{fd}").startswith(str(tmp)):
                out.append(fd)
        except OSError:
            pass
    return out


@gpu
@pytest.mark.parametrize("seed", SEEDS)
def test_image_history(built, oracle, tmp_path, seed):
    import fma_b200

    try:
        eng = fma_b200.Engine(0)
    except _L().FmaError as ex:
        if HOSTSIM or ex.code != _L().FMA_ENODRIVER:
            raise
        pytest.skip("needs a GPU (test_image_histories_against_the_host_simulated_engine runs this on CPU)")
    h = History(eng, oracle, seed, tmp_path)
    try:
        counts = h.run()
    finally:
        eng.close()
    if HOSTSIM:
        lib = C.CDLL(os.environ["FMA_B200_LIB"])
        for f in ("hostsim_live_mapped_bytes", "hostsim_live_handles", "hostsim_live_reservations"):
            getattr(lib, f).restype = C.c_ulonglong
            assert getattr(lib, f)() == 0, (f, h.fail_msg())
    assert _open_fds(tmp_path) == [], h.fail_msg()
    line = json.dumps({"seed": seed, **dict(sorted(counts.items()))})
    print(f"history {line}")
    if os.environ.get("FMA_HISTORY_LOG"):
        with open(os.environ["FMA_HISTORY_LOG"], "a") as f:
            f.write(line + "\n")


# ---- the host-simulated engine ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hostsim_lib(tmp_path_factory):
    if not os.path.exists("/usr/local/cuda/include/cuda_runtime.h"):
        pytest.skip("CUDA headers not installed")
    from tests.test_engine_hostsim import INC, SRCS

    out = str(tmp_path_factory.mktemp("hostsim_histories") / "libfma_b200_hostsim.so")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-shared", "-fPIC", "-fvisibility=hidden", *INC, *SRCS,
                           os.path.join(SIM, "hostsim_verify_kernels.cpp"), "-o", out, "-lpthread"])
    return out


def test_image_histories_against_the_host_simulated_engine(hostsim_lib, oracle, tmp_path):
    log = tmp_path / "histories.jsonl"
    env = dict(os.environ, FMA_B200_LIB=hostsim_lib, FMA_HOSTSIM="1", HOSTSIM_DEVICES="2", FMA_HISTORY_LOG=str(log))
    for key in ("FMA_RESIDENT_MIB", "FMA_NO_RING", "FMA_FILE_BUFFERED", "FMA_HOST_STORE_SHM"):
        env.pop(key, None)
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-rs", "-m", "gpu", "-p", "no:cacheprovider"],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-6000:]
    assert r.returncode == 0, tail
    assert " passed" in r.stdout and "failed" not in r.stdout and "SKIPPED" not in r.stdout, tail
    rows = [json.loads(x) for x in log.read_text().splitlines()]
    assert sorted(x["seed"] for x in rows) == SEEDS
    total = collections.Counter()
    for x in rows:
        seed = x.pop("seed")
        total.update(x)
        print(f"seed {seed}: " + ", ".join(f"{k} {v}" for k, v in x.items()))
    print("all seeds: " + ", ".join(f"{k} {v}" for k, v in sorted(total.items())))
    # every step kind, every tier and both image forms, a refusal and an injected failure of every operation
    need = ["sleep:host", "sleep:local", "sleep:file", "sleep:host_resident", "sleep:peer", "move:host", "move:local", "move:file", "move:peer",
            "prefetch", "verify", "damage", "damage:prefetched_wake", "wake:beside_prefetch", "free:asleep", "alloc", "wake:full", "wake:tags", "file_store",
            "host_release", "form:packed", "form:plain", "refusal:move", "refusal:prefetch", "refusal:verify", "inject:move",
            "inject:prefetch", "inject:verify", "inject:wake"]
    missing = [k for k in need if not total[k]]
    assert not missing, f"the default seeds never ran {missing}: {dict(total)}"
