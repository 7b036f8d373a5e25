"""The wgmma GEMM's work schedule (make_tc_plan in wq_gemm.cu, TcSched in wq_gemm_shared.cuh), restated in Python.

A launch's tiles are its n-groups (128 output channels) times its k-tiles (64 k).  At most as many n-groups as SMs: S equal
k-slices per n-group, one CTA each.  More: each of the grid CTAs takes `rounds` whole n-groups, b + j * grid, and each of
the NR n-groups left over is cut in two at k-tile h: CTA b < NR runs the head [0, h) of n-group nfull + b first, CTA NR + b
runs the tail [h, KT) last, starting from the head's accumulators (h = 0: CTA b < NR runs it whole)."""
from dataclasses import dataclass

H100_SMS = 132
MAX_SPLIT = 6       # B2_GEMM_TC_MAX_SPLIT default


@dataclass
class Plan:
    NG: int
    KT: int
    grid: int
    rounds: int     # whole n-groups per CTA
    S: int          # k-slices per n-group (rounds == 0)
    h: int          # head length of a leftover n-group (0: not split)

    @property
    def nfull(self):
        return self.rounds * self.grid

    @property
    def NR(self):
        return self.NG - self.nfull

    @property
    def multi(self):
        return self.NG > self.grid

    def segments(self, b):
        """CTA b's work in walk order: (ng, kt0, kt1, part, parts, carry), carry 1 = head, 2 = tail."""
        if self.rounds == 0:
            ng, s = divmod(b, self.S)
            return [(ng, s * self.KT // self.S, (s + 1) * self.KT // self.S, s, self.S, 0)]
        out = []
        if b < self.NR:
            out.append((self.nfull + b, 0, self.h or self.KT, 0, 1, 1 if self.h else 0))
        out += [(j * self.grid + b, 0, self.KT, 0, 1, 0) for j in range(self.rounds)]
        if self.h and self.NR <= b < 2 * self.NR:
            out.append((self.nfull + b - self.NR, self.h, self.KT, 0, 1, 2))
        return out

    def tiles(self, b):
        return sum(s[2] - s[1] for s in self.segments(b))

    def max_tiles(self):
        return max(self.tiles(b) for b in range(self.grid))

    def workspace_bytes(self, rows=64):
        if self.S > 1:
            return self.NG * self.S * rows * 128 * 4 + 16
        if self.h:
            return self.NR * (256 * 32 + 64 * 4) * 4 + 16
        return 16


def plan(NG, KT, sms=H100_SMS, max_split=MAX_SPLIT, persist=True):
    max_split = max(1, max_split)
    if NG <= sms or not persist:
        S = max(1, min(sms // NG, KT // 4, max_split))
        return Plan(NG, KT, NG * S, 0, S, 0)
    NR = NG % sms
    h = KT // 2 // 4 * 4 if NR > 0 and max_split > 1 and 2 * NR <= sms else 0
    return Plan(NG, KT, sms, NG // sms, 1, h)
