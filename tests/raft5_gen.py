"""Seeded generator of raft5 programs whose external messages reach every handler of the model (DESIGN.md §3).

The bench and the older suites only ever send BOOT and CLIENT_CMD, so raft5's handlers only see what five correct peers
produce.  An external Send may carry any of the eight message types, from deadLetters, with any payload.  Every program
here comes from one integer seed and one family:

  "forged"  external messages of every type 1-8 with payloads drawn at each handler's edges (terms 0-3, 254, 255;
            indices 0-9 and 255; log terms and values 0 and 0xFF; the grant / ok / has bits both ways; junk in the bits
            the handlers ignore), ticks only with a non-zero payload (ordinary messages), Kill / Start / Partition /
            UnPartition between WaitQuiescence segments;
  "timer"   the same plus ELECTION_TICK / HEARTBEAT_TICK with p0 = p1 = 0, which equal a timer key: the lane engine
            hands such executions to the warp engine, and a HEARTBEAT_TICK sent to a booted actor meets Cancellable.cancel
            when that actor leads and steps down;
  "clean"   forged messages only, no timer keys and no Kill, few enough Sends per segment that the lane engine keeps
            every execution;
  "hardkill" the forged family with HardKill between segments (the warp engine's actor termination).

A raft5 actor with a booted peer always has a repeating ELECTION_TICK pending, so a segment that boots an actor never
quiesces: BOOTs go in the last segment (sometimes earlier, which leaves the later segments unreached), and the segments
before it run the forged messages against actors that have not booted yet.  One actor is sometimes never booted.  The
Sends of a program are distinct, so the lane engine accepts the program.
"""
import random

import demi_b200 as D

BOOT, CLIENT_CMD, ELECTION_TICK, REQUEST_VOTE, VOTE_REPLY, HEARTBEAT_TICK, APPEND_ENTRIES, APPEND_REPLY = range(1, 9)
TIMER_TYPES = (ELECTION_TICK, HEARTBEAT_TICK)
FAMILIES = ("forged", "timer", "clean", "hardkill")

TERMS = [0, 1, 2, 3, 254, 255]
INDICES = list(range(10)) + [255]
LOG_BYTES = [0, 1, 2, 3, 0x7F, 0x80, 0xFE, 0xFF]


class Program(object):
    def __init__(self, seed, family, events):
        self.seed, self.family, self.events = seed, family, events

    @property
    def timer_keyed(self):
        """The Sends that equal a timer key (type 3 or 6, p0 = p1 = 0)."""
        return [e for e in self.events if isinstance(e, D.Send) and e.type in TIMER_TYPES and e.p0 == 0 and e.p1 == 0]

    def __repr__(self):
        return "raft5_gen.Program(seed=%d, family=%r, %d events)" % (self.seed, self.family, len(self.events))


def _junk(rng, bits):
    return rng.getrandbits(bits) if rng.random() < 0.5 else 0


def payload(rng, ty, timer_keyed=False):
    """(p0, p1) of an external message of type `ty`: fields at the handlers' edges, junk in the bits they ignore."""
    t = rng.choice(TERMS)
    if ty == BOOT:
        return rng.choice([0x1F, 0, 0xFFFFFFFF, rng.getrandbits(32)]), _junk(rng, 32)
    if ty == CLIENT_CMD:
        return rng.choice([0, 1, 0x7F, 0x80, 0xFF, rng.getrandbits(32)]), _junk(rng, 32)
    if ty in TIMER_TYPES:
        if timer_keyed:
            return 0, 0
        p0, p1 = rng.choice([(rng.getrandbits(32), 0), (0, 1 + rng.getrandbits(31)), (t, _junk(rng, 32))])
        return (p0, p1) if (p0, p1) != (0, 0) else (1, 0)
    if ty == REQUEST_VOTE:
        li, lt = rng.choice(INDICES), rng.choice(LOG_BYTES + TERMS)
        return t | (li << 8) | (lt << 16) | (_junk(rng, 8) << 24), _junk(rng, 32)
    if ty == VOTE_REPLY:
        return t | (rng.getrandbits(1) << 8) | (_junk(rng, 23) << 9), _junk(rng, 32)
    if ty == APPEND_ENTRIES:
        prev, pt, lc = rng.choice(INDICES), rng.choice(LOG_BYTES + TERMS), rng.choice(INDICES)
        has, et, ev = rng.getrandbits(1), rng.choice(LOG_BYTES + TERMS), rng.choice(LOG_BYTES)
        return (t | (prev << 8) | (pt << 16) | (lc << 24),
                has | (_junk(rng, 7) << 1) | (et << 8) | (ev << 16) | (_junk(rng, 8) << 24))
    if ty == APPEND_REPLY:
        mi = rng.choice(INDICES)
        return t | (rng.getrandbits(1) << 8) | (_junk(rng, 7) << 9) | (mi << 16) | (_junk(rng, 8) << 24), _junk(rng, 32)
    raise ValueError(ty)


def generate(seed, family="forged"):
    assert family in FAMILIES
    rng = random.Random(seed * 4 + FAMILIES.index(family))
    seen = set()
    events = []

    def send(a, ty, timer_keyed=False):
        for _ in range(8):
            p0, p1 = payload(rng, ty, timer_keyed)
            if (a, ty, p0, p1) not in seen:
                seen.add((a, ty, p0, p1))
                events.append(D.Send(a, ty, p0, p1))
                return True
        return False

    def forged(n, types):
        for _ in range(n):
            send(rng.randrange(5), rng.choice(types))

    protocol = [t for t in range(1, 9) if t != BOOT]
    max_per_segment = 6 if family == "clean" else 10
    starts = list(range(5))
    rng.shuffle(starts)
    events += [D.Start(a) for a in starts]
    booted = [a for a in range(5)]
    if rng.random() < 0.35:
        booted.remove(rng.randrange(5))                              # one actor never booted
    n_segments = rng.randint(1, 3)
    boot_segment = n_segments - 1 if rng.random() < 0.85 else rng.randrange(n_segments)
    # timer family: a quarter of the programs keep their timer keys behind the booting segment, where no execution goes
    late_timers = family == "timer" and rng.random() < 0.25
    if late_timers:
        n_segments, boot_segment = max(n_segments, 2), 0
    killed = set()
    for seg in range(n_segments):
        if seg:                                                      # between segments: failures and the network
            for _ in range(rng.randint(0, 3)):
                k = rng.random()
                a, b = rng.randrange(5), rng.randrange(5)
                if family == "hardkill" and k < 0.3:
                    events.append(D.HardKill(a)); killed.add(a)
                elif family != "clean" and k < 0.45:
                    events.append(D.Kill(a)); killed.add(a)
                elif killed and k < 0.6:
                    a = sorted(killed)[rng.randrange(len(killed))]
                    events.append(D.Start(a)); killed.discard(a)     # a restart
                elif a != b and k < 0.85:
                    events.append(D.Partition(a, b))
                elif a != b:
                    events.append(D.UnPartition(a, b))
        n = rng.randint(1, max_per_segment - (len(booted) if seg == boot_segment else 0))
        if seg == boot_segment:
            order = list(booted)
            rng.shuffle(order)
            for a in order:                                          # BOOTs interleaved with the forged messages
                send(a, BOOT)
                forged(rng.randint(0, 1), protocol)
            if family == "timer" and not late_timers:
                send(rng.choice(booted), HEARTBEAT_TICK, timer_keyed=True)   # to an actor that may come to lead
                if rng.random() < 0.5:
                    send(rng.randrange(5), rng.choice(TIMER_TYPES), timer_keyed=True)
            if rng.random() < 0.5:
                send(rng.randrange(5), CLIENT_CMD)
        elif family == "timer" and (seg > boot_segment if late_timers else rng.random() < 0.5):
            send(rng.randrange(5), rng.choice(TIMER_TYPES), timer_keyed=True)
        forged(n, protocol)
        if family != "clean" and rng.random() < 0.3 and seg != n_segments - 1:
            events.append(D.Kill(rng.randrange(5)))                  # a Kill inside the segment, before its messages run
        events.append(D.WaitQuiescence())
    return Program(seed, family, events)


def corpus(n, family, base=0):
    return [generate(base + i, family) for i in range(n)]
