"""Host-side external-event program generator: the reference's Fuzzer, seeded.

Mirrors src/main/scala/verification/fuzzing/Fuzzer.scala:24-194 (`FuzzerWeights`, `Fuzzer.generateNextEvent`,
`generateFuzzTest`, `reset`) and the `RandomizedHashSet` it draws from (schedulers/Util.scala:110-185).
The reference seeds the fuzzer and each of its three sets from `System.currentTimeMillis` (Fuzzer.scala:67-68,
Util.scala:110); here they all take an explicit seed (what constructions within one millisecond give), so a
fuzz test is reproducible.  `java.util.Random` is restated from the Java SE specification.
"""
from . import events as E


class JavaRandom(object):
    MULT, ADD, MASK = 0x5DEECE66D, 0xB, (1 << 48) - 1

    def __init__(self, seed):
        self.s = (seed ^ self.MULT) & self.MASK

    def next(self, bits):
        self.s = (self.s * self.MULT + self.ADD) & self.MASK
        v = self.s >> (48 - bits)
        return v - (1 << bits) if bits == 32 and v >= (1 << 31) else v

    def nextInt(self, bound=None):
        if bound is None:
            return self.next(32)
        if bound <= 0:
            raise ValueError("bound must be positive")
        r = self.next(31)
        m = bound - 1
        if bound & m == 0:
            return (bound * r) >> 31
        u = r
        while True:
            r = u % bound
            if u - r + m < (1 << 31):
                return r
            u = self.next(31)

    def nextDouble(self):
        return ((self.next(26) << 27) + self.next(27)) * (1.0 / (1 << 53))


class RandomizedHashSet(object):
    """schedulers/Util.scala:110-185: O(1) insert / removeRandomElement over an array."""

    def __init__(self, seed):
        self.arr = []
        self.rand = JavaRandom(seed)

    def insert(self, v):
        self.arr.append(v)

    def isEmpty(self):
        return not self.arr

    def removeRandomElement(self):
        i = self.rand.nextInt(len(self.arr))
        v = self.arr[i]
        self.arr[i] = self.arr[-1]
        self.arr.pop()
        return v

    def getRandomElement(self):
        return self.arr[self.rand.nextInt(len(self.arr))]


class FuzzerWeights(object):
    """Fuzzer.scala:24-58."""

    def __init__(self, kill=0.01, send=0.3, wait_quiescence=0.1, partition=0.1, unpartition=0.1):
        self.allWeights = [kill, send, partition, unpartition]
        self.wait_quiescence = wait_quiescence
        self.totalMass = sum(self.allWeights) + wait_quiescence
        self.eventTypes = ["Kill", "Send", "Partition", "UnPartition"]

    def getNextEventType(self, r):
        scaled = r * self.totalMass
        current = 0.0
        for w, t in zip(self.allWeights, self.eventTypes):
            current = current + w
            if scaled < current:
                return t
        return None            # WaitQuiescence


def fuzzer_config(fuzzer):
    """The demi_fuzzer_config of a Fuzzer whose message_gen is a ClientCommandGenerator (what the C ABI generates)."""
    from . import _native as N
    if not isinstance(fuzzer.message_gen, ClientCommandGenerator):
        raise ValueError("the C ABI's Fuzzer generates Send(random alive actor, send_type, counter) only")
    w = fuzzer.weights
    kill, send, partition, unpartition = w.allWeights
    return N.FuzzerConfig(kill, send, w.wait_quiescence, partition, unpartition, fuzzer.num_events, fuzzer.message_gen.msg_type)


class ClientCommandGenerator(object):
    """A MessageGenerator (Fuzzer.scala:8-10): Send(random alive actor, type, counter)."""

    def __init__(self, msg_type=2):
        self.msg_type, self.counter = msg_type, 0

    def generateMessage(self, aliveActors):
        self.counter += 1
        return E.Send(aliveActors.getRandomElement(), self.msg_type, self.counter)


class Fuzzer(object):
    """Fuzzer(num_events, weights, message_gen, prefix, postfix) — Fuzzer.scala:61-194."""

    def __init__(self, num_events, weights, message_gen, prefix, postfix=(), seed=0):
        self.num_events, self.weights, self.message_gen = num_events, weights, message_gen
        self.prefix, self.postfix = list(prefix), list(postfix)
        self.seed = seed
        self.nodes = [e.a for e in self.prefix if isinstance(e, E.Start)]
        self.reset()

    def reset(self):                                       # :176-193
        self.rand = JavaRandom(self.seed)
        self.currentlyAlive = RandomizedHashSet(self.seed)
        for n in self.nodes:
            self.currentlyAlive.insert(n)
        self.currentlyPartitioned = RandomizedHashSet(self.seed)
        self.currentlyUnpartitioned = RandomizedHashSet(self.seed)
        for i in range(len(self.nodes)):
            for j in range(i + 1, len(self.nodes)):
                self.currentlyUnpartitioned.insert((self.nodes[i], self.nodes[j]))

    def generateNextEvent(self):                           # :84-121
        while True:
            t = self.weights.getNextEventType(self.rand.nextDouble())
            if t is None:
                return E.WaitQuiescence()
            if t == "Kill":
                if self.currentlyAlive.isEmpty():
                    return None
                return E.Kill(self.currentlyAlive.removeRandomElement())
            if t == "Send":
                return self.message_gen.generateMessage(self.currentlyAlive)
            if t == "Partition":
                if self.currentlyUnpartitioned.isEmpty():
                    continue                               # "Try again..."
                a, b = self.currentlyUnpartitioned.removeRandomElement()
                self.currentlyPartitioned.insert((a, b))
                return E.Partition(a, b)
            if self.currentlyPartitioned.isEmpty():
                continue
            a, b = self.currentlyPartitioned.removeRandomElement()
            self.currentlyUnpartitioned.insert((a, b))
            return E.UnPartition(a, b)

    def generateFuzzTest(self):                            # :123-174
        self.reset()
        test = list(self.prefix)
        just_wq = bool(test) and isinstance(test[-1], E.WaitQuiescence)
        for _ in range(self.num_events):
            ev = self.generateNextEvent()
            while isinstance(ev, E.WaitQuiescence) and just_wq:      # no two WaitQuiescence in a row
                ev = self.generateNextEvent()
            if ev is None:
                return test
            just_wq = isinstance(ev, E.WaitQuiescence)
            test.append(ev)
        test += self.postfix
        if test and not isinstance(test[-1], E.WaitQuiescence):
            test.append(E.WaitQuiescence())
        for a, b in zip(test, test[1:]):
            assert not (isinstance(a, E.WaitQuiescence) and isinstance(b, E.WaitQuiescence))
        return test
