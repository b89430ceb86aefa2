"""Fungible clocks (minification/wildcard_minimization/): an independent restatement of WildCardMatch inside
STSScheduler, ClockClusterizer, ClockClusterIterator, OneAtATimeIterator and WildcardMinimizer.doMinimize, on top of
the STSScheduler restatement of micro_oracle.py.  Message selectors are real closures over message objects, as in the
Scala; nothing here sees the engine's packed clock rules or its per-delivery mode table."""
from micro_oracle import STSReplay


class FingerprintFactory(object):
    """The two FingerprintFactory hooks the clock clusterizer consults (MessageFingerprints.scala:26-31): closures over
    a message, as in the reference.  Defaults: no clock, nothing increments it (:28, :31)."""

    def __init__(self, getLogicalClock=None, causesClockIncrement=None):
        self.getLogicalClock = getLogicalClock or (lambda msg: None)
        self.causesClockIncrement = causesClockIncrement or (lambda msg: False)


class WildCardMatch(object):
    """WildCardMatch(msgSelector: (Seq[Any], backtrackSetter) => Option[Int], name)."""

    def __init__(self, msgSelector, name):
        self.msgSelector, self.name = msgSelector, name


class BackTrackStrategy(object):                  # AmbiguityResolutionStrategies.scala:44-75
    def resolve(self, msgSelector, pending, backtrackSetter):
        matching = [(msg, i) for i, msg in enumerate(pending) if msgSelector(msg)]
        if matching:
            # the backtrack points it sets go to backtrackSetter, which STSSched passes as a no-op
            return matching[0][1]
        return None


class LastOnlyStrategy(object):                   # :109-117
    def resolve(self, msgSelector, pending, backtrackSetter):
        matching = [(msg, i) for i, msg in enumerate(pending) if msgSelector(msg)]
        return matching[-1][1] if matching else None


class WildcardSTSReplay(STSReplay):
    """STSReplay over a trace whose MsgEvents may carry a WildCardMatch: messagePending (STSScheduler.scala:381-403),
    the WildCardMatch case of schedule_new_message (:696-708), and ignoreAbsentCallback (:529)."""

    def __init__(self, *a, **kw):
        STSReplay.__init__(self, *a, **kw)
        self.ignoredAbsentIndices = []

    def message_pending(self, snd, rcv, msg):
        if not isinstance(msg, WildCardMatch):
            return STSReplay.message_pending(self, snd, rcv, msg)
        self.send_external_messages()
        h = self.pending.get((snd, rcv))
        if h is None:
            return False
        flat = sorted((t for q in h.values() for t in q), key=lambda t: t[0])   # hash.values.flatten.sortBy(_.id)
        if msg.msgSelector([m for _, m in flat], lambda i: None) is None:
            return False
        return rcv not in self.blockedActors

    def advance_replay(self):                    # :405-559, the ignore branch reporting its trace index
        while self.traceIdx < len(self.trace):
            e = self.trace[self.traceIdx]
            k = e[0]
            if k == "Spawn":
                self.events.append(e)
                self.inaccessible.discard(e[1]); self.killed.discard(e[1]); self.blockedActors.discard(e[1])
            elif k == "Kill":
                self.events.append(e)
                self.killed.add(e[1]); self.inaccessible.add(e[1])
            elif k == "Partition":
                self.events.append(e); self.partitioned.add((e[1], e[2]))
            elif k == "UnPartition":
                self.events.append(e); self.partitioned.discard((e[1], e[2]))
            elif k == "MsgSend":
                if self.is_external(e[3]):
                    self.enqueuedExternalMessages.append(e[3])
                    self.messagesToSend.append((None, e[2], e[3]))
            elif k == "MsgEvent":
                if self.message_pending(e[1], e[2], e[3]):
                    return
                self.ignored += 1
                self.ignoredAbsentIndices.append(self.traceIdx)      # ignoreAbsentCallback(event_orchestrator.traceIdx)
            elif k in ("Quiescence", "BeginWaitQuiescence"):
                self.events.append(e)
            self.traceIdx += 1

    def schedule_new_message(self):
        self.send_external_messages()
        self.advance_replay()
        self.send_external_messages()
        if self.traceIdx >= len(self.trace):
            return None
        _, snd, rcv, msg, _, _ = self.trace[self.traceIdx]
        if not isinstance(msg, WildCardMatch):
            return self._deliver(snd, rcv, msg)
        h = self.pending[(snd, rcv)]
        pendingKeyValues = sorted(h.items(), key=lambda kv: kv[1][0][0])   # sortBy(keyValue => keyValue._2.head.id)
        pendingValues = [q[0][1] for _, q in pendingKeyValues]
        selectedMsgIdx = msg.msgSelector(pendingValues, lambda i: None)
        return self._deliver(snd, rcv, pendingKeyValues[selectedMsgIdx][0])

    def _deliver(self, snd, rcv, fingerprint):   # dequeue the head of the chosen queue (:710-750)
        h = self.pending[(snd, rcv)]
        q = h[fingerprint]
        uniq, m = q.pop(0)
        if not q:
            del h[fingerprint]
            if not h:
                del self.pending[(snd, rcv)]
        self.events.append(("MsgEvent", snd, rcv, m, uniq, 0))
        self.traceIdx += 1
        self.delivered += 1
        return (uniq, None, snd, rcv, m)


ALL_TIMERS_FIRST_ITR = "ALL_TIMERS_FIRST_ITR"


class ClockClusterIterator(object):              # ClockClusterizer.scala:138-228
    def __init__(self, originalTrace, fingerprinter):
        self.originalTrace, self.fingerprinter = originalTrace, fingerprinter
        self.allIds = set(e[4] for e in originalTrace if e[0] == "MsgEvent" and
                          not fingerprinter.causesClockIncrement(e[3]) and fingerprinter.getLogicalClock(e[3]) is not None)
        self.firstClusterRemoval = True
        self.nextClockToRemove = -1
        self.blacklist = set()
        self.clocks = []
        self.clocks = self.computeRemainingClocks()

    def computeRemainingClocks(self):
        lowest = self.clocks[0] if self.clocks else 0                 # clocks.headOption.getOrElse(0)
        s = set()
        for e in self.originalTrace:
            if e[0] == "MsgEvent" and e[4] not in self.blacklist:
                c = self.fingerprinter.getLogicalClock(e[3])
                if c is not None:
                    s.add(c)
        out = sorted(s)
        while out and out[0] < lowest:                               # dropWhile(c => c < lowest)
            out.pop(0)
        return out

    def _current(self):
        currentClockToRemove = -1 if self.firstClusterRemoval else self.nextClockToRemove
        out = set()
        for e in self.originalTrace:
            if e[0] != "MsgEvent":
                continue
            msg, uid = e[3], e[4]
            if self.fingerprinter.causesClockIncrement(msg):
                continue
            clock = self.fingerprinter.getLogicalClock(msg)
            if clock is None:
                out.add(uid)
            elif not (clock == currentClockToRemove or uid in self.blacklist):
                out.add(uid)
        return out

    def next(self):
        if self.firstClusterRemoval:
            ret = self._current()
            self.firstClusterRemoval = False
            return ret
        self.nextClockToRemove = self.clocks[0]
        ret = self._current()
        self.clocks = self.clocks[1:]
        return ret

    def hasNext(self):
        return self.firstClusterRemoval or bool(self.clocks)

    def producedViolation(self, previouslyIncluded, ignoredAbsents):
        self.blacklist = self.blacklist | self.inverse(previouslyIncluded)
        if ignoredAbsents:
            self.blacklist = self.blacklist | (self.allIds & ignoredAbsents)
            self.clocks = self.computeRemainingClocks()

    def inverse(self, toInclude):
        return self.allIds - toInclude


class OneAtATimeIterator(object):                # ClockClusterizer.scala:230-290
    @staticmethod
    def fromTrace(originalTrace, fingerprinter):
        return OneAtATimeIterator(set(e[4] for e in originalTrace
                                      if e[0] == "MsgEvent" and fingerprinter.causesClockIncrement(e[3])))

    def __init__(self, all_):
        self.all = all_
        self.toRemove = sorted(all_)
        self.first = True
        self.blacklist = set()

    def _current(self):
        if self.first:
            return self.all - self.blacklist
        return (self.all - {self.toRemove[0]}) - self.blacklist

    def next(self):
        ret = self._current()
        if self.first:
            self.first = False
        else:
            self.toRemove = self.toRemove[1:]
        return ret

    def hasNext(self):
        return self.first or bool(self.toRemove)

    def producedViolation(self, previouslyIncluded, ignoredAbsents):
        self.blacklist = self.blacklist | self.inverse(previouslyIncluded) | (self.all & ignoredAbsents)

    def reset(self):
        self.toRemove = sorted(self.all - self.blacklist)
        self.first = True

    def inverse(self, toInclude):
        return self.all - toInclude


class ClockClusterizer(object):                  # ClockClusterizer.scala:39-134, skipClockClusters = false
    def __init__(self, originalTrace, fingerprinter, resolutionStrategy, is_external, aggressiveness=ALL_TIMERS_FIRST_ITR):
        self.originalTrace, self.fingerprinter, self.resolutionStrategy = originalTrace, fingerprinter, resolutionStrategy
        self.is_external, self.aggressiveness = is_external, aggressiveness
        self.clusterIterator = ClockClusterIterator(originalTrace, fingerprinter)
        assert self.clusterIterator.hasNext()
        self.currentCluster = self.clusterIterator.next()
        self.tryingFirstCluster = True
        self.timerIterator = OneAtATimeIterator.fromTrace(originalTrace, fingerprinter)
        self.currentTimers = set()

    def getNextTrace(self, violationReproducedLastRun, ignoredAbsentIds):
        if violationReproducedLastRun:
            self.timerIterator.producedViolation(self.currentTimers, ignoredAbsentIds)
            self.clusterIterator.producedViolation(self.currentCluster, ignoredAbsentIds)
        if (not self.timerIterator.hasNext() or
                (self.aggressiveness == ALL_TIMERS_FIRST_ITR and violationReproducedLastRun and not self.tryingFirstCluster)):
            self.tryingFirstCluster = False
            if not self.clusterIterator.hasNext():
                return None
            self.timerIterator.reset()
            self.currentCluster = self.clusterIterator.next()
        assert self.timerIterator.hasNext()
        self.currentTimers = self.timerIterator.next()
        return self.wildcarded(self.currentTimers, self.currentCluster)

    def wildcarded(self, currentTimers, currentCluster):     # :100-133, the trace for the current id sets
        fp = self.fingerprinter
        events = []
        for e in self.originalTrace:
            if e[0] != "MsgEvent":
                events.append(e)
                continue
            _, snd, rcv, msg, uid, node = e
            if self.is_external(msg):                                 # EventTypes.isExternal(u)
                events.append(e)
            elif uid in currentTimers:
                def timerSelector(lst, backtrackSetter):              # timers bypass the resolutionStrategy
                    idx = next((i for i, m in enumerate(lst) if fp.causesClockIncrement(m)), -1)
                    return None if idx == -1 else idx
                events.append(("MsgEvent", snd, rcv, WildCardMatch(timerSelector, "CausesClockIncrement"), uid, node))
            elif uid in currentCluster:
                classTag = msg[0]                                     # ClassTag(msg.getClass): the message type

                def messageFilter(pendingMsg, classTag=classTag):
                    return pendingMsg[0] == classTag

                def selector(lst, backtrackSetter, messageFilter=messageFilter):
                    return self.resolutionStrategy.resolve(messageFilter, lst, backtrackSetter)
                events.append(("MsgEvent", snd, rcv, WildCardMatch(selector, str(classTag)), uid, node))
        return events


class WildcardMinimizer(object):
    """WildcardMinimizer.minimize / doMinimize (WildcardMinimizer.scala:133-241), testScheduler = STSSched,
    ClockClusterizer, ALL_TIMERS_FIRST_ITR.  `test(nextTrace)` runs one STSScheduler.test and returns the
    WildcardSTSReplay with its verdict in `.violation`; `project(nextTrace)` is nextTrace.subsequenceIntersection(mcs,
    filterKnownAbsents)."""

    def __init__(self, trace, fingerprinter, resolutionStrategy, is_external, test, project):
        self.trace, self.fingerprinter, self.resolutionStrategy = trace, fingerprinter, resolutionStrategy or BackTrackStrategy()
        self.is_external, self.test, self.project = is_external, test, project
        self.total_replays = 0
        self.internal_sizes = []
        self.tests = []                          # (nextTrace, verdict) in order, for the known-answer tests

    def minimize(self):
        count = lambda tr: sum(1 for e in tr if e[0] == "MsgEvent")     # RunnerUtils.countMsgEvents
        clusterizer = ClockClusterizer(self.trace, self.fingerprinter, self.resolutionStrategy, self.is_external)
        minTrace = self.trace
        nextTrace = clusterizer.getNextTrace(False, set())
        while nextTrace is not None:
            self.total_replays += 1                                      # STSScheduler.test: increment_replays
            sts = self.test(nextTrace)
            ret = sts.events if sts.violation is not None else None
            self.tests.append((nextTrace, ret is not None))
            self.internal_sizes.append(count(minTrace))                  # record_internal_size :210-212
            ignoredAbsentIds = set()
            if ret is not None:
                if len(ret) <= len(minTrace):
                    minTrace = ret
                adjustedTrace = self.project(nextTrace)
                for i in sts.ignoredAbsentIndices:
                    ignoredAbsentIds.add(adjustedTrace[i][4])
            nextTrace = clusterizer.getNextTrace(ret is not None, ignoredAbsentIds)
        self.internal_sizes.append(count(minTrace))                      # fencepost :184
        return minTrace
