"""A second, independently written restatement of the reference's RandomScheduler path — in Python, object for object as
the Scala reads (actor names are strings, messages are tuples, the structures are the reference's own: RandomizedHashSet,
DepTracker, EventOrchestrator, the ExternalEventInjector queue, Instrumenter's timer maps) — plus DDMin.ddmin2.

It shares NOTHING with oracle/*.c or include/*.h: no headers, no hash functions, no capacity rules; the actors are
written a third time from DESIGN.md §3.  tests/test_micro_oracle.py cross-checks it against liboracle.so event by
event on 10^4 seeds, so an error in the C oracle's reading of the Scala has to be made twice, independently, to pass.
Test infrastructure only.

Reference (src/main/scala/verification/): schedulers/RandomScheduler.scala:226-321, :352-485, :525-559, :635-697;
schedulers/Util.scala:110-185, :470-489; DepTracker.scala:82-135; schedulers/EventOrchestrator.scala:132-241, :314-351;
schedulers/ExternalEventInjector.scala:258-365, :367-441, :541-580, :601-610; Instrumenter.scala:159-168, :1000-1016,
:1090-1096, :1145-1200; minification/DeltaDebugging.scala:27-109; minification/Util.scala:9-37, :197-265.
"""

DEADLETTERS = "deadLetters"
INJECTED = "injected"                            # messagesToSend's sender of an external Send (deadLetters on the wire)


class JavaRandom(object):                       # java.util.Random, Java SE specification
    def __init__(self, seed):
        self.seed = (seed ^ 0x5DEECE66D) & ((1 << 48) - 1)

    def _next(self, bits):
        self.seed = (self.seed * 0x5DEECE66D + 0xB) & ((1 << 48) - 1)
        r = self.seed >> (48 - bits)
        return r - (1 << 32) if r >= (1 << 31) and bits == 32 else r

    def nextInt(self, bound):
        r = self._next(31)
        m = bound - 1
        if (bound & m) == 0:
            return (bound * r) >> 31
        u = r
        while True:
            r = u % bound
            if u - r + m <= 0x7FFFFFFF:          # no int overflow
                return r
            u = self._next(31)


class RandomizedHashSet(object):                # schedulers/Util.scala:110-185
    def __init__(self, seed):
        self.arr = []                            # ArrayBuffer[(E, Int)]
        self.hash = {}                           # (E, counter) -> index
        self.rand = JavaRandom(seed)

    def insert(self, value):
        c = 0
        while (id(value), c) in self.hash:       # the uniqueness counter only matters for equal tuples
            c += 1
        t = (value, c)
        self.hash[(id(value), c)] = len(self.arr)
        self.arr.append(t)

    def remove(self, t):
        i = self.hash[(id(t[0]), t[1])]
        d = self.arr[-1]
        self.arr[i] = d
        self.hash[(id(d[0]), d[1])] = i
        self.arr.pop()                           # arr.dropRight(1)
        del self.hash[(id(t[0]), t[1])]

    def removeRandomElement(self):
        idx = self.rand.nextInt(len(self.arr))
        v = self.arr[idx]
        self.remove(v)
        return v[0]

    def isEmpty(self):
        return not self.arr


class Unique(object):
    def __init__(self, event, uid):
        self.event, self.id = event, uid


class DepTracker(object):                        # DepTracker.scala:27-135
    def __init__(self):
        self.root = Unique(("null", "null", None), 0)
        self.next_id = 1
        self.parent_of = {0: 0}
        self.children = {0: []}                  # inNeighbors of a node, in creation order
        self.parentEvent = self.root
        self.lastQuiescence = self.root          # noopWaitQuiescence: the root stands for every quiescence (:139-150)

    def _getMessage(self, snd, rcv, msg):        # :82-109
        for c in self.children[self.parentEvent.id]:
            s, r, m = c.event
            if s == snd and r == rcv and m == msg:
                return c, False
        u = Unique((snd, rcv, msg), self.next_id)
        self.next_id += 1
        return u, True

    def reportNewlyEnabled(self, snd, rcv, msg):  # :126-130 with addNodeAndEdge :111-116
        child, new = self._getMessage(snd, rcv, msg)
        if new:
            self.parent_of[child.id] = self.parentEvent.id
            self.children[self.parentEvent.id].append(child)
            self.children[child.id] = []
        return child

    def reportNewlyEnabledExternal(self, snd, rcv, msg):   # :119-122
        self.parentEvent = self.lastQuiescence
        return self.reportNewlyEnabled(snd, rcv, msg)

    def reportNewlyDelivered(self, u):           # :132-135
        self.parentEvent = u


class Execution(object):
    """One RandomScheduler.explore(trace) with max_executions = 1, FullyRandom(seed), checkpointing off."""

    def __init__(self, actors, externals, seed, max_messages, invariant_check_interval, invariant, external_filter,
                 blocked=(), looking_for=None, user_filter=None, fresh_actor=None, ignore_timers=False):
        self.userDefinedFilter = user_filter or (lambda snd, rcv, msg: True)      # FullyRandom ctor arg (:636)
        self.fresh_actor = fresh_actor                                             # name -> new instance (HardKill + Start)
        self.dead = set()
        self.actors = actors                     # name -> actor object with receive(ctx, sender, msg)
        self.externals = externals               # [("Start", name) | ("Kill", name) | ("Send", name, msg) | ("Partition", a, b) | ...]
        self.pendingEvents = RandomizedHashSet(seed)
        self.maxMessages = max_messages if max_messages >= 0 else 0x7FFFFFFF
        self.interval = invariant_check_interval
        self.invariant = invariant
        self.is_external = external_filter
        self.blockedActors = set(blocked)
        self.ignoreTimers = ignore_timers        # SchedulerConfig.ignoreTimers
        self.lookingFor = looking_for
        self.depTracker = DepTracker()
        # ExternalEventInjector
        self.messagesToSend = []                 # (sender, None for a timer or INJECTED for an external Send, receiver, msg)
        self.injecting = False                   # event_produced is handling an injected Send
        self.enqueuedExternalMessages = []       # MultiSet
        # RandomScheduler
        self.justScheduledTimers = set()
        self.timersToResend = []
        self.messagesScheduledSoFar = 0
        self.violationFound = None
        # EventOrchestrator
        self.events = []                         # the EventTrace
        self.traceIdx = 0
        self.killed, self.inaccessible, self.partitioned = set(), set(actors), set()   # populateActorSystem isolates everyone
        # Instrumenter
        self.timerToCancellable = {}             # (rcv, msg) -> ongoing?
        self.timersCancelledThisStep = set()
        self.uniq_counter = 0
        self.max_pending = 0

    # ---- EventOrchestrator
    def crosses_partition(self, snd, rcv):       # :345-351
        if snd == rcv and snd not in self.killed:
            return False
        return ((snd, rcv) in self.partitioned or (rcv, snd) in self.partitioned or rcv in self.inaccessible or
                snd in self.inaccessible)

    def inject_until_quiescence(self):           # :132-189
        loop = True
        while loop and self.traceIdx < len(self.externals):
            e = self.externals[self.traceIdx]
            if e[0] == "Start":
                self.events.append(("Spawn", e[1]))
                self.inaccessible.discard(e[1]); self.killed.discard(e[1]); self.dead.discard(e[1])
                self.blockedActors.discard(e[1])
            elif e[0] == "Kill":
                self.events.append(("Kill", e[1]))
                self.killed.add(e[1]); self.inaccessible.add(e[1])
            elif e[0] == "HardKill":                                 # trigger_hard_kill (EventOrchestrator.scala:243-310)
                self.events.append(("HardKill", e[1]))
                for t in list(self.pendingEvents.arr):               # actorTerminated -> FullyRandom.removeAll (:686-696)
                    if t[0][3] == e[1]:
                        self.pendingEvents.remove(t)
                self.blockedActors.discard(e[1])
                for key in [k for k in self.timerToCancellable if k[0] == e[1]]:
                    del self.timerToCancellable[key]
                self.killed.add(e[1]); self.inaccessible.add(e[1]); self.dead.add(e[1])
                self.actors[e[1]] = self.fresh_actor(e[1])
            elif e[0] == "Send":
                self.enqueuedExternalMessages.append(e[2])           # enqueue_message :258-268
                self.messagesToSend.append((INJECTED, e[1], e[2]))
            elif e[0] == "Partition":
                self.events.append(("Partition", e[1], e[2])); self.partitioned.add((e[1], e[2]))
            elif e[0] == "UnPartition":
                self.events.append(("UnPartition", e[1], e[2])); self.partitioned.discard((e[1], e[2]))
            elif e[0] == "WaitQuiescence":
                self.events.append(("BeginWaitQuiescence",))
                loop = False
            self.traceIdx += 1

    # ---- Instrumenter: `!`, timers
    def tell(self, sender, rcv, msg):            # aroundDispatch :1033-1108
        if rcv not in self.actors:                                   # receiverIsAlive (Instrumenter.scala:397-401)
            return                                                   # "Dropping message to non-existent receiver"
        if (rcv, msg) in self.timersCancelledThisStep:               # :1090-1096
            self.timersCancelledThisStep.discard((rcv, msg))
            return
        self.event_produced(sender, rcv, msg)

    def registerCancellable(self, ongoing, rcv, msg):                # :1145-1174
        if (rcv, msg) in self.timerToCancellable:
            return                                                   # "Non-unique timer"
        self.timerToCancellable[(rcv, msg)] = ongoing
        self.handleTick(rcv, msg)

    def handleTick(self, rcv, msg):              # :1185-1200
        ongoing = self.timerToCancellable[(rcv, msg)]
        self.enqueue_timer(rcv, msg)
        if not ongoing:
            del self.timerToCancellable[(rcv, msg)]                  # removeCancellable

    def cancelTimer(self, rcv, msg):             # :159-168
        self.timersCancelledThisStep.add((rcv, msg))
        self.timerToCancellable.pop((rcv, msg), None)
        self.notify_timer_cancel(rcv, msg)

    # ---- RandomScheduler
    def event_produced(self, snd, rcv, msg):     # :274-321
        self.uniq_counter += 1
        uniq = self.uniq_counter & 0xFFFF                            # Uniq ids are 16-bit and wrap (DESIGN.md §2)
        is_timer = False
        # handle_event_produced :504-507 asks enqueuedExternalMessages.contains(msg); this project classifies a message
        # by where it came from, an injected Send (DESIGN.md §3, raft5)
        if self.injecting:
            unique = self.depTracker.reportNewlyEnabledExternal(snd, rcv, msg)
            self.pendingEvents.insert((uniq, unique, snd, rcv, msg))
        else:
            if snd == DEADLETTERS:
                is_timer = True
            unique = self.depTracker.reportNewlyEnabled(snd, rcv, msg)
            if not self.crosses_partition(snd, rcv):
                self.pendingEvents.insert((uniq, unique, snd, rcv, msg))
        self.max_pending = max(self.max_pending, len(self.pendingEvents.arr))
        self.events.append(("MsgSend", "Timer" if is_timer else snd, rcv, msg, uniq, unique.id))

    def handle_timer(self, rcv, msg):            # ExternalEventInjector :282-297
        if self.ignoreTimers:                    # the one place the reference reads ignoreTimers (:283-285)
            return
        self.messagesToSend.append((None, rcv, msg))

    def enqueue_timer(self, rcv, msg):           # :549-559
        if (rcv, msg) in self.justScheduledTimers:
            self.timersToResend.append((rcv, msg))
            return
        self.handle_timer(rcv, msg)

    def notify_timer_cancel(self, rcv, msg):     # :525-534 + handle_timer_cancel (ExternalEventInjector :601-610)
        for i, (s, r, m) in enumerate(self.messagesToSend):
            if r == rcv and m == msg:
                del self.messagesToSend[i]
                return
        for t in self.pendingEvents.arr:         # FullyRandom.remove :653-664
            _, _, s, r, m = t[0]
            if s == DEADLETTERS and r == rcv and m == msg:
                self.pendingEvents.remove(t)
                return

    def send_external_messages(self):            # ExternalEventInjector :306-365
        queue, self.messagesToSend = self.messagesToSend, []
        for sender, rcv, msg in queue:
            if rcv in self.dead:                                     # "Dropping message to non-existent receiver" (:343-346)
                continue
            self.injecting = sender is INJECTED
            self.tell(DEADLETTERS if sender in (None, INJECTED) else sender, rcv, msg)
            self.injecting = False

    def violationMatches(self, v):               # :138-154
        if v is None:
            return None
        if self.lookingFor is None or v == self.lookingFor:
            return v
        return None

    def schedule_new_message(self):              # :352-485
        if self.violationFound is not None:
            return None
        if self.messagesScheduledSoFar > self.maxMessages:
            self.traceIdx = len(self.externals)                      # finish_early
            return None
        if self.interval > 0 and self.messagesScheduledSoFar % self.interval == 0 and self.messagesScheduledSoFar != 0:
            # lastCheckpoint stays 0 without checkpointing, so the guard `lastCheckpoint != n` is `n != 0`
            self.violationFound = self.violationMatches(self.invariant(self.actors))
            if self.violationFound is not None:
                return None
        self.send_external_messages()
        e = self.pick_non_blocked()
        if e is None:
            return None
        uniq, unique, snd, rcv, msg = e
        self.messagesScheduledSoFar += 1
        self.events.append(("MsgEvent", snd, rcv, msg, uniq, unique.id))
        self.depTracker.reportNewlyDelivered(unique)
        if (rcv, msg) in self.timerToCancellable:                    # updateRepeatingTimer :405-421
            self.justScheduledTimers.add((rcv, msg))
        else:
            for r, t in self.timersToResend:
                self.handle_timer(r, t)
            self.timersToResend = []
            self.justScheduledTimers.clear()
        return e

    def pick_non_blocked(self):                  # find_non_blocked_message (Util.scala:470-489) over the strategy
        if self.pendingEvents.isEmpty():
            return None
        blocked = []
        e = self.strategy_removeRandomElement()
        while e[3] in self.blockedActors:
            blocked.append(e)
            if self.pendingEvents.isEmpty():
                for b in blocked:
                    self.pendingEvents.insert(b)
                return None
            e = self.strategy_removeRandomElement()
        for b in blocked:
            self.pendingEvents.insert(b)
        return e

    def strategy_removeRandomElement(self):      # FullyRandom.removeRandomElement (:666-684), as written
        ret = self.pendingEvents.removeRandomElement()
        rejected = []
        while len(self.pendingEvents.arr) > 1 and not self.userDefinedFilter(ret[2], ret[3], ret[4]):
            rejected.append(ret)
            ret = self.pendingEvents.removeRandomElement()
        for r in rejected:
            self.pendingEvents.insert(r)
        return ret

    def dispatch_new_message(self, e):           # Instrumenter :913-1017
        _, _, snd, rcv, msg = e
        if self.timerToCancellable.get((rcv, msg)):                  # a repeating timer is re-armed right after the hand-off
            self.handleTick(rcv, msg)
        self.actors[rcv].receive(Context(self, rcv), snd, msg)

    def run(self):
        while True:                              # execute_trace / advanceTrace / handle_quiescence
            self.inject_until_quiescence()
            while True:
                e = self.schedule_new_message()
                if e is None:
                    break
                self.dispatch_new_message(e)
            if self.violationFound is not None:  # notify_quiescence :487-500
                break
            if self.traceIdx < len(self.externals):
                self.events.append(("Quiescence",))
                continue
            break
        if self.violationFound is None and self.messagesScheduledSoFar <= self.maxMessages:   # explore :256 + checkIfBugFound
            self.violationFound = self.violationMatches(self.invariant(self.actors))
        return self.violationFound


class SrcDstFifoExecution(Execution):
    """RandomScheduler over the SrcDstFIFO strategy (RandomScheduler.scala:702-870): one FIFO per (src, dst) pair, timers
    and externals in a FullyRandom of their own.  The reference seeds both generators from the clock; here both are
    java.util.Random(seed), the convention DESIGN.md states for the `seed parameter added` to the strategy."""

    def __init__(self, *a, **kw):
        Execution.__init__(self, *a, **kw)
        seed = a[2]
        self.timersAndExternals = self.pendingEvents              # the FullyRandom(seed) Execution made
        self.rand = JavaRandom(seed)
        self.srcDsts = []
        self.srcDstToMessages = {}
        outer = self

        class View(object):                                          # what Execution touches of `pendingEvents`
            def insert(_, t):                                        # SrcDstFIFO.+= (:786-805)
                if t[2] == DEADLETTERS:
                    outer.timersAndExternals.insert(t)
                    return
                key = (t[2], t[3])
                if key not in outer.srcDstToMessages:
                    outer.srcDsts.append(key)
                    outer.srcDstToMessages[key] = []
                outer.srcDstToMessages[key].append(t)

            def remove(_, t):                                        # only timers are ever removed (cancel)
                outer.timersAndExternals.remove(t)

            @property
            def arr(_):
                return outer.timersAndExternals.arr + [(t, 0) for q in outer.srcDstToMessages.values() for t in q]

            def isEmpty(_):
                return not outer.timersAndExternals.arr and not outer.srcDstToMessages
        self.pendingEvents = View()

    def _timer_non_blocked(self):                # find_non_blocked_message over timersAndExternals
        te = self.timersAndExternals
        if te.isEmpty():
            return None
        blocked = []
        e = te.removeRandomElement()
        while e[3] in self.blockedActors:
            blocked.append(e)
            if te.isEmpty():
                for b in blocked:
                    te.insert(b)
                return None
            e = te.removeRandomElement()
        for b in blocked:
            te.insert(b)
        return e

    def pick_non_blocked(self):                  # getNonBlockedMessage (:716-756) + dequeue (:758-768)
        if not any(k[1] not in self.blockedActors for k in self.srcDstToMessages):
            return self._timer_non_blocked()                         # "Only timers left"
        n_all = len(self.timersAndExternals.arr) + sum(len(q) for q in self.srcDstToMessages.values())
        if self.rand.nextInt(n_all) < len(self.timersAndExternals.arr):
            t = self._timer_non_blocked()
            if t is not None:
                return t
        idx = self.rand.nextInt(len(self.srcDsts))
        while self.srcDsts[idx][1] in self.blockedActors:
            idx = self.rand.nextInt(len(self.srcDsts))
        key = self.srcDsts[idx]
        q = self.srcDstToMessages[key]
        ret = q.pop(0)
        if not q:
            del self.srcDstToMessages[key]
            del self.srcDsts[idx]
        return ret


class Context(object):
    """What an actor can do inside receive(): `!`, scheduleOnce, schedule, cancel."""

    def __init__(self, ex, name):
        self.ex, self.name = ex, name

    def send(self, dst, msg):
        self.ex.tell(self.name, dst, msg)

    def schedule_repeating(self, msg):
        self.ex.registerCancellable(True, self.name, msg)

    def schedule_once(self, msg):
        self.ex.registerCancellable(False, self.name, msg)

    def cancel(self, msg):
        self.ex.cancelTimer(self.name, msg)


# ---------------------------------------------------------------- the applications (DESIGN.md §3), a third time
class PingPongActor(object):
    def __init__(self, idx):
        self.idx, self.pings, self.pongs = idx, 0, 0

    def receive(self, ctx, sender, msg):
        t, p0, _ = msg
        if t == 1:
            self.pings += 1
            ctx.send(str((self.idx + 1) % 3), (2, p0, 0))
        elif t == 2:
            self.pongs += 1


BOOT, CLIENT_CMD, ELECTION_TICK, REQUEST_VOTE, VOTE_REPLY, HEARTBEAT_TICK, APPEND_ENTRIES, APPEND_REPLY = range(1, 9)
INIT, FOLLOWER, CANDIDATE, LEADER = range(4)


class RaftActor(object):
    """Raft Fig. 2, 5 nodes, tick timers, log capacity 8, one entry per AppendEntries, leader no-op on election."""

    def __init__(self, idx, flags):
        self.idx, self.flags = idx, flags
        self.role, self.term, self.voted, self.votes, self.heard, self.commit = INIT, 0, None, set(), False, 0
        self.log = []                            # [(term, value)]
        self.next, self.match = [0] * 5, [0] * 5

    def step_down(self, ctx, t):
        if self.role == LEADER:
            ctx.cancel((HEARTBEAT_TICK, 0, 0))
        if t > self.term:
            self.term, self.voted = t, None
        self.role, self.votes = FOLLOWER, set()

    def send_append(self, ctx, j):
        prev = self.next[j]
        pt = self.log[prev - 1][0] if prev else 0
        has = 1 if prev < len(self.log) else 0
        et, ev = self.log[prev] if has else (0, 0)
        ctx.send(str(j), (APPEND_ENTRIES, self.term | (prev << 8) | (pt << 16) | (self.commit << 24), has | (et << 8) | (ev << 16)))

    def reply(self, ctx, src, msg):
        if src is not None:                      # DESIGN.md §3 raft5 R1: no reply to deadLetters
            ctx.send(str(src), msg)

    def receive(self, ctx, sender, msg):
        ty, p0, p1 = msg
        src = int(sender) if sender.isdigit() else None
        last_idx = len(self.log)
        last_term = self.log[-1][0] if self.log else 0
        t = p0 & 0xFF
        if ty not in (BOOT, CLIENT_CMD) and self.role == INIT:
            return
        if ty == BOOT:
            if self.role == INIT:
                self.role = FOLLOWER
                ctx.schedule_repeating((ELECTION_TICK, 0, 0))
        elif ty == CLIENT_CMD:
            if self.role == LEADER and len(self.log) < 8:
                self.log.append((self.term, p0 & 0x7F))
        elif ty == ELECTION_TICK:
            if self.role == LEADER:
                return
            if self.heard:
                self.heard = False
                return
            if self.term == 255:
                return
            self.term += 1
            self.role, self.voted, self.votes = CANDIDATE, self.idx, {self.idx}
            for j in range(5):
                if j != self.idx:
                    ctx.send(str(j), (REQUEST_VOTE, self.term | (last_idx << 8) | (last_term << 16), 0))
        elif ty == REQUEST_VOTE:
            li, lt = (p0 >> 8) & 0xFF, (p0 >> 16) & 0xFF
            if t > self.term:
                self.step_down(ctx, t)
            up_to_date = lt > last_term or (lt == last_term and li >= last_idx)
            can_vote = self.voted is None or self.voted == src or (self.flags & 1)
            grant = 1 if (t == self.term and can_vote and up_to_date) else 0
            if grant:
                self.voted, self.heard = src, True
            self.reply(ctx, src, (VOTE_REPLY, self.term | (grant << 8), 0))
        elif ty == VOTE_REPLY:
            if t > self.term:
                self.step_down(ctx, t)
                return
            if src is None:                      # R2: no vote from deadLetters
                return
            if self.role == CANDIDATE and t == self.term and (p0 >> 8) & 1:
                self.votes.add(src)
                if len(self.votes) >= 3:
                    self.role = LEADER
                    self.next, self.match = [len(self.log)] * 5, [0] * 5
                    if len(self.log) < 8:
                        self.log.append((self.term, 0x80 | self.idx))
                    for j in range(5):
                        if j != self.idx:
                            self.send_append(ctx, j)
                    ctx.schedule_repeating((HEARTBEAT_TICK, 0, 0))
        elif ty == HEARTBEAT_TICK:
            if self.role == LEADER:
                for j in range(5):
                    if j != self.idx:
                        self.send_append(ctx, j)
        elif ty == APPEND_ENTRIES:
            prev, pt, lc = (p0 >> 8) & 0xFF, (p0 >> 16) & 0xFF, (p0 >> 24) & 0xFF
            has, et, ev = p1 & 1, (p1 >> 8) & 0xFF, (p1 >> 16) & 0xFF
            if t < self.term:
                self.reply(ctx, src, (APPEND_REPLY, self.term, 0))
                return
            if t > self.term or self.role != FOLLOWER:
                self.step_down(ctx, t)
            self.heard = True
            ok = prev <= len(self.log) and (prev == 0 or self.log[prev - 1][0] == pt)
            if not ok:
                self.reply(ctx, src, (APPEND_REPLY, self.term, 0))
                return
            mi = prev
            if has:
                if len(self.log) > prev and self.log[prev][0] != et:
                    del self.log[prev:]
                if len(self.log) == prev and prev < 8:
                    self.log.append((et, ev))
                if len(self.log) > prev:
                    mi = prev + 1
            self.commit = max(self.commit, min(lc, mi))
            self.reply(ctx, src, (APPEND_REPLY, self.term | (1 << 8) | (mi << 16), 0))
        elif ty == APPEND_REPLY:
            ok, mi = (p0 >> 8) & 1, (p0 >> 16) & 0xFF
            if t > self.term:
                self.step_down(ctx, t)
                return
            if self.role != LEADER or t != self.term or src is None:   # R2: nothing indexed by deadLetters
                return
            if ok:
                self.match[src] = max(self.match[src], mi)
                self.next[src] = max(self.next[src], mi)
                for i in range(len(self.log), self.commit, -1):
                    if self.log[i - 1][0] != self.term and not (self.flags & 2):
                        continue
                    if 1 + sum(1 for k in range(5) if k != self.idx and self.match[k] >= i) >= 3:
                        self.commit = i
                        break
            elif self.next[src] > 0:
                self.next[src] -= 1


def raft_invariant(actors):
    """1: two leaders in one term; 2: committed prefixes disagree (1 wins; else the first pair in (i, j) order)."""
    a = [actors[str(i)] for i in range(5)]
    code = None
    for i in range(5):
        for j in range(i + 1, 5):
            if a[i].role == LEADER and a[j].role == LEADER and a[i].term == a[j].term:
                return 1
            if code is None:                     # entries past the log's end are the cleared (0, 0) of the state bytes
                c = min(a[i].commit, a[j].commit)
                if (a[i].log + [(0, 0)] * 8)[:c] != (a[j].log + [(0, 0)] * 8)[:c]:
                    code = 2
    return code


def pingpong_invariant(flags):
    return lambda actors: 7 if (flags & 1) and actors["0"].pongs >= (flags >> 8) else None


# ---------------------------------------------------------------- loaded models (include/demi_model_ir.h), read from the header alone
IR_OPS = dict(HALT=0, LDI=1, MOV=2, ADD=3, SUB=4, MUL=5, AND=6, OR=7, XOR=8, SHL=9, SHR=10, MOD=11, LDW=12, STW=13, LDA=14,
              JMP=15, JEQ=16, JNE=17, JLT=18, JGE=19, SEND=20, SCHED_ONCE=21, SCHED_REPEAT=22, CANCEL=23, RET=24)
IR_NAME = {v: k for k, v in IR_OPS.items()}
IR_ACTORS, IR_WORDS, IR_OUTBOX, IR_MAX_STEPS = 16, 8, 16, 4096
U32 = 0xFFFFFFFF


class OperationLimit(Exception):
    """One receive() issued more than IR_OUTBOX operations: the execution ends with the queue-overflow status."""


class IRModel(object):
    """A demi_load_model blob, parsed word by word: header, receive() and invariant programs, initial states."""

    def __init__(self, blob):
        w = [int.from_bytes(blob[i:i + 4], "little") for i in range(0, len(blob) - len(blob) % 4, 4)]
        assert w[0] == 0x52494D44 and w[1] == 1
        self.n_actors, self.state_words, self.n_types = w[2], w[3], w[4]
        rl, il = w[5], w[6]
        self.ext_mask, self.fanout = w[7], w[8]
        self.recv = w[16:16 + rl]
        self.inv = w[16 + rl:16 + rl + il]
        init = w[16 + rl + il:16 + rl + il + self.n_actors * self.state_words]
        self.init = [init[a * self.state_words:(a + 1) * self.state_words] for a in range(self.n_actors)]
        self.stats = {}                          # opcode name / event -> count, over every program this model ran

    def is_external(self, msg):                  # a 32-bit filter: types >= 32 are never external
        return msg[0] < 32 and (self.ext_mask >> msg[0]) & 1 == 1

    def names(self):
        return [str(a) for a in range(self.n_actors)]

    def make_actors(self, flags):
        return {n: IRActor(self, int(n), flags) for n in self.names()}

    def fresh(self, flags):
        return lambda name: IRActor(self, int(name), flags)

    def _count(self, k):
        self.stats[k] = self.stats.get(k, 0) + 1

    def run(self, code, r, own, all_words, emit):
        """-> (code, affected) of RET, else (0, 0).  own: list of IR_WORDS words or None; all_words(a, i) or None."""
        pc = steps = 0
        while pc < len(code):
            if steps >= IR_MAX_STEPS:
                self._count("step_limit")
                return 0, 0
            steps += 1
            ins = code[pc]; pc += 1
            op, a, b, c = ins & 0xFF, (ins >> 8) & 15, (ins >> 16) & 15, (ins >> 24) & 15
            imm = 0
            if op == 1 or 15 <= op <= 19:
                if pc >= len(code):
                    return 0, 0
                imm = code[pc]; pc += 1
            name = IR_NAME.get(op)
            if name is None:
                return 0, 0
            self._count(name)
            if name == "HALT":
                return 0, 0
            elif name == "LDI":
                r[a] = imm
            elif name == "MOV":
                r[a] = r[b]
            elif name in ("ADD", "SUB", "MUL", "AND", "OR", "XOR", "SHL", "SHR", "MOD"):
                x, y = r[b], r[c]
                if name == "MUL" and x * y > U32:
                    self._count("mul_overflow")
                if name in ("SHL", "SHR") and y >= 32:
                    self._count("wide_shift")
                if name == "MOD" and y == 0:
                    self._count("mod_zero")
                r[a] = {"ADD": x + y, "SUB": x - y, "MUL": x * y, "AND": x & y, "OR": x | y, "XOR": x ^ y,
                        "SHL": x << (y % 32), "SHR": x >> (y % 32), "MOD": x % y if y else 0}[name] & U32
            elif name == "LDW":
                r[a] = own[r[b]] if own is not None and r[b] < IR_WORDS else 0
            elif name == "STW":
                if own is not None and r[a] < IR_WORDS:
                    own[r[a]] = r[b]
            elif name == "LDA":
                r[a] = all_words(r[b], r[c]) if all_words is not None and r[b] < IR_ACTORS and r[c] < IR_WORDS else 0
            elif name == "JMP":
                pc = imm
            elif name in ("JEQ", "JNE", "JLT", "JGE"):
                x, y = r[a], r[b]
                if {"JEQ": x == y, "JNE": x != y, "JLT": x < y, "JGE": x >= y}[name]:
                    pc = imm
            elif name == "SEND":
                emit(name, r[a] & 0xFF, (r[b] & 0xFF, r[c], r[(c + 1) % 16]))
            elif name in ("SCHED_ONCE", "SCHED_REPEAT", "CANCEL"):
                emit(name, None, (r[a] & 0xFF, r[b], r[c]))
            elif name == "RET":
                return r[a], r[(a + 1) % 16]
        return 0, 0

    def invariant(self, flags):
        def inv(actors):
            def word(a, i):
                act = actors.get(str(a))
                return act.st[i] if act is not None else 0
            r = [0] * 16
            r[5] = flags & U32
            code, _ = self.run(self.inv, r, None, word, lambda *x: None)
            if code:
                self._count("violation")
            return code or None
        return inv


class IRActor(object):
    def __init__(self, model, idx, flags):
        self.model, self.idx, self.flags = model, idx, flags & U32
        self.st = list(model.init[idx]) + [0] * (IR_WORDS - model.state_words)

    def receive(self, ctx, sender, msg):
        m = self.model
        r = [0] * 16
        r[0], r[1] = self.idx, int(sender) if sender.isdigit() else 0xFF
        r[2], r[3], r[4], r[5] = msg[0], msg[1], msg[2], self.flags
        ops = []

        def emit(kind, dst, message):
            if kind == "SEND" and dst >= m.n_actors:
                m._count("dropped_send")                             # not one of the model's actors
                return
            ops.append((kind, dst, message))
        m.run(m.recv, r, self.st, None, emit)
        if len(ops) > IR_OUTBOX:
            m._count("op_limit")
            raise OperationLimit()
        for kind, dst, message in ops:
            if kind == "SEND":
                ctx.send(str(dst), message)
            elif kind == "SCHED_ONCE":
                m._count("timer_armed"); ctx.schedule_once(message)
            elif kind == "SCHED_REPEAT":
                m._count("timer_armed"); ctx.schedule_repeating(message)
            else:
                ctx.cancel(message)


# ---------------------------------------------------------------- STSScheduler (schedulers/STSScheduler.scala, EventTrace.scala)
def subsequence_intersection(events, original_externals, subseq, is_external, filter_known_absents):
    """EventTrace.subsequenceIntersection (EventTrace.scala:290-380) -> filterSends (:382-452) -> filterKnownAbsentInternals
    (:458-534), as written.  `subseq`: increasing indices into original_externals.  Events are the tuples Execution records."""
    remaining = [original_externals[i] for i in subseq if original_externals[i][0] != "Send"]
    result = []
    for event in events:
        k = event[0]
        if not remaining:
            if k in ("MsgSend", "MsgEvent"):                         # isMessageType
                result.append(event)
            elif k not in ("Spawn", "Kill", "Partition", "UnPartition", "HardKill"):   # !isExternal (EventTypes :184-201)
                result.append(event)
        else:
            head = remaining[0]
            if k == "Kill":
                if head[0] == "Kill" and head[1] == event[1]:
                    result.append(event); remaining = remaining[1:]
            elif k == "Partition":
                if head[0] == "Partition" and (head[1], head[2]) == (event[1], event[2]):
                    result.append(event); remaining = remaining[1:]
            elif k == "UnPartition":
                if head[0] == "UnPartition" and (head[1], head[2]) == (event[1], event[2]):
                    result.append(event); remaining = remaining[1:]
            elif k == "Spawn":
                if head[0] == "Start" and head[1] == event[1]:
                    result.append(event); remaining = remaining[1:]
            elif k == "HardKill":
                if head[0] == "HardKill" and head[1] == event[1]:
                    result.append(event); remaining = remaining[1:]
            else:
                result.append(event)                                 # "Always include all other internal events"
    # filterSends: the i-th external MsgSend belongs to the i-th Send of original_externals (FIFO assumption)
    original_sends = [i for i, e in enumerate(original_externals) if e[0] == "Send"]
    in_subseq = set(subseq)
    missing_indices = set(k for k, i in enumerate(original_sends) if i not in in_subseq)
    msg_send_idx = -1
    pruned_msg_ids = set()
    remaining_events = []
    for e in result:
        if e[0] == "MsgSend":
            if is_external(e[3]):
                msg_send_idx += 1
                if msg_send_idx not in missing_indices:
                    remaining_events.append(e)
                else:
                    pruned_msg_ids.add(e[4])
            else:
                remaining_events.append(e)
        elif e[0] == "MsgEvent":
            if e[4] not in pruned_msg_ids:
                remaining_events.append(e)
        else:
            remaining_events.append(e)
    if not filter_known_absents:
        return remaining_events
    # filterKnownAbsentInternals, as written — including that a PartitionEvent marks the pair as NOT partitioned and an
    # UnPartitionEvent marks it partitioned (:523-528)
    alive = {DEADLETTERS: True, "Timer": True}
    partitioned = {}
    pruned_sends = set()
    out = []
    for e in remaining_events:
        k = e[0]
        if k == "MsgSend":
            snd, rcv = e[1], e[2]
            if alive.get(snd, False) and not partitioned.get((snd, rcv), False):
                out.append(e)
            else:
                pruned_sends.add(e[4])
        elif k == "MsgEvent":
            snd, rcv = e[1], e[2]
            if alive.get(rcv, False) and not partitioned.get((snd, rcv), False) and e[4] not in pruned_sends:
                out.append(e)
        elif k == "Spawn":
            alive[e[1]] = True; out.append(e)
        elif k == "Kill":
            alive[e[1]] = False; out.append(e)
        elif k == "Partition":
            partitioned[(e[1], e[2])] = False; out.append(e)
        elif k == "UnPartition":
            partitioned[(e[1], e[2])] = True; out.append(e)
        else:
            out.append(e)
    return out


class STSReplay(Execution):
    """STSScheduler.test (STSScheduler.scala:199-310) with allowPeek = false, no failure detector, no checkpointing,
    abortUponDivergence off: advanceReplay (:405-559), event_produced (:561-623), schedule_new_message (:643-776),
    notify_timer_cancel (:846-868).  The Instrumenter side (`!`, timers, dispatch) is Execution's."""

    def __init__(self, actors, original_events, original_externals, invariant, is_external, filter_known_absents=False,
                 looking_for=None, blocked=(), ignore_timers=False):
        Execution.__init__(self, actors, [], 0, -1, 0, invariant, is_external, blocked=blocked, looking_for=looking_for,
                           ignore_timers=ignore_timers)
        self.original_events, self.original_externals = original_events, original_externals
        self.filterKnownAbsents = filter_known_absents
        self.pending = {}                        # (snd, rcv) -> {fingerprint -> [(uniq, msg)]}   (:112-114)
        self.delivered = self.ignored = 0

    # ---- scheduler callbacks
    def event_produced(self, snd, rcv, msg):     # :561-623
        self.uniq_counter += 1
        uniq = self.uniq_counter & 0xFFFF                            # Uniq ids are 16-bit and wrap (DESIGN.md §2)
        is_timer = False
        if msg in self.enqueuedExternalMessages:                     # handle_event_produced: ExternalMessage
            self.pending.setdefault((snd, rcv), {}).setdefault(msg, []).append((uniq, msg))
        else:
            if snd == DEADLETTERS:
                is_timer = True
            if not self.crosses_partition(snd, rcv):
                self.pending.setdefault((snd, rcv), {}).setdefault(msg, []).append((uniq, msg))
        self.events.append(("MsgSend", "Timer" if is_timer else snd, rcv, msg, uniq, 0))

    def enqueue_timer(self, rcv, msg):           # :870
        self.handle_timer(rcv, msg)

    def notify_timer_cancel(self, rcv, msg):     # :846-868
        for i, (s, r, m) in enumerate(self.messagesToSend):          # handle_timer_cancel
            if r == rcv and m == msg:
                del self.messagesToSend[i]
                return
        h = self.pending.get((DEADLETTERS, rcv))
        if h is not None and msg in h:
            q = h[msg]
            for i, (_, m) in enumerate(q):
                if m == msg:
                    del q[i]
                    break
            if not q:
                del h[msg]
                if not h:
                    del self.pending[(DEADLETTERS, rcv)]

    def message_pending(self, snd, rcv, msg):    # :381-403
        self.send_external_messages()
        h = self.pending.get((snd, rcv))
        if h is None or msg not in h:
            return False
        return rcv not in self.blockedActors

    def advance_replay(self):                    # :405-559
        while self.traceIdx < len(self.trace):
            e = self.trace[self.traceIdx]
            k = e[0]
            if k == "Spawn":                                         # trigger_start
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
                if self.is_external(e[3]):                           # enqueue_message(None, receiver, message)
                    self.enqueuedExternalMessages.append(e[3])
                    self.messagesToSend.append((None, e[2], e[3]))
            elif k == "MsgEvent":
                if self.message_pending(e[1], e[2], e[3]):
                    return                                           # "Yay, it's already enabled."
                self.ignored += 1                                    # "Ignoring message"
            elif k in ("Quiescence", "BeginWaitQuiescence"):
                self.events.append(e)
            self.traceIdx += 1

    def schedule_new_message(self):              # :643-776
        self.send_external_messages()
        self.advance_replay()
        self.send_external_messages()
        if self.traceIdx >= len(self.trace):
            return None
        _, snd, rcv, msg, _, _ = self.trace[self.traceIdx]           # a MsgEvent advanceReplay found enabled
        h = self.pending[(snd, rcv)]
        q = h[msg]
        uniq, m = q.pop(0)                                           # Queue.dequeue: oldest first
        if not q:
            del h[msg]
            if not h:
                del self.pending[(snd, rcv)]
        self.events.append(("MsgEvent", snd, rcv, m, uniq, 0))
        self.traceIdx += 1
        self.delivered += 1
        return (uniq, None, snd, rcv, m)

    def test(self, subseq):
        self.trace = subsequence_intersection(self.original_events, self.original_externals, subseq, self.is_external,
                                              self.filterKnownAbsents)
        self.traceIdx = 0
        self.advance_replay()                                        # "Start playing back trace"
        while True:
            e = self.schedule_new_message()
            if e is None:
                break
            self.dispatch_new_message(e)
        return self.violationMatches(self.invariant(self.actors))


# ---------------------------------------------------------------- ProvenanceTracker (schedulers/Util.scala:267-376)
class ProvenanceTracker(object):
    """trace: [(unique id, receiver name)] = DepTracker.initialTrace (the root first); parent_of: the DepTracker tree.
    happensBefore = first-order pairs (same receiver, earlier or the event itself; a receive and the messages sent as
    its result) closed transitively — by plain reachability here, the relation is what matters."""

    def __init__(self, trace, parent_of):
        self.trace = trace
        kids = {}
        for c, p in parent_of.items():
            if p is not None:
                kids.setdefault(p, []).append(c)
        first = set()
        prior = {}
        for u, rcv in trace:
            prior.setdefault(rcv, []).append(u)
            for p in prior[rcv]:
                first.add((p, u))
            for c in kids.get(u, []):
                first.add((u, c))
        succ = {}
        for a, b in first:
            if a != b:
                succ.setdefault(a, set()).add(b)
        verts = set(x for pr in first if pr[0] != pr[1] for x in pr)
        self.hb = set(first)
        for v in verts:                                              # v's transitive closure includes v itself
            seen, stack = {v}, [v]
            while stack:
                x = stack.pop()
                for y in succ.get(x, ()):
                    if y not in seen:
                        seen.add(y); stack.append(y)
            for y in seen:
                self.hb.add((v, y))

    def pruneConcurrentEvents(self, affected_nodes):
        last = []
        for node in affected_nodes:                                  # findLastEventForNode
            for u, rcv in reversed(self.trace):
                if rcv == node:
                    last.append(u)
                    break
        def concurrent_or_after_all(u):
            return all((not ((o, u) in self.hb or (u, o) in self.hb)) or (o, u) in self.hb for o in last)
        return [i for i, (u, _) in enumerate(self.trace) if not concurrent_or_after_all(u)]


# ---------------------------------------------------------------- internal-event minimization
class LeftToRightOneAtATime(object):
    """OneAtATimeStrategy + LeftToRightOneAtATime (internal_minimization/OneAtATimeRemoval.scala:17-137)."""

    def __init__(self, verified_events, is_external):
        from collections import Counter
        self.triedIgnoring = Counter()
        for e in verified_events:                                    # init(): external deliveries are unignorable
            if e[0] == "MsgEvent" and is_external(e[3]):
                self.triedIgnoring[(e[1], e[2], e[3])] += 1
        self.unignorable = sum(self.triedIgnoring.values())

    def getNextTrace(self, trace, alreadyRemoved, violationTriggered):
        from collections import Counter
        keysThisIteration = Counter(alreadyRemoved)
        found = [False]

        def checkDelivery(snd, rcv, msg):
            key = (snd, rcv, msg)
            keysThisIteration[key] += 1
            if found[0]:
                return True
            if keysThisIteration[key] > self.triedIgnoring[key]:     # choiceFilter is `true`
                found[0] = True
                self.triedIgnoring[key] += 1
                return False
            return True
        modified = [e for e in trace if e[0] != "MsgEvent" or checkDelivery(e[1], e[2], e[3])]
        return modified if found[0] else None


class SrcDstFIFORemoval(LeftToRightOneAtATime):
    """SrcDstFIFORemoval (OneAtATimeRemoval.scala:139-251): only the last delivery of each (src, dst) FIFO is tried, plus
    timers; the per-pair bookkeeping and its recomputation after a successful removal as written."""

    def __init__(self, verified_events, is_external):
        LeftToRightOneAtATime.__init__(self, verified_events, is_external)
        self.verified = verified_events
        self.srcDstToMessages = {}
        for e in verified_events:
            if e[0] == "MsgEvent" and e[1] != DEADLETTERS:
                self.srcDstToMessages.setdefault((e[1], e[2]), []).append(e[3])
        self.previouslyChosenSrcDst = None
        self.srcDstToCurrentIdx = {}
        self.reset_idx()

    def reset_idx(self):
        for k in self.srcDstToMessages:
            self.srcDstToCurrentIdx[k] = -1

    def choiceFilter(self, snd, rcv, msg):
        key = (snd, rcv)
        if key in self.srcDstToMessages:
            self.srcDstToCurrentIdx[key] += 1
            idx = self.srcDstToCurrentIdx[key]
            lst = self.srcDstToMessages[key]
            if idx == len(lst) - 1:
                self.srcDstToMessages[key] = lst[:-1]
                if not self.srcDstToMessages[key]:
                    del self.srcDstToMessages[key]
                self.previouslyChosenSrcDst = key
                return True
        self.previouslyChosenSrcDst = None
        return snd == DEADLETTERS                                    # a timer

    def getNextTrace(self, trace, alreadyRemoved, violationTriggered):
        from collections import Counter
        if not violationTriggered and self.previouslyChosenSrcDst is not None:
            self.srcDstToMessages.pop(self.previouslyChosenSrcDst, None)
        if violationTriggered:
            self.srcDstToMessages = {}
            left = Counter(alreadyRemoved)
            for e in reversed(self.verified):
                if e[0] == "MsgEvent" and e[1] != DEADLETTERS:
                    t = (e[1], e[2], e[3])
                    if left[t] > 0:
                        left[t] -= 1
                    else:
                        self.srcDstToMessages[(e[1], e[2])] = [e[3]] + self.srcDstToMessages.get((e[1], e[2]), [])
        self.reset_idx()
        keysThisIteration = Counter(alreadyRemoved)
        found = [False]

        def checkDelivery(snd, rcv, msg):
            key = (snd, rcv, msg)
            keysThisIteration[key] += 1
            if found[0]:
                return True
            if keysThisIteration[key] > self.triedIgnoring[key] and self.choiceFilter(snd, rcv, msg):
                found[0] = True
                self.triedIgnoring[key] += 1
                return False
            return True
        modified = [e for e in trace if e[0] != "MsgEvent" or checkDelivery(e[1], e[2], e[3])]
        return modified if found[0] else None


class STSSchedMinimizer(object):
    """STSSchedMinimizer.minimize (internal_minimization/ScheduleCheckers.scala:19-107)."""

    def __init__(self, mcs, verified_events, violation, strategy, test):
        self.mcs, self.verified, self.violation, self.strategy, self.test = mcs, verified_events, violation, strategy, test
        self.total_replays = 0
        self.internal_sizes = []

    def minimize(self):
        from collections import Counter
        count = lambda tr: sum(1 for e in tr if e[0] == "MsgEvent")
        deliveries = lambda tr: Counter((e[1], e[2], e[3]) for e in tr if e[0] == "MsgEvent")
        last = self.verified
        lastSize = count(last)
        prunedOverall = Counter()
        triggered = False
        nxt = self.strategy.getNextTrace(last, prunedOverall, triggered)
        while nxt is not None:
            self.total_replays += 1                                  # STSScheduler.test: stats.increment_replays
            got = self.test(nxt)                                     # RunnerUtils.testWithStsSched -> Option[EventTrace]
            if got is not None:
                triggered = True
                prunedOverall += deliveries(last) - deliveries(got)  # MultiSet.setDifference
                last = got
                lastSize = count(got)
                self.internal_sizes.append(lastSize)
            else:
                triggered = False
                self.internal_sizes.append(lastSize)
            nxt = self.strategy.getNextTrace(last, prunedOverall, triggered)
        return last


# ---------------------------------------------------------------- DPORwHeuristics (schedulers/DPORwHeuristics.scala)
class DPORSearch(object):
    """DPORwHeuristics.test for external programs of Start / Send events: DefaultBacktrackOrdering, trackHistory on,
    checkpointing off (invariant at the end of every interleaving), prioritizePendingUponDivergence off, no depth
    bound.  Two choices the Scala leaves to scala-library internals are fixed as DESIGN.md §6 fixes them: the divergent
    choice (`pendingEvents.find` over a HashMap, :454-456) takes the first non-empty queue in (sender, receiver) order
    with deadLetters last, and backtrack points of equal branch depth leave the PriorityQueue oldest first.
    `blocked` is the blockedActors set schedule_new_message is called with (:421); nothing here reads ignoreTimers,
    because DPORwHeuristics sends a timer at once (enqueue_timer = enqueue_message, Scheduler.scala:73) and never
    reaches ExternalEventInjector.handle_timer."""

    def __init__(self, make_actors, externals, invariant, max_messages, stop_if_found=True, looking_for=None, blocked=()):
        self.make_actors, self.externals, self.invariant = make_actors, externals, invariant
        self.blockedActors = set(blocked)
        self.max_messages, self.stopIfViolationFound, self.lookingFor = max_messages, stop_if_found, looking_for
        # the dependency graph (child -> parent edges), ids from one counter, root = Unique(MsgEvent("null","null",null), 0)
        self.event = {0: ("null", "null", None)}
        self.parent_of = {0: None}
        self.kids = {0: []}
        self.next_id = 1
        self.backTrack = []                      # (branchI, seq, (e1, e2), replayThis)
        self.seq = 0
        self.explored = set()                    # ExploredTacker: ordered pairs, whatever the index
        self.interleavingCounter = 0
        self.shortestTraceSoFar = None
        self.nextTrace = []
        self.races = 0
        self.traces = []                         # every finished currentTrace (with the root at index 0)
        self.violations = []                     # (interleaving index, code)

    # ---- graph helpers
    def path_from_root(self, n):
        out = []
        while n is not None:
            out.append(n); n = self.parent_of[n]
        return out[::-1]

    def has_path_to(self, frm, to):              # laterN.pathTo(earlierN): edges point from a message to its parent
        while frm is not None:
            if frm == to:
                return True
            frm = self.parent_of[frm]
        return False

    # ---- Instrumenter: `!`, timers (enqueue_timer = enqueue_message = an immediate `!` from deadLetters, Scheduler.scala:73)
    def tell(self, snd, rcv, msg):
        if (rcv, msg) in self.timersCancelledThisStep:               # aroundDispatch :1090-1096
            self.timersCancelledThisStep.discard((rcv, msg))
            return
        self.event_produced(snd, rcv, msg)

    def registerCancellable(self, ongoing, rcv, msg):
        if (rcv, msg) in self.timerToCancellable:
            return
        self.timerToCancellable[(rcv, msg)] = ongoing
        self.handleTick(rcv, msg)

    def handleTick(self, rcv, msg):
        ongoing = self.timerToCancellable[(rcv, msg)]
        self.tell(DEADLETTERS, rcv, msg)
        if not ongoing:
            del self.timerToCancellable[(rcv, msg)]

    def cancelTimer(self, rcv, msg):
        self.timersCancelledThisStep.add((rcv, msg))
        self.timerToCancellable.pop((rcv, msg), None)
        q = self.pending.get((DEADLETTERS, rcv))                     # notify_timer_cancel :961-985
        if q is not None:
            for i, (_, m) in enumerate(q):
                if m == msg:
                    del q[i]
                    break

    # ---- scheduler
    def get_message(self, snd, rcv, msg):        # :773-801
        for c in self.kids[self.parentEvent]:
            if self.event[c] == (snd, rcv, msg):
                return c
        c = self.next_id
        self.next_id += 1
        self.event[c] = (snd, rcv, msg)
        return c

    def event_produced(self, snd, rcv, msg):     # :803-847
        u = self.get_message(snd, rcv, msg)
        self.pending.setdefault((snd, rcv), []).append((u, msg))
        if u not in self.parent_of:                                  # addGraphNode + addEdge(unique, parentEvent)
            self.parent_of[u] = self.parentEvent
            self.kids[self.parentEvent].append(u)
            self.kids[u] = []

    def get_matching_message(self):              # :474-537 through getNextTraceMessage :363-372
        while self.nextTrace:
            u = self.nextTrace.pop(0)
            if u == 0:
                continue                                             # "All system messages need to ignored" (the root)
            snd, rcv, _ = self.event[u]
            if rcv in self.blockedActors:
                return None                                          # :478, :518: the entry is consumed all the same
            q = self.pending.get((snd, rcv))
            if q is not None:
                for i, (v, m) in enumerate(q):
                    if v == u:                                       # equivalentTo: same receiver and id
                        del q[i]
                        return (u, snd, rcv, m)
            return None
        return None

    def get_pending_event(self):                 # :452-472
        def order(key):
            snd, rcv = key
            return (10 ** 6 if snd == DEADLETTERS else int(snd), int(rcv))
        for key in sorted(self.pending, key=order):
            q = self.pending[key]
            if q and key[1] not in self.blockedActors:             # :455
                u, m = q.pop(0)
                return (u, key[0], key[1], m)
        return None

    def schedule_new_message(self):              # :421-648
        while True:
            if self.foundLookingFor:
                return None
            self.messagesScheduledSoFar += 1
            if self.messagesScheduledSoFar > self.max_messages:
                return None
            res = self.get_matching_message()
            if res is None:
                res = self.get_pending_event()
            if res is None:
                return None
            u, snd, rcv, m = res
            if snd in self.isolatedActors or rcv in self.isolatedActors:
                continue                                             # "Discarding event ... due to not yet started node"
            self.currentTrace.append(u)
            self.parentEvent = u
            return res

    def run_interleaving(self):
        self.actors = self.make_actors()
        self.isolatedActors = set(self.actors)
        self.pending = {}
        self.timerToCancellable, self.timersCancelledThisStep = {}, set()
        self.currentTrace = [0]
        self.parentEvent = 0
        self.messagesScheduledSoFar = 0
        self.foundLookingFor = False
        for e in self.externals:                                     # runExternal :684-721
            if e[0] == "Start":
                self.isolatedActors.discard(e[1])
            elif e[0] == "Send":
                self.tell(DEADLETTERS, e[1], e[2])
            else:
                raise ValueError("unsuported external event")
        while True:
            res = self.schedule_new_message()
            if res is None:
                break
            u, snd, rcv, m = res
            if self.timerToCancellable.get((rcv, m)):                # a repeating timer is re-armed after the hand-off
                self.handleTick(rcv, m)
            self.actors[rcv].receive(_DporContext(self, rcv), snd, m)
        v = self.invariant(self.actors)                              # notify_quiescence -> checkInvariant :394-418
        if v is not None and (self.lookingFor is None or v == self.lookingFor):
            self.foundLookingFor = True
            if self.shortestTraceSoFar is None or len(self.currentTrace) < len(self.shortestTraceSoFar):
                self.shortestTraceSoFar = list(self.currentTrace)
            return v
        return None

    def dpor(self, trace):                       # :1020-1185
        self.interleavingCounter += 1
        n = len(trace)
        for laterI in range(n):
            later = trace[laterI]
            for earlierI in range(laterI):
                earlier = trace[earlierI]
                if self.event[earlier][1] != self.event[later][1]:   # isCoEnabeled: same receiver ...
                    continue
                if self.has_path_to(later, earlier):                 # ... and no dependency path from later to earlier
                    continue
                lp, ep = self.path_from_root(later), self.path_from_root(earlier)
                common = [x for x in lp if x in ep]                  # laterPath.intersect(earlierPath)
                branchI = trace.index(common[-1])
                needToReplay = [x for x in trace[branchI + 1:laterI + 1] if x != earlier]
                assert branchI < laterI
                self.explored.add((earlier, later))
                self.races += 1
                self.backTrack.append((branchI, self.seq, (later, earlier), needToReplay))
                self.seq += 1
        while True:                                                  # getNext :1142-1162
            if not self.backTrack or (self.stopIfViolationFound and self.shortestTraceSoFar is not None):
                return None
            best = max(range(len(self.backTrack)), key=lambda i: (self.backTrack[i][0], -self.backTrack[i][1]))
            maxIndex, _, (e1, e2), replayThis = self.backTrack.pop(best)
            if (e1, e2) in self.explored:
                continue
            self.explored.add((e1, e2))
            return trace[:maxIndex + 1] + replayThis

    def search(self, max_interleavings):
        """test(): interleavings until the backtrack set is empty, a violation stops the search, or the budget is used."""
        exhausted = False
        while True:
            v = self.run_interleaving()
            k = len(self.traces)
            self.traces.append(list(self.currentTrace))
            if v is not None:
                self.violations.append((k, v))
                if self.stopIfViolationFound:
                    break
            if len(self.traces) >= max_interleavings:
                break
            nxt = self.dpor(self.currentTrace)
            if nxt is None:
                exhausted = not self.backTrack
                break
            self.nextTrace = nxt
        return exhausted


class ResumableDPORInstance(DPORSearch):
    """One DPORwHeuristics instance as RunnerUtils.editDistanceDporDDMin configures it (RunnerUtils.scala:822-835) and
    ResumableDPOR drives it (IncrementalDeltaDebugging.scala:90-122): setInitialDepGraph / setInitialTrace,
    prioritizePendingUponDivergence, ArvindDistanceOrdering (BacktrackOrdering.scala:99-173), setMaxDistance, and test()
    called repeatedly (:1193-1242)."""

    def __init__(self, make_actors, externals, invariant, max_messages, init_nodes=None, init_trace=None, arvind=False,
                 prioritize_pending=False, stop_if_found=True, looking_for=None, blocked=()):
        DPORSearch.__init__(self, make_actors, externals, invariant, max_messages, stop_if_found, looking_for, blocked)
        self.arvind, self.prioritize = arvind, prioritize_pending
        self.init_trace = list(init_trace) if init_trace is not None else None
        self.originalIndices = {}
        if init_nodes is not None:                                   # depGraph ++= initialGraph
            for i, (snd, rcv, msg, par) in enumerate(init_nodes):
                if i == 0:
                    continue
                self.event[i] = (snd, rcv, msg)
                self.parent_of[i] = par
                self.kids.setdefault(par, []).append(i)
                self.kids.setdefault(i, [])
            self.next_id = len(init_nodes)
        if self.init_trace is not None:
            for i, e in enumerate(self.init_trace):                  # ArvindDistanceOrdering.init: later occurrences overwrite
                self.originalIndices[e] = i
        self.started = False
        self.currentTrace = []
        self.max_distance = None

    def get_matching_message(self):              # getNextMatchingMessage :542-555 when prioritizePendingUponDivergence
        res = DPORSearch.get_matching_message(self)
        while res is None and self.prioritize and self.nextTrace:
            res = DPORSearch.get_matching_message(self)
        return res

    def distance(self, key):                     # arvindDistance :119-146 (DefaultBacktrackOrdering: 0)
        if not self.arvind:
            return 0
        _, _, (e1, e2), replayThis = key
        path = self.path_from_root(e1) + list(replayThis) + [e1, e2]
        d = 0
        for i, e in enumerate(path):
            if e not in self.originalIndices:
                d += 1
            else:
                for pred in path[:i]:
                    if pred in self.originalIndices and self.originalIndices[pred] > self.originalIndices[e]:
                        d += 1
        return d

    def dpor(self, trace):
        self.interleavingCounter += 1
        n = len(trace)
        for laterI in range(n):
            later = trace[laterI]
            for earlierI in range(laterI):
                earlier = trace[earlierI]
                if self.event[earlier][1] != self.event[later][1] or self.has_path_to(later, earlier):
                    continue
                lp, ep = self.path_from_root(later), self.path_from_root(earlier)
                common = [x for x in lp if x in ep]
                branchI = trace.index(common[-1])
                needToReplay = [x for x in trace[branchI + 1:laterI + 1] if x != earlier]
                self.explored.add((earlier, later))
                self.races += 1
                key = (branchI, self.seq, (later, earlier), needToReplay)
                # a key's distance never changes (the graph only grows below its events): computed once, like the
                # ordering's `distances` cache (:107, :148-154)
                self.backTrack.append(key + (self.distance(key),))
                self.seq += 1
        while True:                                                  # getNext :1142-1162
            if not self.backTrack:
                return None
            rank = lambda i: (self.backTrack[i][4], self.backTrack[i][0], -self.backTrack[i][1])
            best = max(range(len(self.backTrack)), key=rank)          # the larger distance is served first, as written
            if self.max_distance is not None and self.backTrack[best][4] >= self.max_distance:
                return None
            if self.stopIfViolationFound and self.shortestTraceSoFar is not None:
                return None
            maxIndex, _, (e1, e2), replayThis, _ = self.backTrack.pop(best)
            if (e1, e2) in self.explored:
                continue
            self.explored.add((e1, e2))
            return trace[:maxIndex + 1] + replayThis

    def test(self, max_distance, max_interleavings):
        """One DPORwHeuristics.test after ResumableDPOR's setMaxDistance.  Returns (traces run in this call, found)."""
        if self.stopIfViolationFound and self.shortestTraceSoFar is not None:
            return [], True                                          # "Already have shortestTrace!"
        self.max_distance = None if max_distance < 0 else max_distance
        nxt = None
        if self.started and self.backTrack:
            nxt = self.dpor(self.currentTrace)                       # startFromBackTrackPoints :1219-1220
        elif self.init_trace is not None:
            nxt = list(self.init_trace)
        self.nextTrace = list(nxt) if nxt is not None else []
        self.started = True
        ran, found = [], False
        while len(self.traces) < max_interleavings:
            v = self.run_interleaving()
            k = len(self.traces)
            self.traces.append(list(self.currentTrace)); ran.append(list(self.currentTrace))
            if v is not None:
                self.violations.append((k, v)); found = True
                if self.stopIfViolationFound:
                    break
            if len(self.traces) >= max_interleavings:
                break
            nxt = self.dpor(self.currentTrace)
            if nxt is None:
                break
            self.nextTrace = nxt
        return ran, found


class _DporContext(object):
    def __init__(self, s, name):
        self.s, self.name = s, name

    def send(self, dst, msg):
        self.s.tell(self.name, dst, msg)

    def schedule_repeating(self, msg):
        self.s.registerCancellable(True, self.name, msg)

    def schedule_once(self, msg):
        self.s.registerCancellable(False, self.name, msg)

    def cancel(self, msg):
        self.s.cancelTimer(self.name, msg)


def hash6(a, b, c, d, e, f):
    """demi_hash6 (include/demi_limits.h): only used to compare schedules with the C oracle's per-interleaving hashes."""
    M = (1 << 64) - 1
    acc = (a * 0x9E3779B1 + b * 0x85EBCA77 + c * 0xC2B2AE3D + d * 0x27D4EB2F + e * 0x165667B1 + f * 0xD3A2646D + 0x6A09E667BB67AE85) & M
    acc ^= acc >> 32
    acc = (acc * 0x9E3779B97F4A7C15) & M
    acc ^= acc >> 29
    return acc


# ---------------------------------------------------------------- DDMin (minification/DeltaDebugging.scala, Util.scala)
def split_list(l, split_ways):                   # minification/Util.scala:9-37
    if split_ways < 1:
        raise ValueError("Split ways must be greater than 0")
    splits, split_interval = [], len(l) // split_ways
    remainder = len(l) % split_ways
    start_idx = 0
    while len(splits) < split_ways:
        split_idx = start_idx + split_interval
        if remainder > 0:                        # the first `remainder` chunks get one extra element
            split_idx += 1
            remainder -= 1
        splits.append(l[start_idx:split_idx])
        start_idx = split_idx
    return splits


def atomic_events(events):                       # UnmodifiedEventDag.get_atomic_events, minification/Util.scala:197-265
    prev, atomics = {}, []
    for idx, e in events:
        if e[0] == "Kill":
            atomics.append([prev.pop(e[1]), (idx, e)])
        elif e[0] == "Partition":
            prev[(e[1], e[2])] = (idx, e)
        elif e[0] == "Start":
            prev[e[1]] = (idx, e)
        elif e[0] == "UnPartition":
            atomics.append([prev.pop((e[1], e[2])), (idx, e)])
        else:
            atomics.append([(idx, e)])
    for v in prev.values():
        atomics.append([v])
    return sorted(atomics, key=lambda a: a[0][0])


class DDMin(object):                             # minification/DeltaDebugging.scala:7-109
    def __init__(self, test):
        self.test, self.total_replays, self.tests = test, 0, []

    def minimize(self, events):
        return self.ddmin2(list(enumerate(events)), [])

    def ddmin2(self, dag, remainder):
        atoms = atomic_events(dag)
        if len(atoms) <= 1:
            return dag
        keep = split_list(atoms, 2)
        for chunk in keep:                       # splits = [dag - chunk0, dag - chunk1].reverse: left half, then right half
            split = sorted([x for a in chunk for x in a])
            union = sorted(set(split) | set(remainder))
            self.total_replays += 1
            self.tests.append(tuple(i for i, _ in union))
            if self.test([e for _, e in union]):
                return self.ddmin2(split, remainder)
        s0 = sorted([x for a in keep[0] for x in a]); s1 = sorted([x for a in keep[1] for x in a])
        left = self.ddmin2(s0, sorted(set(s1) | set(remainder)))
        right = self.ddmin2(s1, sorted(set(s0) | set(remainder)))
        return sorted(set(left) | set(right))
