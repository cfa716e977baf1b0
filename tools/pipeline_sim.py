"""Randomised-schedule replay of the plane-gather producer / consumer pipelines with mbarrier PARITY-wait semantics (host
only, no GPU).  A parity wait tells "completed an odd / even number of times", so a waiter must see EVERY phase of a
barrier it waits on.  The replay (random interleavings, overwrite / wrong-data / deadlock detection) shows which role
assignments are sound for `k_wgrad_pl` (and, without the gout ring, `k_conv_pl`):
  * producers: warp w fills unit slots w, w + Wu, ... — sound iff Wu divides `stages` (each warp then owns fixed stages);
  * consumers (the kernels): nc warpgroups each consume EVERY slot in order; a stage is free once all nc have arrived
    (`every=True`) — sound for any nc;
  * one warp fills every gout tile (double buffer).
The earlier kernels split the units over nm MMA issuers instead (issuer m owned units u = m (mod nm), `every=False`),
which is sound only if nm divides both `nunits` and `stages`; the two issuer configurations that hung / corrupted tiles on
the GPU (7 producers on 8 stages with 2 issuers, 4 issuers on 6 stages) still fail here and pin the rule.
    python tools/pipeline_sim.py"""
import random
def passed(cnt, parity): return (cnt & 1) != parity
def sim(Wu, nunits, stages, nm, rts, seed, every=False):
    rnd=random.Random(seed)
    full=[0]*stages; empty=[0]*stages; gfull=[0,0]; gempty=[0,0]; arrived=[0]*stages
    data=[None]*stages   # which ord currently in stage (to detect overwrite-before-consume)
    consumed=set(); err=[]
    total=rts*nunits
    def g_filler():
        for rti in range(rts):
            gb=rti&1
            while not passed(gempty[gb], ((rti>>1)&1)^1): yield
            gfull[gb]+=1; yield
    def producer(w):
        o=w; st=w; ph=0
        while o<total:
            while not passed(empty[st], ph^1): yield
            if data[st] is not None and data[st] not in consumed: err.append(('overwrite',o,data[st]))
            data[st]=o; full[st]+=1
            o+=Wu; st+=Wu
            if st>=stages: st-=stages; ph^=1
            yield
    def issuer(m):
        st=0; ph=0
        for git in range(rts):
            gb=git&1
            while not passed(gfull[gb], (git>>1)&1): yield
            for u in range(nunits):
                if every or u%nm==m:
                    while not passed(full[st], ph): yield
                    o=git*nunits+u
                    if data[st]!=o: err.append(('wrongdata',o,data[st]))
                    arrived[st]+=1
                    if not every or arrived[st]==nm:   # every=True: the stage is free once all nm consumers arrived
                        arrived[st]=0; consumed.add(o); empty[st]+=1
                st+=1
                if st==stages: st=0; ph^=1
                yield
            gcommit[gb]+=1
            if gcommit[gb]%nm==0: gempty[gb]+=1
    gcommit=[0,0]
    agents=[g_filler()]+[producer(w) for w in range(Wu)]+[issuer(m) for m in range(nm)]
    alive=list(range(len(agents))); idle=0
    while alive:
        i=rnd.choice(alive)
        before=(tuple(full),tuple(empty),tuple(gfull),tuple(gempty),len(consumed))
        for _ in range(rnd.randint(1,8)):
            try: next(agents[i])
            except StopIteration: alive.remove(i); break
        after=(tuple(full),tuple(empty),tuple(gfull),tuple(gempty),len(consumed))
        idle=0 if after!=before else idle+1
        if idle>30000: return 'DEADLOCK'
    return 'ERR' if err else 'ok'
def producer_choice(stages, max_producers=7):
    """The unit-producer count k_wgrad_pl derives from the ring depth: the largest divisor of `stages` <= 7."""
    return max(d for d in range(1, max_producers + 1) if stages % d == 0)


def host_choice(nunits, stages, max_issuers=4, max_producers=7):
    """Role counts of the earlier multi-issuer kernels (kept to replay the configurations that failed)."""
    Wu = max(d for d in range(1, max_producers + 1) if stages % d == 0)
    nm = 1
    for c in range(2, max_issuers + 1):        # k_wgrad_pl takes any count; k_conv_pl only the powers of two among them
        if nunits % c == 0 and stages % c == 0:
            nm = c
    return Wu, nm


if __name__ == "__main__":
    for stages in range(2, 9):                      # the current kernels: two consumer warpgroups see every slot
        res=[sim(producer_choice(stages),4,stages,2,14,s,every=True) for s in range(40)]
        print("consumers", stages, {k:res.count(k) for k in set(res)})
    for (Wu,nunits,stages,nm) in ((7,8,8,2),(4,8,8,2),(4,8,8,4),(6,8,6,2),(6,6,6,3),(4,4,4,4),(5,4,5,1),(7,7,8,1),(2,2,2,2),(6,8,6,4)):
        res=[sim(Wu,nunits,stages,nm,14,s) for s in range(80)]
        print((Wu,nunits,stages,nm), {k:res.count(k) for k in set(res)})
