"""Large-scale CPU check of the Seidel-shortcut model with the min-x closure (tests/closure_model.c on top of
oracle/shortcut_model.c) against the sequential restatement:
random 7-DOF / 200-gridpoint paths in four flavours (benchmark-like, velocity-limited, randomly scaled waypoints and
limits, non-uniform grids), 4096 paths per job, every 2-variable LP compared bit for bit.
usage: python scripts/shortcut_campaign.py <processes> <jobs>      (10000 jobs = 1.63e10 LPs, about 25 min on 8 cores)
       python scripts/shortcut_campaign.py <processes> <jobs> varied   (1-14 DOF, 20-400 gridpoints, non-uniform knots, both
       discretisations, non-zero boundary speeds incl. failing paths, torque rows; 20000 jobs = 2.3e9 LPs, 4 min)"""
import sys, time, numpy as np, multiprocessing as mp
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
def work(args):
    seed, B, kind = args
    from oracle import oracle as orc
    from problems import make_batch_fast
    from closure_model import closure_model
    rng=np.random.RandomState(seed)
    with closure_model() as sm:
        grid=np.linspace(0,1,200)
        ss,way,vlim,alim=make_batch_fast(B, seed)
        if kind==1: vlim=vlim*0.03           # velocity-limited
        if kind==2: way=way*rng.uniform(0.01,3,size=(B,1,1)); alim=alim*rng.uniform(0.05,5,size=(B,1,1))
        if kind==3: grid=np.sort(np.r_[0,rng.rand(198),1.0])   # non-uniform grid
        c=np.stack([orc.cubic_spline_fit(ss,way[b]) for b in range(B)])
        r=orc.solve_velacc_batch(c,np.tile(ss,(B,1)),grid,vlim,alim,nthreads=1)
        st=sm.stats()
    return st['lps'], st['mismatches'], st['a_used'], st['a_declined'], st['b_used'], st['b_declined'], st['closed'], st['close_declined'], int((r['status']!=0).sum())
def work_varied(seed):
    from oracle import oracle as orc
    from problems import make_torque_problem, inv_dyn_numpy
    from closure_model import closure_model
    rng=np.random.RandomState(seed)
    with closure_model() as sm:
        nfail=0
        for it in range(24):
            dof=rng.randint(1,15); nway=rng.randint(3,11); G=rng.randint(20,400); B=16
            way=rng.randn(B,nway,dof)*rng.choice([0.1,1.0,1.0,3.0])
            vl=(10+rng.rand(B,dof)*20)*rng.choice([1.0,1.0,0.05]); al=10+rng.rand(B,dof)*2
            vlim=np.stack((-vl,vl),-1); alim=np.stack((-al,al),-1)
            ss=np.sort(np.r_[0,rng.rand(nway-2),1.0]) if it%2 else np.linspace(0,1,nway)
            if np.min(np.diff(ss))<1e-3: ss=np.linspace(0,1,nway)
            grid=np.linspace(0,1,G)
            interp = bool(it%3)
            bc = 'not-a-knot' if nway>3 else 'natural'
            c=np.stack([orc.cubic_spline_fit(ss,way[b],bc) for b in range(B)])
            s0=rng.rand(B)*rng.choice([0,0.5]); s1=rng.rand(B)*rng.choice([0,0.5])
            r=orc.solve_velacc_batch(c,np.tile(ss,(B,1)),grid,vlim,alim,interp,sd_start=s0,sd_end=s1,nthreads=1)
            nfail+=int((r['status']!=0).sum())
        # torque rows (cfg-3 shape): vel + acc + torque rows via the generic row interface
        for it in range(2):
            way,vlim,alim,taulim=make_torque_problem(seed*10+it)
            ssw=np.linspace(0,1,5); G=rng.randint(50,300); grid=np.linspace(0,1,G)
            c=orc.cubic_spline_fit(ssw,way)
            base=orc.solve_velacc(c,ssw,grid,vlim,alim,True,0,0,want_rows=True)
            q=orc.ppoly_eval(c,ssw,grid,0); qd=orc.ppoly_eval(c,ssw,grid,1); qdd=orc.ppoly_eval(c,ssw,grid,2)
            z=np.zeros(6)
            cc=np.array([inv_dyn_numpy(a,z,z) for a in q]); aa=np.array([inv_dyn_numpy(a,z,b) for a,b in zip(q,qd)])-cc
            bb=np.array([inv_dyn_numpy(a,b,d) for a,b,d in zip(q,qd,qdd)])-cc
            tl=taulim*rng.choice([1.0,0.3])
            rows=np.stack((np.c_[aa,-aa],np.c_[bb,-bb],np.c_[cc-tl[:,1],-cc+tl[:,0]]),axis=1)
            rows=np.concatenate((base['rows'],rows),axis=2)
            o=orc.solve_rows(rows,base['xbound'],grid,0,0); nfail+=o['status']!=0
        st=sm.stats()
    return st['lps'], st['mismatches'], st['a_used'], st['a_declined'], st['b_used'], st['b_declined'], st['closed'], st['close_declined'], nfail
if __name__=='__main__':
    nproc=int(sys.argv[1]); njobs=int(sys.argv[2]); B=4096
    varied = len(sys.argv) > 3 and sys.argv[3] == 'varied'
    t=time.time(); tot=np.zeros(9,dtype=np.int64)
    import closure_model; closure_model.build()
    with mp.Pool(nproc) as pool:
        jobs = pool.imap_unordered(work_varied, range(700000, 700000 + njobs)) if varied else \
            pool.imap_unordered(work, [(5000000 + j, B, j % 4) for j in range(njobs)])
        for i, res in enumerate(jobs):
            tot+=np.array(res)
            if (i+1)%500==0: print(i+1,'jobs', tot, '%.0fs'%(time.time()-t), flush=True)
    print('TOTAL lps mismatches a_used a_decl b_used b_decl closed close_decl failed_paths:', tot, '%.0fs'%(time.time()-t))
