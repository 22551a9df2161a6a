"""Pure-numpy simulation of the two halo-exchange schemes (used by test_halo_equivalence.py, the
shallow-water emulation and the GPU tests of ops.halo_exchange).  Both work on any dtype: pass
int32 views of float32 arrays to move NaN payloads and -0.0 bit for bit (a wall zero is 0 bits)."""
import numpy as np
rng = np.random.default_rng(0)

def neighbors(py, px, PY, PX, periodic_x=True):
    flat = lambda iy, ix: iy * PX + ix
    def side(dx):
        ix = px+dx
        if not periodic_x and not 0<=ix<PX: return None
        return flat(py, ix%PX)
    nb = dict(south=flat(py-1,px) if py>0 else None, north=flat(py+1,px) if py<PY-1 else None,
              west=side(-1), east=side(1))
    def diag(dy,dx):
        iy, ix = py+dy, px+dx
        if not 0<=iy<PY: return None
        if not periodic_x and not 0<=ix<PX: return None
        return flat(iy,ix%PX)
    dg = dict(sw=diag(-1,-1), se=diag(-1,1), nw=diag(1,-1), ne=diag(1,1))
    return nb, dg

def ref_exchange(arrs, PY, PX, kind, periodic_x=True):
    """The reference's four message rounds (west, north, east, south), then the wall conditions."""
    P = PY*PX
    send_order = ("west","north","east","south"); recv_order=("east","south","west","north")
    sidx = dict(south=(1,slice(None)), west=(slice(None),1), north=(-2,slice(None)), east=(slice(None),-2))
    ridx = dict(south=(0,slice(None)), west=(slice(None),0), north=(-1,slice(None)), east=(slice(None),-1))
    for sd, rd in zip(send_order, recv_order):
        msgs = {}
        for r in range(P):
            py,px = divmod(r,PX); nb,_ = neighbors(py,px,PY,PX,periodic_x)
            if nb[sd] is not None:
                msgs[(r, nb[sd])] = arrs[r][sidx[sd]].copy()
        for r in range(P):
            py,px = divmod(r,PX); nb,_ = neighbors(py,px,PY,PX,periodic_x)
            if nb[rd] is not None:
                arrs[r][ridx[rd]] = msgs[(nb[rd], r)]
    for r in range(P):
        py,px = divmod(r,PX)
        if kind=="u" and not periodic_x and px==PX-1: arrs[r][:,-2]=0
        if kind=="v" and py==PY-1: arrs[r][-2,:]=0

def new_exchange(arrs, PY, PX, kind, periodic_x=True):
    """The single-phase eight-neighbour exchange of b2_k_halo_ll: halo columns over rows [jlo, jhi)
    (the wall rows too where there is no y neighbour), halo rows over the interior columns, corners
    from the diagonal ranks; then u's east-wall column (non-periodic x) and v's north-wall row are 0."""
    P=PY*PX; ny,nx = arrs[0].shape
    snap = [a.copy() for a in arrs]   # all sends read pre-exchange values
    for r in range(P):
        py,px = divmod(r,PX); nb,dg = neighbors(py,px,PY,PX,periodic_x)
        a = arrs[r]
        jlo = 1 if nb["south"] is not None else 0
        jhi = ny-1 if nb["north"] is not None else ny
        if nb["east"] is not None: a[jlo:jhi,nx-1] = snap[nb["east"]][jlo:jhi,1]    # east neighbour's column 1
        if nb["west"] is not None: a[jlo:jhi,0] = snap[nb["west"]][jlo:jhi,nx-2]
        if nb["south"] is not None: a[0,1:nx-1] = snap[nb["south"]][ny-2,1:nx-1]
        if nb["north"] is not None: a[ny-1,1:nx-1] = snap[nb["north"]][1,1:nx-1]
        if dg["sw"] is not None: a[0,0] = snap[dg["sw"]][ny-2,nx-2]
        if dg["se"] is not None: a[0,nx-1] = snap[dg["se"]][ny-2,1]
        if dg["nw"] is not None: a[ny-1,0] = snap[dg["nw"]][1,nx-2]
        if dg["ne"] is not None: a[ny-1,nx-1] = snap[dg["ne"]][1,1]
        if kind=="u" and not periodic_x and px==PX-1: a[:,nx-2]=0
        if kind=="v" and py==PY-1: a[ny-2,:]=0
