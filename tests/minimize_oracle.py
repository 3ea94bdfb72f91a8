"""Numpy restatement of the reference's energy minimizers (src/minimize/minimizer_sd.cu,
minimizer_fire.cu, minimizer_fire_box_change.cu): one iteration as a pure function of the state, in the
reference's order of operations, and the loops around them with the reference's progress lines.

Arrays are [3, n] positions / velocities / forces, U [n], the virial W [9, n] in GPUMD's block order
xx yy zz xy xz yz yx zx zy, h [9] row-major with the lattice vectors as columns."""
import numpy as np

TIME_UNIT_CONVERSION = 1.018051e+1   # src/utilities/common.cuh:26
# minimizer_fire.cuh:24-36 (the same in minimizer_fire_box_change.cuh)
F_INC, F_DEC, ALPHA_START, F_ALPHA = 1.1, 0.5, 0.25, 0.99
DT_0 = 1 / TIME_UNIT_CONVERSION
DT_MAX, DT_MIN = 10 * DT_0, 0.02 * DT_0
N_MIN, MASS = 20, 5.0
STRESS_TOLERANCE_GPA = 1e-4          # minimizer_fire_box_change.cu:254
SD_STEP_0, SD_DECREASE, SD_INCREASE, SD_MIN_STEP = 0.1, 0.2, 1.2, 1e-8  # minimizer_sd.cu:25-28,78
VIRIAL_ROW_MAJOR = (0, 3, 4, 6, 1, 5, 7, 8, 2)  # minimizer_fire_box_change.cu:262-274


def fire_state(box_change=False, L=0.0):
    return dict(dt=DT_0, alpha=ALPHA_START, n_neg=0, v_box=np.zeros(9), L=float(L))


def fire_step(x, v, F, U, W, h, state, tol, box_change=False, hydrostatic=False):
    """One FIRE iteration after the force evaluation at x (minimizer_fire.cu:113-176 / box change
    minimizer_fire_box_change.cu:258-403).  Returns (x, v, h, state, rec); nothing moves when converged.
    rec: f_max, u, converged, P, F_mod, v_mod, uphill, scale, and for box change pressure, stress, f_box,
    d_eps."""
    x, v, F = (np.array(a, dtype=np.float64).reshape(3, -1) for a in (x, v, F))
    h = np.array(h, dtype=np.float64).reshape(9)
    st = dict(state, v_box=np.array(state["v_box"], dtype=np.float64))
    f_max = np.sqrt(np.max(F * F))
    rec = dict(f_max=f_max, u=float(np.sum(U)))
    P, F2, v2 = float(np.sum(v * F)), float(np.sum(F * F)), float(np.sum(v * v))
    converged = f_max < tol
    if box_change:
        vir = np.asarray(W, dtype=np.float64).reshape(9, -1).sum(axis=1)[list(VIRIAL_ROW_MAJOR)]
        volume = abs(np.linalg.det(h.reshape(3, 3)))
        stress = vir / volume * 160.2176621
        pressure = (stress[0] + stress[4] + stress[8]) / 3.0
        if hydrostatic:
            stress_max = abs(pressure)
            trace = vir[0] + vir[4] + vir[8]
            vir = np.zeros(9)
            vir[[0, 4, 8]] = trace / 3.0
        else:
            stress_max = np.max(np.abs(stress))
        f_box = vir / st["L"]
        P += float(np.dot(st["v_box"], f_box))
        F2 += float(np.dot(f_box, f_box))
        v2 += float(np.dot(st["v_box"], st["v_box"]))
        converged = converged and stress_max < STRESS_TOLERANCE_GPA
        rec.update(pressure=pressure, stress=stress_max, f_box=f_box)
    rec.update(converged=bool(converged), P=P)
    if converged:
        return x, v, h, st, rec
    dt, alpha, n_neg = st["dt"], st["alpha"], st["n_neg"]
    uphill = not P > 0
    if not uphill:
        if n_neg > N_MIN:
            next_dt = dt * F_INC
            if box_change:
                dt = min(next_dt, DT_MAX)  # clamped
            elif next_dt < DT_MAX:
                dt = next_dt               # otherwise left unchanged
            alpha *= F_ALPHA
        n_neg += 1
    else:
        next_dt = dt * F_DEC
        if box_change:
            dt = max(next_dt, DT_MIN)
        elif next_dt > DT_MIN:
            dt = next_dt
        alpha = ALPHA_START
        if not box_change:
            x = x + v * (-0.5 * dt)        # the move-back uses the NEW dt
        v = np.zeros_like(v)
        st["v_box"] = np.zeros(9)
        n_neg = 0
        v2 = 0.0
    F_mod, v_mod = np.sqrt(F2), np.sqrt(v2)
    scale = 0.0 if (box_change and not F_mod > 1e-12) else alpha * v_mod / F_mod
    v = v + F * (dt / MASS)
    v = v * (1 - alpha) + F * scale
    x_old = x
    x = x + v * dt
    if box_change:
        fb = rec["f_box"]
        vb = st["v_box"] + fb * (dt / MASS)
        vb = vb * (1 - alpha) + fb * scale
        st["v_box"] = vb
        d_eps = vb * dt / st["L"]
        E = d_eps.reshape(3, 3)
        x = x + ((E[:, 0:1] * x_old[0] + E[:, 1:2] * x_old[1]) + E[:, 2:3] * x_old[2])  # (x + v dt) + dEps x_old
        h = h + (E @ h.reshape(3, 3)).reshape(9)
        rec["d_eps"] = d_eps
    st.update(dt=dt, alpha=alpha, n_neg=n_neg)
    rec.update(uphill=uphill, F_mod=F_mod, v_mod=v_mod, scale=scale)
    return x, v, h, st, rec


def sd_trial(x, F, f_max, step, label=None, fixed_group=-1):
    """Trial positions x + F step / f_max; atoms of the fixed group stay put (minimizer_sd.cu:32-66)."""
    x, F = np.asarray(x, np.float64).reshape(3, -1), np.asarray(F, np.float64).reshape(3, -1)
    change = F * (step / f_max)
    if fixed_group >= 0:
        change = np.where(np.asarray(label)[None, :] != fixed_group, change, 0.0)
    return x + change


def sd_decide(U, U_trial, step):
    """minimizer_sd.cu:126-137: (uphill, new step, the lower total energy)."""
    u, ut = float(np.sum(U)), float(np.sum(U_trial))
    uphill = ut > u
    return uphill, step * (SD_DECREASE if uphill else SD_INCREASE), (u if uphill else ut)


def _base(number_of_steps):
    return number_of_steps // 10 if number_of_steps >= 10 else 1


def run_sd(compute, x, tol, number_of_steps, label=None, fixed_group=-1):
    """Minimizer_SD::compute (minimizer_sd.cu:70-169).  compute(x) -> (x_wrapped, F, U).
    Returns the final x and the progress lines."""
    x, F, U = compute(np.array(x, np.float64))
    step, lines, base = SD_STEP_0, [], _base(number_of_steps)
    for it in range(number_of_steps):
        f_max = float(np.sqrt(np.max(F * F)))
        if f_max < tol:
            lines.append("    step %d: f_max = %g eV/A." % (it, f_max))
            break
        xt, Ft, Ut = compute(sd_trial(x, F, f_max, step, label, fixed_group))
        uphill, step, u_small = sd_decide(U, Ut, step)
        if not uphill:
            x, F, U = xt, Ft, Ut
        if step < SD_MIN_STEP:
            lines.append("    step %d: total_potential = %.10f eV, f_max = %.10f eV/A." % (it + 1, u_small, f_max))
            lines.append("    Position step is 0, SD minimizer can't find a better solution")
            break
        if it == 0:
            lines.append("    step 0: total_potential = %.10f eV, f_max = %.10f eV/A." % (u_small, f_max))
        if (it + 1) % base == 0:
            lines.append("    step %d: total_potential = %.10f eV, f_max = %.10f eV/A." % (it + 1, u_small, f_max))
    return x, lines


def run_fire(compute, x, h, tol, number_of_steps, box_change=False, hydrostatic=False):
    """Minimizer_FIRE::compute / Minimizer_FIRE_Box_Change::compute.  compute(x, h) -> (x_wrapped, F, U, W).
    Returns the final x, h and the progress lines."""
    x = np.array(x, np.float64).reshape(3, -1)
    h = np.array(h, np.float64).reshape(9)
    v = np.zeros_like(x)
    st = fire_state(L=np.cbrt(abs(np.linalg.det(h.reshape(3, 3)))))
    lines, base = [], _base(number_of_steps)
    for it in range(number_of_steps):
        x, F, U, W = compute(x, h)
        x, v, h, st, rec = fire_step(x, v, F, U, W, h, st, tol, box_change, hydrostatic)
        if it == 0 or (it + 1) % base == 0 or rec["converged"]:
            lines.append(progress_line_fire(0 if it == 0 else it + 1, rec, box_change))
            if rec["converged"]:
                if box_change:
                    lines.append("  Converged! f_max_atom = %.2e < %.2e AND max_stress = %.2e GPa < %.2e GPa"
                                 % (rec["f_max"], tol, rec["stress"], STRESS_TOLERANCE_GPA))
                break
    return x, h, lines


def progress_line_fire(step, rec, box_change):
    if box_change:
        return ("    step %d: total_potential = %.10f eV, f_max_atom = %.10f eV/A, pressure = %.6f GPa."
                % (step, rec["u"], rec["f_max"], rec["pressure"]))
    return "    step %d: total_potential = %.10f eV, f_max = %.10f eV/A." % (step, rec["u"], rec["f_max"])
