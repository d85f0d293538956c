"""TEST INFRASTRUCTURE -- the rollout oracle (oracle/rollout_oracle.py) with mesh obstacles in the scene term.

The fused kernels add each sphere's mesh terms to its cuboid + ESDF terms, and grad_q is linear in the sphere gradients, so the
evaluation with meshes is the oracle's evaluation without them plus the mesh terms' cost and their J^T (oracle fk_backward).  The
mesh SDF is oracle/mesh_oracle.mesh_sdf_grad -- brute-force closest point with a ray-parity sign, sharing neither the BVH nor the
pseudo-normal sign with the product -- queried with query_distance = r + eta, as the product's obstacle_sdf does.  Discrete
collision only (the IK rows)."""
import numpy as np

from curobo_b200.world import _inv_pose_from_pose
from oracle import mesh_oracle as MO
from oracle import rollout_oracle as O

F = np.float32


def mesh_scene_collision(spheres, weight, eta, world_mesh, env_query_idx=None, enable=None):
    """cost [B,H,S] and gradient [B,H,S,4] of the mesh obstacles of `world_mesh` (curobo_b200.mesh.MeshWorld), discrete
    (wp_collision_kernel.py:112-166 with data_mesh.py:643-700 as the SDF).  enable [n_env, max_n] (optional): 0 skips a slot."""
    sph = np.asarray(spheres, F)
    B, H, S, _ = sph.shape
    w, eta = F(weight), F(eta)
    cost = np.zeros((B, H, S), F)
    grad = np.zeros((B, H, S, 4), F)
    envs = np.zeros(B, np.int64) if env_query_idx is None else np.asarray(env_query_idx).astype(np.int64)
    for env in np.unique(envs):
        e = int(env) if env < len(world_mesh.envs) else 0
        bsel = np.nonzero(envs == env)[0]
        sp = sph[bsel].reshape(-1, 4)
        c_env = np.zeros(sp.shape[0], F)
        g_env = np.zeros((sp.shape[0], 3), F)
        for i, m in enumerate(world_mesh.envs[e][:world_mesh.max_n]):
            if enable is not None and int(enable[e][i]) != 1:
                continue
            ip, iq = O._load_inv_transform(_inv_pose_from_pose(m.get("pose", (0, 0, 0, 1, 0, 0, 0))))
            loc = O._quat_rotate(np.broadcast_to(iq, (sp.shape[0], 4)), sp[:, :3]) + ip
            fq = np.array([-iq[0], -iq[1], -iq[2], iq[3]], F)
            radj = (sp[:, 3] + eta).astype(F)
            for r in np.unique(radj[sp[:, 3] >= 0]):
                sel = np.nonzero((radj == r) & (sp[:, 3] >= 0))[0]
                sdf, gl = MO.mesh_sdf_grad(m["vertices"], m["faces"], loc[sel], query_distance=float(r))
                pen = (r - sdf).astype(F)
                ac, ak = O.collision_activation(pen, eta)
                hit = pen > 0
                c_env[sel] += np.where(hit, w * ac, F(0)).astype(F)
                gw = O._quat_rotate(np.broadcast_to(fq, (sel.shape[0], 4)), gl)
                g_env[sel] += np.where(hit[:, None], (w * ak)[:, None] * gw, F(0)).astype(F)
        cost[bsel] = c_env.reshape(len(bsel), H, S)
        grad[bsel, ..., :3] = g_env.reshape(len(bsel), H, S, 3)
    return cost, grad


def rollout_cost_grad(rm, q, cfg, world_mesh=None, mesh_enable=None, **kw):
    """oracle/rollout_oracle.rollout_cost_grad(rm, q, cfg, **kw) with the mesh obstacles of `world_mesh` added."""
    out = O.rollout_cost_grad(rm, q, cfg, **kw)
    if world_mesh is None or cfg.get("scene_weight", 0) <= 0:
        return out
    if cfg.get("sweep"):
        raise NotImplementedError("mesh oracle: discrete collision only")
    if np.asarray(rm.link_spheres).ndim == 3 and np.asarray(rm.link_spheres).shape[0] > 1:
        raise NotImplementedError("mesh oracle: one link-sphere configuration only")
    B, H, D = np.asarray(q).shape
    c, g = mesh_scene_collision(out["spheres"], cfg["scene_weight"], cfg.get("scene_eta", 0.0), world_mesh,
                                kw.get("env_query_idx"), mesh_enable)
    gq = O.fk_backward(rm, out["cumul"], g.reshape(B * H, -1, 4), None, None).reshape(B, H, D)
    out["scene_cost"] = (out["scene_cost"] + c).astype(F) if "scene_cost" in out else c
    out["grad_q"] = (out["grad_q"] + gq).astype(F)
    out["cost_bh"] = (out["cost_bh"] + np.sum(c, axis=-1)).astype(F)
    out["cost"] = np.sum(out["cost_bh"], axis=1).astype(F)
    return out
