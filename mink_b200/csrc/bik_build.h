// bik_build.h -- host-side lowering: BIKM model blob + task/limit descriptors -> problem image.
// Shared by the C-ABI implementation (bik_api.cu) and the host emulation used by CPU tests.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <limits>
#include <string>
#include <vector>

#include "../../include/bik.h"
#include "bik_layout.h"

namespace bik {

struct HostModel {
  int nq = 0, nv = 0, nnode = 0, ncom = 0;
  std::vector<int32_t> node_parent, node_type, node_qadr, node_dadr, dof_node, dof_qadr, dof_limited, com_node;
  std::vector<double> node_pos, node_quat, node_axis, node_jpos, qpos0, dof_lo, dof_hi, com_pos, com_mass;
};

inline bool blob_section(const uint8_t* blob, size_t nbytes, const char* name, const uint8_t** data, uint32_t* dtype, uint32_t* count) {
  const uint32_t* h = reinterpret_cast<const uint32_t*>(blob);
  uint32_t nsec = h[3];
  for (uint32_t s = 0; s < nsec; ++s) {
    const uint8_t* t = blob + 48 + 32 * s;
    if (48 + 32 * (s + 1) > nbytes) return false;
    if (strncmp(reinterpret_cast<const char*>(t), name, 20) == 0) {
      memcpy(dtype, t + 20, 4); memcpy(count, t + 24, 4);
      uint32_t off; memcpy(&off, t + 28, 4);
      size_t bytes = size_t(*count) * (*dtype == 0 ? 4 : 8);
      if (off + bytes > nbytes) return false;
      *data = blob + off;
      return true;
    }
  }
  return false;
}

inline bool parse_model_blob(const void* blob_, size_t nbytes, HostModel* m, std::string* err) {
  const uint8_t* blob = static_cast<const uint8_t*>(blob_);
  if (nbytes < 48) { *err = "blob too small"; return false; }
  const uint32_t* h = reinterpret_cast<const uint32_t*>(blob);
  if (h[0] != 0x4D4B4942u || h[1] != 1u || h[2] != nbytes) { *err = "not a BIKM v1 blob"; return false; }
  const int32_t* hi = reinterpret_cast<const int32_t*>(blob + 16);
  m->nq = hi[0]; m->nv = hi[1]; m->nnode = hi[2]; m->ncom = hi[3];
  auto geti = [&](const char* name, std::vector<int32_t>* v, size_t expect) {
    const uint8_t* d; uint32_t dt, cnt;
    if (!blob_section(blob, nbytes, name, &d, &dt, &cnt) || dt != 0 || cnt != expect) { *err = std::string("bad section ") + name; return false; }
    v->resize(cnt); if (cnt) memcpy(v->data(), d, cnt * 4); return true;
  };
  auto getd = [&](const char* name, std::vector<double>* v, size_t expect) {
    const uint8_t* d; uint32_t dt, cnt;
    if (!blob_section(blob, nbytes, name, &d, &dt, &cnt) || dt != 1 || cnt != expect) { *err = std::string("bad section ") + name; return false; }
    v->resize(cnt); if (cnt) memcpy(v->data(), d, cnt * 8); return true;
  };
  size_t nn = m->nnode, nv = m->nv, nc = m->ncom;
  return geti("node_parent", &m->node_parent, nn) && geti("node_type", &m->node_type, nn) && geti("node_qadr", &m->node_qadr, nn) &&
         geti("node_dadr", &m->node_dadr, nn) && getd("node_pos", &m->node_pos, 3 * nn) && getd("node_quat", &m->node_quat, 4 * nn) &&
         getd("node_axis", &m->node_axis, 3 * nn) && getd("node_jpos", &m->node_jpos, 3 * nn) && getd("qpos0", &m->qpos0, m->nq) &&
         geti("dof_node", &m->dof_node, nv) && geti("dof_qadr", &m->dof_qadr, nv) && geti("dof_limited", &m->dof_limited, nv) &&
         getd("dof_lo", &m->dof_lo, nv) && getd("dof_hi", &m->dof_hi, nv) && geti("com_node", &m->com_node, nc) &&
         getd("com_pos", &m->com_pos, 3 * nc) && getd("com_mass", &m->com_mass, nc);
}

// List scheduling of the tree onto G lanes: a node may run one step after its parent.
// Priority = height of the subtree below the node (critical path first).
// `needed` (optional): only these nodes are visited -- it must be closed under "parent of".
inline void lane_program(const HostModel& m, int G, std::vector<int32_t>* prog, int* nsteps, const std::vector<char>* needed = nullptr) {
  int n = m.nnode;
  std::vector<int> height(n, 0), done_step(n, -1);
  auto want = [&](int i) { return !needed || (*needed)[i]; };
  for (int i = n - 1; i >= 0; --i) { int p = m.node_parent[i]; if (p >= 0 && want(i)) height[p] = std::max(height[p], height[i] + 1); }
  std::vector<char> done(n, 0);
  int remaining = 0, step = 0;
  for (int i = 0; i < n; ++i) { if (want(i)) ++remaining; else done[i] = 1; }
  prog->clear();
  while (remaining > 0) {
    std::vector<int> ready;
    for (int i = 0; i < n; ++i) if (!done[i]) { int p = m.node_parent[i]; if (p < 0 || (done[p] && want(p) && done_step[p] < step)) ready.push_back(i); }
    std::stable_sort(ready.begin(), ready.end(), [&](int a, int b) { return height[a] > height[b]; });
    for (int g = 0; g < G; ++g) {
      if (g < (int)ready.size()) { int i = ready[g]; prog->push_back(i); done[i] = 1; done_step[i] = step; --remaining; }
      else prog->push_back(-1);
    }
    ++step;
  }
  *nsteps = step;
}

struct ImageBuilder {
  std::vector<uint32_t> w;
  int alloc(int words) { int off = (int)w.size(); w.resize(w.size() + ((words + 3) & ~3), 0u); return off; }
  float* f(int off) { return reinterpret_cast<float*>(w.data() + off); }
  int32_t* i(int off) { return reinterpret_cast<int32_t*>(w.data() + off); }
};

inline void put_frame(const bik_frame& fr, int32_t* node, float* lpos, float* lquat) {
  *node = fr.node;
  double n = sqrt(fr.quat[0] * fr.quat[0] + fr.quat[1] * fr.quat[1] + fr.quat[2] * fr.quat[2] + fr.quat[3] * fr.quat[3]);
  if (!(n > 0)) n = 1;
  for (int k = 0; k < 3; ++k) lpos[k] = (float)fr.pos[k];
  for (int k = 0; k < 4; ++k) lquat[k] = (float)(fr.quat[k] / n);
}

inline void put_frame64(const bik_frame& fr, double* lpos, double* lquat) {
  double n = sqrt(fr.quat[0] * fr.quat[0] + fr.quat[1] * fr.quat[1] + fr.quat[2] * fr.quat[2] + fr.quat[3] * fr.quat[3]);
  if (!(n > 0)) n = 1;
  for (int k = 0; k < 3; ++k) lpos[k] = fr.pos[k];
  for (int k = 0; k < 4; ++k) lquat[k] = fr.quat[k] / n;
}

// Returns false and sets *err on unsupported input.
inline bool build_image(const HostModel& m, const bik_task_desc* tasks, int ntasks, const bik_limit_desc* limits, int nlimits, int G,
                        std::vector<uint32_t>* image, std::string* err) {
  const float INF = std::numeric_limits<float>::infinity();
  ImageBuilder b;
  int hoff = b.alloc(sizeof(PHeader) / 4);
  PHeader H;
  memset(&H, 0, sizeof H);
  H.nq = m.nq; H.nv = m.nv; H.nnode = m.nnode;
  if (m.nv > 64) { *err = "nv > 64 is not supported by the warp-per-problem solver"; return false; }
  if (m.nnode > 32767) { *err = "too many nodes"; return false; }
  for (int t = 0; t < ntasks; ++t) {
    if (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) H.F++;
    else if (tasks[t].kind == BIK_TASK_POSTURE) H.P++;
    else if (tasks[t].kind == BIK_TASK_COM) H.C++;
    else { *err = "unknown task kind"; return false; }
    if (!(tasks[t].gain >= 0.0 && tasks[t].gain <= 1.0)) { *err = "`gain` must be in the range [0, 1]"; return false; }
    if (tasks[t].lm_damping < 0.0) { *err = "`lm_damping` must be >= 0"; return false; }
  }
  H.K = 6 * H.F + 3 * H.C;

  // nodes
  H.off_nodes = b.alloc(NODE_WORDS * m.nnode);
  for (int n = 0; n < m.nnode; ++n) {
    NodeRec r; memset(&r, 0, sizeof r);
    r.parent = m.node_parent[n]; r.type = m.node_type[n]; r.qadr = m.node_qadr[n]; r.dadr = m.node_dadr[n];
    if (r.parent >= n) { *err = "nodes must be ordered parents first"; return false; }
    for (int k = 0; k < 3; ++k) { r.pos[k] = (float)m.node_pos[3 * n + k]; r.axis[k] = (float)m.node_axis[3 * n + k]; r.jpos[k] = (float)m.node_jpos[3 * n + k]; }
    for (int k = 0; k < 4; ++k) r.quat[k] = (float)m.node_quat[4 * n + k];
    memcpy(b.w.data() + H.off_nodes + NODE_WORDS * n, &r, sizeof r);
  }
  H.off_qpos0 = b.alloc(m.nq);
  for (int k = 0; k < m.nq; ++k) b.f(H.off_qpos0)[k] = (float)m.qpos0[k];
  H.off_dofnode = b.alloc(m.nv); H.off_dofqadr = b.alloc(m.nv); H.off_range = b.alloc(2 * m.nv);
  for (int d = 0; d < m.nv; ++d) {
    b.i(H.off_dofnode)[d] = m.dof_node[d]; b.i(H.off_dofqadr)[d] = m.dof_qadr[d];
    b.f(H.off_range)[d] = m.dof_limited[d] ? (float)m.dof_lo[d] : -INF;
    b.f(H.off_range)[m.nv + d] = m.dof_limited[d] ? (float)m.dof_hi[d] : INF;
  }

  // frame tasks + ancestor-dof column lists
  H.off_frames = b.alloc(FRAME_WORDS * std::max(H.F, 1));
  std::vector<int32_t> cols;
  int pk = 0;   // running offset in the packed K1 -> K2 record (frame tasks first, then CoM tasks, each in task order)
  {
    int fi = 0, ci = 0, row = 0;
    for (int t = 0; t < ntasks; ++t) {
      if (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) {
        FrameRec r; memset(&r, 0, sizeof r);
        put_frame(tasks[t].frame, &r.node, r.lpos, r.lquat);
        if (r.node >= m.nnode) { *err = "frame node out of range"; return false; }
        for (int k = 0; k < 6; ++k) { if (tasks[t].cost[k] < 0) { *err = "cost should be >= 0"; return false; } r.cost[k] = (float)tasks[t].cost[k]; }
        r.gain = (float)tasks[t].gain; r.lm = (float)tasks[t].lm_damping; r.row0 = row;
        r.col_off = (int)cols.size();
        r.relative = tasks[t].kind == BIK_TASK_RELATIVE_FRAME;
        H.nrel += r.relative;
        r.rnode = -1;
        std::vector<int> chain_f, chain_r;
        for (int n = r.node; n >= 0; n = m.node_parent[n]) chain_f.push_back(n);
        if (r.relative) {
          put_frame(tasks[t].root, &r.rnode, r.rlpos, r.rlquat);
          if (r.rnode >= m.nnode) { *err = "root frame node out of range"; return false; }
          for (int n = r.rnode; n >= 0; n = m.node_parent[n]) chain_r.push_back(n);
          // dofs of common ancestors move both frames rigidly: their columns vanish identically
          while (!chain_f.empty() && !chain_r.empty() && chain_f.back() == chain_r.back()) { chain_f.pop_back(); chain_r.pop_back(); }
        }
        std::vector<int32_t> mine;
        for (int side = 0; side < 2; ++side)
          for (int n : (side ? chain_r : chain_f)) {
            int nd = m.node_type[n] == JNT_FREE ? 6 : (m.node_type[n] == JNT_BALL ? 3 : 1);
            for (int k = 0; k < nd; ++k) mine.push_back((m.node_dadr[n] + k) | (n << 16) | (side ? (int32_t)0x80000000 : 0));
          }
        std::sort(mine.begin(), mine.end(), [](int32_t a, int32_t b) { return (a & 0xffff) < (b & 0xffff); });
        r.ncols = (int)mine.size();
        r.pk_off = pk;
        pk += 6 * r.ncols + 6;
        cols.insert(cols.end(), mine.begin(), mine.end());
        memcpy(b.w.data() + H.off_frames + FRAME_WORDS * fi, &r, sizeof r);
        ++fi; row += 6;
      } else if (tasks[t].kind == BIK_TASK_COM) { ++ci; row += 3; }
    }
  }
  // CoM bookkeeping (always emitted; cheap) -- mj_jacSubtreeCom(body 1) restated per node.
  H.off_comnodes = b.alloc(COMNODE_WORDS * std::max(m.nnode, 1));
  {
    std::vector<double> own_m(m.nnode, 0.0), sub_m(m.nnode, 0.0), own_c(3 * (size_t)m.nnode, 0.0);
    double total = 0, fixed[3] = {0, 0, 0};
    for (int c = 0; c < m.ncom; ++c) {
      int n = m.com_node[c]; double ms = m.com_mass[c]; total += ms;
      if (n < 0) { for (int k = 0; k < 3; ++k) fixed[k] += ms * m.com_pos[3 * c + k]; continue; }
      own_m[n] += ms; for (int k = 0; k < 3; ++k) own_c[3 * n + k] += ms * m.com_pos[3 * c + k];
    }
    for (int n = m.nnode - 1; n >= 0; --n) { sub_m[n] += own_m[n]; if (m.node_parent[n] >= 0) sub_m[m.node_parent[n]] += sub_m[n]; }
    for (int n = 0; n < m.nnode; ++n) {
      ComNodeRec r; memset(&r, 0, sizeof r);
      r.own_m = (float)own_m[n]; r.sub_m = (float)sub_m[n];
      for (int k = 0; k < 3; ++k) r.own_c[k] = (float)own_c[3 * n + k];
      memcpy(b.w.data() + H.off_comnodes + COMNODE_WORDS * n, &r, sizeof r);
    }
    H.com_total_mass = (float)total;
    for (int k = 0; k < 3; ++k) H.com_fixed[k] = (float)fixed[k];
    H.com_cols_off = (int)cols.size();
    for (int d = 0; d < m.nv; ++d) { int n = m.dof_node[d]; if (sub_m[n] > 0) cols.push_back(d | (n << 16)); }
    H.com_ncols = (int)cols.size() - H.com_cols_off;
    if (H.C > 0 && !(total > 0)) { *err = "ComTask needs a model with mass in the subtree of body 1"; return false; }
  }
  H.off_cols = b.alloc((int)std::max<size_t>(cols.size(), 1));
  if (!cols.empty()) memcpy(b.i(H.off_cols), cols.data(), cols.size() * 4);

  // posture + com task records
  H.off_posture = b.alloc(std::max(H.P, 1) * (2 + m.nv));
  H.off_com = b.alloc(std::max(H.C, 1) * 8);
  {
    int pi = 0, ci = 0, row = 0;
    for (int t = 0; t < ntasks; ++t) {
      if (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) { row += 6; continue; }
      if (tasks[t].kind == BIK_TASK_POSTURE) {
        float* p = b.f(H.off_posture) + pi * (2 + m.nv);
        p[0] = (float)tasks[t].gain; p[1] = (float)tasks[t].lm_damping;
        if (!tasks[t].dof_cost) { *err = "posture task needs dof_cost[nv]"; return false; }
        for (int d = 0; d < m.nv; ++d) {
          if (tasks[t].dof_cost[d] < 0) { *err = "cost should be >= 0"; return false; }
          bool isfree = m.node_type[m.dof_node[d]] == JNT_FREE;
          p[2 + d] = isfree ? 0.f : (float)tasks[t].dof_cost[d];  // e and J are zeroed on free dofs (posture_task.py:115-116,139-140)
        }
        ++pi;
      } else {
        float* p = b.f(H.off_com) + ci * 8;
        for (int k = 0; k < 3; ++k) { if (tasks[t].cost[k] < 0) { *err = "cost must be >= 0"; return false; } p[k] = (float)tasks[t].cost[k]; }
        p[3] = (float)tasks[t].gain; p[4] = (float)tasks[t].lm_damping;
        reinterpret_cast<int32_t*>(p)[5] = row;
        reinterpret_cast<int32_t*>(p)[6] = pk;
        pk += 3 * H.com_ncols + 3;
        ++ci; row += 3;
      }
    }
  }

  H.pk_stride = (pk + 3) & ~3;
  // per-row (cost, gain, lm) table for the stacked rows
  H.off_rowinfo = b.alloc(3 * std::max(H.K, 1));
  {
    int row = 0;
    for (int t = 0; t < ntasks; ++t) {
      int k = (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) ? 6 : (tasks[t].kind == BIK_TASK_COM ? 3 : 0);
      for (int r = 0; r < k; ++r) {
        b.f(H.off_rowinfo)[row + r] = (float)tasks[t].cost[r];
        b.f(H.off_rowinfo)[H.K + row + r] = (float)tasks[t].gain;
        b.f(H.off_rowinfo)[2 * H.K + row + r] = (float)tasks[t].lm_damping;
      }
      row += k;
    }
  }

  // limits
  int ncfg = 0;
  for (int l = 0; l < nlimits; ++l) if (limits[l].kind == BIK_LIMIT_CONFIGURATION) ++ncfg;
  if (ncfg > MAX_CFG_LIMITS) { *err = "at most 2 ConfigurationLimits per problem"; return false; }
  H.ncfg = ncfg;
  H.off_cfg = b.alloc(std::max(ncfg, 1) * (2 + 2 * m.nv));
  H.off_vmax = b.alloc(m.nv);
  for (int d = 0; d < m.nv; ++d) b.f(H.off_vmax)[d] = INF;
  int ci = 0, ncoll = 0;
  for (int l = 0; l < nlimits; ++l) {
    const bik_limit_desc& L = limits[l];
    if (L.kind == BIK_LIMIT_CONFIGURATION) {
      if (!(L.gain > 0.0 && L.gain <= 1.0)) { *err = "ConfigurationLimit gain must be in the range (0, 1]"; return false; }
      float* p = b.f(H.off_cfg) + ci * (2 + 2 * m.nv);
      p[0] = (float)L.gain;
      for (int d = 0; d < m.nv; ++d) { p[2 + d] = -INF; p[2 + m.nv + d] = INF; }
      for (int k = 0; k < L.n; ++k) {
        int d = L.dof[k];
        if (d < 0 || d >= m.nv || m.dof_qadr[d] < 0) { *err = "ConfigurationLimit: only slide/hinge dofs are supported"; return false; }
        p[2 + d] = (float)L.lower[k]; p[2 + m.nv + d] = (float)L.upper[k];
      }
      ++ci;
    } else if (L.kind == BIK_LIMIT_VELOCITY) {
      H.has_vel = 1;
      for (int k = 0; k < L.n; ++k) {
        int d = L.dof[k];
        if (d < 0 || d >= m.nv) { *err = "VelocityLimit dof out of range"; return false; }
        if (m.node_type[m.dof_node[d]] == JNT_FREE) { *err = "Free joint is not supported"; return false; }
        b.f(H.off_vmax)[d] = std::min(b.f(H.off_vmax)[d], (float)L.vmax[k]);
      }
    } else if (L.kind == BIK_LIMIT_COLLISION) {
      if (++ncoll > 1) { *err = "at most one CollisionAvoidanceLimit per problem"; return false; }
      H.ngeoms = L.ngeoms; H.npairs = L.n;
      H.coll_gain = (float)L.gain; H.coll_dmin = (float)L.minimum_distance; H.coll_ddet = (float)L.detection_distance; H.coll_relax = (float)L.bound_relaxation;
      H.off_geoms = b.alloc(GEOM_WORDS * std::max(L.ngeoms, 1)); H.off_pairs = b.alloc(2 * std::max(L.n, 1));
      for (int g = 0; g < L.ngeoms; ++g) {
        GeomRec r; memset(&r, 0, sizeof r);
        r.type = L.geoms[g].type;
        if (r.type != BIK_GEOM_PLANE && r.type != BIK_GEOM_SPHERE && r.type != BIK_GEOM_CAPSULE && r.type != BIK_GEOM_BOX) { *err = "collision geoms must be plane, sphere, capsule or box"; return false; }
        put_frame(L.geoms[g].frame, &r.node, r.lpos, r.lquat);
        for (int k = 0; k < 3; ++k) r.size[k] = (float)L.geoms[g].size[k];
        memcpy(b.w.data() + H.off_geoms + GEOM_WORDS * g, &r, sizeof r);
      }
      for (int k = 0; k < 2 * L.n; ++k) {
        if (L.pairs[k] < 0 || L.pairs[k] >= L.ngeoms) { *err = "collision pair index out of range"; return false; }
        b.i(H.off_pairs)[k] = L.pairs[k];
      }
      for (int k = 0; k < L.n; ++k) {
        const int t1 = L.geoms[L.pairs[2 * k]].type, t2 = L.geoms[L.pairs[2 * k + 1]].type;
        if (t1 == BIK_GEOM_PLANE && t2 == BIK_GEOM_PLANE) { *err = "plane-plane pair"; return false; }
        if (t1 == BIK_GEOM_BOX && t2 == BIK_GEOM_BOX) { *err = "box-box pairs are not supported (no convex-convex distance on the device)"; return false; }
      }
    } else { *err = "unknown limit kind"; return false; }
  }
  if (!H.off_geoms) { H.off_geoms = b.alloc(GEOM_WORDS); H.off_pairs = b.alloc(4); }
  // coupled dofs: a dof whose column is zero in every task Jacobian and every general row only sees the
  // diagonal of H, so its optimum is a closed-form clamp; the QP proper runs on the coupled set.
  {
    std::vector<char> coupled(m.nv, 0);
    for (size_t k = 0; k < cols.size(); ++k) {
      bool is_com = (int)k >= H.com_cols_off && (int)k < H.com_cols_off + H.com_ncols;
      if (is_com && H.C == 0) continue;
      coupled[cols[k] & 0xffff] = 1;
    }
    if (H.npairs > 0) std::fill(coupled.begin(), coupled.end(), 1);
    H.off_umap = b.alloc(std::max(m.nv, 1));
    std::vector<int32_t> ucols;
    for (int d = 0; d < m.nv; ++d) { b.i(H.off_umap)[d] = coupled[d] ? (int)ucols.size() : -1; if (coupled[d]) ucols.push_back(d); }
    H.nu = (int)ucols.size();
    H.off_ucols = b.alloc(std::max(H.nu, 1));
    for (int k = 0; k < H.nu; ++k) b.i(H.off_ucols)[k] = ucols[k];
    // Leading coupled dofs that no limit bounds (free-joint dofs, unlimited joints without a velocity limit): the QP is
    // minimised over them in closed form once, the active-set iterations run on the rest (bik_k2t.h).  Only a prefix
    // of the (ascending) coupled list qualifies, which is where MuJoCo's dof order puts a floating base.
    H.nfree = 0;
    H.k2_sweeps = 3;   // BIK_K2_SWEEPS overrides it (bik_problem_create)
    if (H.npairs == 0) {
      auto bounded = [&](int d) {
        if (b.f(H.off_vmax)[d] < INF) return true;
        for (int c = 0; c < ncfg; ++c) {
          const float* p = b.f(H.off_cfg) + c * (2 + 2 * m.nv);
          if (p[2 + d] > -INF || p[2 + m.nv + d] < INF) return true;
        }
        return false;
      };
      while (H.nfree < H.nu && !bounded(ucols[H.nfree])) ++H.nfree;
    }
  }
  // Lane program over the nodes the outputs depend on: ancestors of task frames / roots, of collision geoms
  // and (CoM tasks) of every massive body.  mj_kinematics visits every body; nothing downstream of this
  // path reads the others (G1 headline config: 13 of 38 nodes).  Without tasks (model image used by
  // bik_fk / bik_frame_jacobian) every node is visited.
  {
    std::vector<char> needed(m.nnode, ntasks == 0 && nlimits == 0 ? 1 : 0);
    auto mark = [&](int n) { for (; n >= 0 && !needed[n]; n = m.node_parent[n]) needed[n] = 1; };
    for (int t = 0; t < ntasks; ++t)
      if (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) {
        mark(tasks[t].frame.node);
        if (tasks[t].kind == BIK_TASK_RELATIVE_FRAME) mark(tasks[t].root.node);
      }
    if (H.C > 0) for (int c = 0; c < m.ncom; ++c) mark(m.com_node[c]);
    for (int l = 0; l < nlimits; ++l)
      if (limits[l].kind == BIK_LIMIT_COLLISION) for (int g = 0; g < limits[l].ngeoms; ++g) mark(limits[l].geoms[g].frame.node);
    int cnt = 0; for (char c : needed) cnt += c;
    // G <= 0: pick the lanes per instance from the visited tree -- wide enough that the per-warp tile stays small
    // (occupancy), narrow enough that the program keeps the lanes busy
    if (G <= 0) G = cnt > 4 ? 4 : 2;
    H.G = G;
    std::vector<int32_t> prog; int nsteps = 0;
    lane_program(m, G, &prog, &nsteps, &needed);
    H.nsteps = nsteps;
    H.off_prog = b.alloc((int)std::max<size_t>(prog.size(), 1));
    if (!prog.empty()) memcpy(b.i(H.off_prog), prog.data(), prog.size() * 4);
    H.nneeded = cnt;
    // Rows of K1's per-instance pose state: only visited nodes get one (G1 headline config: 13 rows instead of 38, which
    // is what bounds the resident warps of K1).  CoM tasks index first moments by node id and collision geoms are posed
    // through node ids, so those problems keep the identity.
    const bool compact = cnt < m.nnode && H.C == 0 && H.npairs == 0;
    std::vector<int32_t> slot(m.nnode, -1);
    int ns = 0;
    for (int n = 0; n < m.nnode; ++n) slot[n] = compact ? (needed[n] ? ns++ : -1) : n;
    H.nslots = compact ? ns : m.nnode;
    for (int n = 0; n < m.nnode; ++n) {
      NodeRec* r = reinterpret_cast<NodeRec*>(b.w.data() + H.off_nodes + NODE_WORDS * n);
      r->slot = slot[n];
      r->pslot = r->parent >= 0 ? slot[r->parent] : -1;
    }
    for (int f = 0; f < H.F; ++f) {
      FrameRec* r = reinterpret_cast<FrameRec*>(b.w.data() + H.off_frames + FRAME_WORDS * f);
      r->slot = r->node >= 0 ? slot[r->node] : -1;
      r->rslot = (r->relative && r->rnode >= 0) ? slot[r->rnode] : -1;
    }
  }
  // fp64 side tables: the kinematic constants at full precision for the fp64 instantiation of K1 (ill-conditioned problems:
  // an fp32-rounded link offset moves e by ~1e-7, which cost / (2 sqrt(damping)) can amplify past the 1e-4 rad budget)
  H.words32 = (int)b.w.size();
  {
    H.off_nodes64 = b.alloc(NODE64_WORDS * std::max(m.nnode, 1));
    for (int n = 0; n < m.nnode; ++n) {
      NodeRec64 r; memset(&r, 0, sizeof r);
      for (int k = 0; k < 3; ++k) { r.pos[k] = m.node_pos[3 * n + k]; r.axis[k] = m.node_axis[3 * n + k]; r.jpos[k] = m.node_jpos[3 * n + k]; }
      for (int k = 0; k < 4; ++k) r.quat[k] = m.node_quat[4 * n + k];
      memcpy(b.w.data() + H.off_nodes64 + NODE64_WORDS * n, &r, sizeof r);
    }
    H.off_frames64 = b.alloc(FRAME64_WORDS * std::max(H.F, 1));
    int fi = 0;
    for (int t = 0; t < ntasks; ++t)
      if (tasks[t].kind == BIK_TASK_FRAME || tasks[t].kind == BIK_TASK_RELATIVE_FRAME) {
        FrameRec64 r; memset(&r, 0, sizeof r);
        put_frame64(tasks[t].frame, r.lpos, r.lquat);
        if (tasks[t].kind == BIK_TASK_RELATIVE_FRAME) put_frame64(tasks[t].root, r.rlpos, r.rlquat);
        memcpy(b.w.data() + H.off_frames64 + FRAME64_WORDS * fi, &r, sizeof r);
        ++fi;
      }
    H.off_qpos064 = b.alloc(2 * std::max(m.nq, 1));
    memcpy(b.w.data() + H.off_qpos064, m.qpos0.data(), sizeof(double) * m.nq);
    H.off_comnodes64 = b.alloc(COMNODE64_WORDS * std::max(m.nnode, 1));
    H.off_com64 = b.alloc(16);   // { total mass, fixed first moment[3], collision gain, minimum / detection distance, relaxation }
    {
      std::vector<double> own_m(m.nnode, 0.0), sub_m(m.nnode, 0.0), own_c(3 * (size_t)m.nnode, 0.0);
      double tot[4] = {0, 0, 0, 0};
      for (int c = 0; c < m.ncom; ++c) {
        int n = m.com_node[c]; double ms = m.com_mass[c]; tot[0] += ms;
        if (n < 0) { for (int k = 0; k < 3; ++k) tot[1 + k] += ms * m.com_pos[3 * c + k]; continue; }
        own_m[n] += ms; for (int k = 0; k < 3; ++k) own_c[3 * n + k] += ms * m.com_pos[3 * c + k];
      }
      for (int n = m.nnode - 1; n >= 0; --n) { sub_m[n] += own_m[n]; if (m.node_parent[n] >= 0) sub_m[m.node_parent[n]] += sub_m[n]; }
      for (int n = 0; n < m.nnode; ++n) {
        ComNodeRec64 r; memset(&r, 0, sizeof r);
        r.own_m = own_m[n]; r.sub_m = sub_m[n];
        for (int k = 0; k < 3; ++k) r.own_c[k] = own_c[3 * n + k];
        memcpy(b.w.data() + H.off_comnodes64 + COMNODE64_WORDS * n, &r, sizeof r);
      }
      memcpy(b.w.data() + H.off_com64, tot, sizeof tot);
      double coll[4] = {0, 0, 0, 0};
      for (int l = 0; l < nlimits; ++l)
        if (limits[l].kind == BIK_LIMIT_COLLISION) { coll[0] = limits[l].gain; coll[1] = limits[l].minimum_distance; coll[2] = limits[l].detection_distance; coll[3] = limits[l].bound_relaxation; }
      memcpy(b.w.data() + H.off_com64 + 8, coll, sizeof coll);
    }
    H.off_geoms64 = b.alloc(GEOM64_WORDS * std::max(H.ngeoms, 1));
    for (int l = 0; l < nlimits; ++l)
      if (limits[l].kind == BIK_LIMIT_COLLISION)
        for (int g = 0; g < limits[l].ngeoms; ++g) {
          GeomRec64 r; memset(&r, 0, sizeof r);
          put_frame64(limits[l].geoms[g].frame, r.lpos, r.lquat);
          for (int k = 0; k < 3; ++k) r.size[k] = limits[l].geoms[g].size[k];
          memcpy(b.w.data() + H.off_geoms64 + GEOM64_WORDS * g, &r, sizeof r);
        }
  }
  // K2 tables (bik_k2t.h reads them; see PHeader).  Every value is derived from the fp32 records above exactly as the kernel
  // derived it per tile, and the products are exact or rounded once in double as the kernel rounds them, so K2's results do
  // not change.  (b.alloc reallocates: the tables above are copied out first.)
  H.words64 = (int)b.w.size();
  {
    const int nt = H.F + H.C, nv = m.nv;
    const std::vector<int32_t> umap(b.i(H.off_umap), b.i(H.off_umap) + nv);
    const std::vector<float> posture(b.f(H.off_posture), b.f(H.off_posture) + H.P * (2 + nv));
    const std::vector<float> cfg(b.f(H.off_cfg), b.f(H.off_cfg) + ncfg * (2 + 2 * nv));
    const std::vector<float> vmax(b.f(H.off_vmax), b.f(H.off_vmax) + nv);
    const std::vector<float> com(b.f(H.off_com), b.f(H.off_com) + 8 * H.C);
    K2Header kh; memset(&kh, 0, sizeof kh);
    const int khoff = b.alloc(8);
    kh.tasks = b.alloc(8 * std::max(nt, 1));
    kh.w = b.alloc(2 * std::max(H.pk_stride, 1));
    for (int t = 0; t < nt; ++t) {
      K2TaskRec k; memset(&k, 0, sizeof k);
      float cost[6], gain;
      if (t < H.F) {
        FrameRec fr; memcpy(&fr, b.w.data() + H.off_frames + FRAME_WORDS * t, sizeof fr);
        k.nr = 6; k.nc = fr.ncols; k.coff = fr.col_off; k.row0 = fr.row0; k.pk_off = fr.pk_off; k.lm = fr.lm;
        memcpy(cost, fr.cost, sizeof cost); gain = fr.gain;
      } else {
        const float* cr = com.data() + 8 * (t - H.F);
        k.nr = 3; k.nc = H.com_ncols; k.coff = H.com_cols_off; memcpy(&k.row0, cr + 5, 4); memcpy(&k.pk_off, cr + 6, 4); k.lm = cr[4];
        memcpy(cost, cr, 3 * sizeof(float)); gain = cr[3];
      }
      for (int e = 0; e < k.nr * k.nc; ++e) reinterpret_cast<double*>(b.w.data() + kh.w)[k.pk_off + e] = (double)cost[e % k.nr];
      for (int r = 0; r < k.nr; ++r) reinterpret_cast<double*>(b.w.data() + kh.w)[k.pk_off + k.nr * k.nc + r] = (double)cost[r] * (double)(-gain);
      // pair schedule of k2t_task_accumulate_nr: where H entry (ia, ib), ib <= ia, lands in the packed triangle
      k.pairs = b.alloc((k.nc * (k.nc + 1) / 2 + 1) / 2);
      k.ucol = b.alloc((k.nc + 1) / 2);
      int16_t* pairs = reinterpret_cast<int16_t*>(b.w.data() + k.pairs);
      int16_t* ucol = reinterpret_cast<int16_t*>(b.w.data() + k.ucol);
      for (int ia = 0; ia < k.nc; ++ia) {
        const int ua = umap[cols[k.coff + ia] & 0xffff];
        ucol[ia] = (int16_t)ua;
        for (int ib = 0; ib <= ia; ++ib) {
          const int ub = umap[cols[k.coff + ib] & 0xffff], hi = std::max(ua, ub), lo = std::min(ua, ub);
          pairs[ia * (ia + 1) / 2 + ib] = (int16_t)(hi * (hi + 1) / 2 + lo);
        }
      }
      memcpy(b.w.data() + kh.tasks + 8 * t, &k, sizeof k);
    }
    kh.dofs = b.alloc(12 * std::max(nv, 1));
    for (int d = 0; d < nv; ++d) {
      K2DofRec r; memset(&r, 0, sizeof r);
      r.qa = m.dof_qadr[d]; r.u = umap[d]; r.vmax = vmax[d];
      for (int c = 0; c < ncfg; ++c) {
        const float* p = cfg.data() + c * (2 + 2 * nv);
        r.cfg[c][0] = p[0]; r.cfg[c][1] = p[2 + d]; r.cfg[c][2] = p[2 + nv + d];
      }
      memcpy(b.w.data() + kh.dofs + 12 * d, &r, sizeof r);
    }
    // w^2 is exact in double, as is w gain; (gain w) w rounds once, as the kernel's left-to-right product did
    kh.post = b.alloc(8 * std::max(H.P * nv, 1));
    for (int p = 0; p < H.P; ++p)
      for (int d = 0; d < nv; ++d) {
        const double g = posture[p * (2 + nv)], w = posture[p * (2 + nv) + 2 + d];
        K2PostRec r = {w * w, (g * w) * w, w * g, 0.0};
        memcpy(b.w.data() + kh.post + 8 * (p * nv + d), &r, sizeof r);
      }
    std::vector<int32_t> quat;
    for (int n = 0; n < m.nnode; ++n) if (m.node_type[n] == JNT_FREE || m.node_type[n] == JNT_BALL) quat.push_back(n);
    kh.nquat = (int)quat.size();
    kh.quat = b.alloc(std::max(kh.nquat, 1));
    if (!quat.empty()) memcpy(b.i(kh.quat), quat.data(), quat.size() * 4);
    memcpy(b.w.data() + khoff, &kh, sizeof kh);
  }
  H.words = (int)b.w.size();
  memcpy(b.w.data() + hoff, &H, sizeof H);
  *image = b.w;
  return true;
}

// Conditioning estimate for the automatic choice of K1's precision: the error e enters dq amplified by about
// cost / (2 sqrt(regularisation)); regularisation = damping + the smallest posture weight on a coupled dof.
// max_cost2: largest squared frame / CoM task cost.  min_post2: smallest squared posture cost over the coupled dofs outside
// free joints (0 when there is none).
struct K1Conditioning { double max_cost2 = 0, min_post2 = 0; };
inline K1Conditioning k1_conditioning(const HostModel& m, const std::vector<uint32_t>& image, const bik_task_desc* tasks, int ntasks) {
  double mc = 0, mp = std::numeric_limits<double>::infinity();
  for (int t = 0; t < ntasks; ++t) {
    if (tasks[t].kind == BIK_TASK_POSTURE) continue;
    const int nr = tasks[t].kind == BIK_TASK_COM ? 3 : 6;
    for (int r = 0; r < nr; ++r) mc = std::max(mc, tasks[t].cost[r] * tasks[t].cost[r]);
  }
  const PHeader& h = *reinterpret_cast<const PHeader*>(image.data());
  const int32_t* ucols = reinterpret_cast<const int32_t*>(image.data() + h.off_ucols);
  for (int k = 0; k < h.nu; ++k) {
    const int d = ucols[k];
    if (m.node_type[m.dof_node[d]] == JNT_FREE) continue;
    double s = 0;
    for (int t = 0; t < ntasks; ++t) if (tasks[t].kind == BIK_TASK_POSTURE) s += tasks[t].dof_cost[d] * tasks[t].dof_cost[d];
    mp = std::min(mp, s);
  }
  K1Conditioning k;
  k.max_cost2 = mc;
  k.min_post2 = std::isfinite(mp) ? mp : 0.0;
  return k;
}
// Whether K1 runs in fp64 for an fp32 caller of this problem and damping (BIK_K1_PRECISION aside).  posture_weighted: the call
// scales the posture costs per instance (..._weighted_ex with posture weights), possibly down to 0, so only the damping is
// certain to regularise.
inline bool k1_auto_double(const PHeader& h, const K1Conditioning& k, double damping, bool posture_weighted = false) {
  if (h.npairs > 0) return true;   // contact points of nearly parallel capsules are ill-conditioned in fp32
  const double reg = damping + (posture_weighted ? 0.0 : k.min_post2);
  return !(reg > 0) || k.max_cost2 / reg > 1e6;
}

}  // namespace bik
