// bik_layout.h -- the compiled problem image ("pimage") shared by host builder and device kernels.
//
// bik_problem_create lowers (model blob, task descs, limit descs) into ONE contiguous array of
// 32-bit words: a header of word offsets followed by fp32/int32 tables.  Every CTA stages the image
// into shared memory once (single bulk copy, cp.async.bulk + mbarrier) and then works out of
// shared memory only; a few KB for the BASELINE robots (G1: ~5 KB).
#pragma once
#include <stdint.h>

namespace bik {

enum { JNT_FREE = 0, JNT_BALL = 1, JNT_SLIDE = 2, JNT_HINGE = 3 };
enum { MAX_CFG_LIMITS = 2 };

// words per record
enum { NODE_WORDS = 20, FRAME_WORDS = 36, COMNODE_WORDS = 8, GEOM_WORDS = 16 };
// words per record of the fp64 side tables (kinematic constants for the fp64 instantiation of K1; they sit at the END of the
// image, past PHeader::words32, so that the fp32 kernels neither stage nor pay shared memory for them)
enum { NODE64_WORDS = 28, FRAME64_WORDS = 28, COMNODE64_WORDS = 12, GEOM64_WORDS = 20 };

struct NodeRec {  // 20 words, 16-byte aligned
  int32_t parent, type, qadr, dadr;
  float pos[3];
  float quat[4];
  float axis[3];
  float jpos[3];
  int32_t slot, pslot;   // rows of the per-instance pose state (7 floats each) of this node and of its parent: the state only
  float pad;             // holds the nodes the lane program visits (identity when there is a CoM task or a collision limit)
};
struct FrameRec {  // 32 words.  Column entries: dof | node << 16 | (belongs to the ROOT chain) << 31
  int32_t node;
  float lpos[3];
  float lquat[4];
  float cost[6];
  float gain, lm;
  int32_t ncols, col_off, row0;
  int32_t relative;   // 1: RelativeFrameTask, pose of this frame in the root frame below
  int32_t rnode;
  float rlpos[3];
  float rlquat[4];
  int32_t slot, rslot;   // state rows of `node` / `rnode` (-1: world); filled by the image builder, equal to the node ids in
  float pad;             // frames passed by value to bik_fk (model image: every node is visited)
  int32_t pk_off;        // offset of this task's block in the packed K1 -> K2 record: [ncols][6] Jacobian columns, then e[6]
  int32_t pad2[3];
};
struct NodeRec64 { double pos[3], quat[4], axis[3], jpos[3], pad; };          // 28 words
struct FrameRec64 { double lpos[3], lquat[4], rlpos[3], rlquat[4]; };         // 28 words
struct ComNodeRec64 { double own_m, own_c[3], sub_m, pad; };                  // 12 words
struct GeomRec64 { double lpos[3], lquat[4], size[3]; };                      // 20 words
struct ComNodeRec {  // 8 words: own mass of the node's weld group, its first moment in the node frame, subtree mass
  float own_m, own_c[3], sub_m, pad[3];
};
struct GeomRec {  // 16 words
  int32_t type, node;
  float lpos[3], lquat[4], size[3];
  float pad[4];
};

// Small-group K2 tables.  One frame / CoM task: its block in the packed record and its column schedule.
struct K2TaskRec {  // 8 words
  int32_t nr, nc, coff, row0, pk_off;
  int32_t pairs;  // word offset of int16 [tri(nc)]: packed-triangle offset tri(ua) + ub of H entry (ia, ib), ib <= ia, at tri(ia) + ib
  int32_t ucol;   // word offset of int16 [nc]: coupled index ua of each column
  float lm;
};
struct K2DofRec {  // 12 words: what the box of one dof reads (box_dof), and where the dof sits
  int32_t qa, u;          // qpos address (-1: free / ball dof); coupled index (-1: decoupled)
  float cfg[MAX_CFG_LIMITS][3];   // per ConfigurationLimit: gain, lower, upper
  float vmax;
  int32_t pad[3];
};
struct K2PostRec { double w2, gw2, wg, pad; };   // posture task p, dof d: w^2, (gain w) w, w gain (w = cost_eff[d])
// The small-group K2's tables sit at the end of the image (PHeader::words64), so that no K1 instantiation stages them.  They
// hold problem constants that the step would otherwise re-derive per tile through chains of dependent loads.
struct K2Header {  // 8 words; offsets in words from the start of the image
  int32_t tasks;  // K2TaskRec[F + C]
  int32_t w;      // double[pk_stride]: the weight of every element of the packed record (cost_r, or cost_r (-gain))
  int32_t dofs;   // K2DofRec[nv]
  int32_t post;   // K2PostRec[P][nv]
  int32_t quat;   // int[nquat]: nodes of the free and ball joints (the quaternion update of integrate)
  int32_t nquat;
  int32_t pad[2];
};

struct PHeader {  // all offsets in 32-bit words from the start of the image
  int32_t words;       // total image size in words (multiple of 4)
  int32_t nq, nv, nnode;
  int32_t F, P, C, K;  // frame / posture / com task counts, stacked rows K = 6F + 3C
  int32_t npairs, ngeoms, ncfg, has_vel;
  int32_t G, nsteps;   // lane program: nsteps x G node ids (-1 idle)
  int32_t off_nodes, off_qpos0, off_prog, off_frames, off_cols;
  int32_t off_posture;  // P x { gain, lm, cost_eff[nv] }  (stride 2 + nv)
  int32_t off_com;      // C x { cost[3], gain, lm, row0, pk_off, pad } (8 words each)
  int32_t off_comnodes; // ComNodeRec[nnode]
  int32_t com_cols_off, com_ncols;  // dofs with non-zero CoM column
  int32_t off_cfg;      // ncfg x { gain, pad, lower[nv], upper[nv] } (stride 2 + 2 nv); +-inf where not listed
  int32_t off_vmax;     // float[nv], +inf where not listed
  int32_t off_dofnode;  // int[nv]
  int32_t off_dofqadr;  // int[nv], -1 for free/ball dofs
  int32_t off_range;    // float[2 nv] joint range lo|hi for check_limits (+-inf if unlimited)
  int32_t off_geoms, off_pairs;  // GeomRec[ngeoms], int2[npairs]
  float coll_gain, coll_dmin, coll_ddet, coll_relax;
  float com_total_mass, com_fixed[3];  // total mass of subtree(body 1); first moment of its world-fixed part
  int32_t off_rowinfo;  // float[3 K]: per stacked row cost | gain | lm_damping of its task
  int32_t nu;           // number of COUPLED dofs: columns touched by some task Jacobian or general row
  int32_t off_umap;     // int[nv]: compact index of a coupled dof, -1 for a decoupled one (H row is diagonal there)
  int32_t off_ucols;    // int[nu]: dof of each compact index
  int32_t nrel;         // number of RelativeFrameTasks among the F frame-like tasks
  int32_t nneeded;      // nodes visited by the lane program (ancestors of frames / masses / collision geoms)
  int32_t nfree;        // leading coupled dofs (compact indices 0..nfree-1) without any finite bound: eliminated once by K2
  int32_t nslots;       // rows of the pose state = nodes visited by the lane program (nnode when slots are the identity)
  int32_t k2_sweeps;    // projected Gauss-Seidel sweeps (1..16) that guess the active set before the small-group K2's pivoting
  int32_t k2_rule;      // reserved: nothing reads it (the small-group K2 has one pivoting rule)
  int32_t words32;      // words the fp32 kernels stage (everything before the fp64 side tables)
  int32_t pk_stride;    // elements per instance of the packed K1 -> K2 record (multiple of 4)
  int32_t off_nodes64, off_frames64, off_qpos064, off_comnodes64, off_geoms64;   // fp64 side tables (word offsets, 8-byte aligned)
  int32_t off_com64;    // double { total_mass, fixed[3], coll_gain, coll_dmin, coll_ddet, coll_relax }
  int32_t words64;      // words the fp64 kernels of K1 stage; the small-group K2's tables follow, starting with their K2Header
  int32_t reserved[2];
};
static_assert(sizeof(PHeader) % 16 == 0, "header must stay 16-byte aligned");

}  // namespace bik
