// lasso_b200 — the checker and slot allocator of the straight-line programs of custom strategies and combining
// functions (host only).  capi.cu runs it on every program a caller hands in; the kernel test harness runs the same
// code, so the instructions it launches are the ones the library would launch.
#pragma once
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.cuh"

namespace lb {

// Checks a straight-line program over alpha inputs (slots 0..alpha-1) with its constants and declared degree (named
// `what` in the reasons) and maps its SSA slots to physical slots: ins receives the instructions, *n_slots_out the
// number of physical slots.  Shared by custom strategies and combining functions.  "" = valid, else the reason.
inline std::string program_check(int alpha, const int32_t* prog, int n_ops, const uint64_t* consts, int n_consts, int degree,
                                 const std::string& what, std::vector<CustomIns>& ins, int* n_slots_out) {
  if (n_ops < 1 || n_ops > kCustomMaxOps) return "the program needs 1..128 instructions";
  if (n_consts < 0 || n_consts > kCustomMaxConsts) return "at most 64 constants";
  if (n_consts > 0 && !consts) return "null constants";
  for (int k = 0; k < n_consts; k++) {
    fr_t x;
    memcpy(x.v, consts + 4 * k, 32);
    if (!fr_eq(fr_reduce_once(x.v), x)) return "constant " + std::to_string(k) + " is not a canonical Montgomery residue";
  }
  // operands refer to earlier slots; degree by propagation (an input has degree 1)
  const int nvals = alpha + n_ops;
  std::vector<int> deg(nvals, 1), last_use(nvals, -1);
  for (int j = 0; j < n_ops; j++) {
    const int op = prog[3 * j], a = prog[3 * j + 1], b = prog[3 * j + 2];
    if (op < CUSTOM_ADD || op > CUSTOM_ADDK) return "instruction " + std::to_string(j) + ": unknown opcode";
    const bool konst = op == CUSTOM_MULK || op == CUSTOM_ADDK;
    if (a < 0 || a >= alpha + j) return "instruction " + std::to_string(j) + ": operand a does not name an earlier slot";
    if (konst ? (b < 0 || b >= n_consts) : (b < 0 || b >= alpha + j))
      return "instruction " + std::to_string(j) + (konst ? ": constant index out of range" : ": operand b does not name an earlier slot");
    int d = op == CUSTOM_MUL ? deg[a] + deg[b] : (konst ? deg[a] : std::max(deg[a], deg[b]));
    deg[alpha + j] = std::min(d, 1 << 20);
    last_use[a] = j;
    if (!konst) last_use[b] = j;
  }
  const int gdeg = deg[nvals - 1];
  if (degree < 1 || degree > kCustomMaxDegree) return what + " must be in 1..16";
  if (degree < gdeg)
    return "declared " + what + " " + std::to_string(degree) + " is below the program's degree " + std::to_string(gdeg);
  // physical slots by liveness: an operand's slot is free again after its last use, before the result is stored
  std::vector<int> phys(nvals, -1), free_slots;
  int n_slots = 0;
  ins.resize(n_ops);
  for (int j = 0; j < n_ops; j++) {
    const int op = prog[3 * j], a = prog[3 * j + 1], b = prog[3 * j + 2];
    const bool konst = op == CUSTOM_MULK || op == CUSTOM_ADDK;
    ins[j].op = op;
    ins[j].a = a < alpha ? -1 - a : phys[a];
    ins[j].b = konst ? b : (b < alpha ? -1 - b : phys[b]);
    for (int v : {a, konst ? -1 : b})
      if (v >= alpha && last_use[v] == j && phys[v] >= 0) {
        free_slots.push_back(phys[v]);
        phys[v] = -1;
      }
    if (j + 1 == n_ops) {
      ins[j].dst = -1;  // g itself stays in registers
      break;
    }
    int s;
    if (!free_slots.empty()) {
      s = free_slots.back();
      free_slots.pop_back();
    } else {
      s = n_slots++;
    }
    ins[j].dst = s;
    if (last_use[alpha + j] < 0) free_slots.push_back(s);  // dead value: stored, never read
    else phys[alpha + j] = s;
  }
  if (n_slots > kCustomMaxSlots) return "the program keeps more than 16 intermediate values live at once";
  *n_slots_out = n_slots;
  return "";
}

}  // namespace lb
