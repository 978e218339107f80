#pragma once
#include <vector>

#include "ir.h"
#include "vm.h"

namespace b200q {

struct OutDesc { DType type; bool nullable; int slots; };

struct CompiledProgram {
  VmProgram prog;
  std::vector<int> used_cols;   // program column slot -> index in the stage's input schema
  std::vector<OutDesc> outs;
  bool has_strings = false;          // reads a Utf8 column or uses a Utf8 constant: only the generic VM kernels run it
  std::vector<uint32_t> str_relocs;  // pool indices holding a str_pool offset, to be turned into a device address at upload
  bool vm_only = false;              // uses VM_XXHASH64 / VM_BLOOM_PROBE, which only the generic VM kernels implement
  // bloom filters probed by the program: pool[pool_index] becomes the device address of the uploaded words
  struct BloomRef { uint32_t pool_index; std::shared_ptr<const BloomFilterDef> filter; };
  std::vector<BloomRef> blooms;
};

// filters: conjuncts in evaluation order; outs: projections (FilterExec/ProjectExec kernel) or
// grouping keys followed by aggregate arguments (HashAgg kernel).
// sel_out >= 0: after the outputs, the source row of each surviving row is written to output `sel_out` (VM_OUT_SEL)
CompiledProgram compile_program(const std::vector<ExprP>& filters, const std::vector<ExprP>& outs, bool with_compact, int sel_out = -1);

// the program with its Utf8 constants relocated to `device_copy`, the address it will live at on the device
VmProgram relocated_program(const CompiledProgram& cp, const void* device_copy);

// replace column references by the expressions that define them (fusing Project/Filter chains)
ExprP substitute(const ExprP& e, const std::vector<ExprP>& cols);

PhysKind phys_of(const DType& t);

}  // namespace b200q
