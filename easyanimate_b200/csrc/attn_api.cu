// ea_attn_fwd: argument checks and kernel selection.  The library carries ONE attention kernel (attn_tc6.cu).
#include "host.h"
#include "../../include/ea_b200.h"

namespace ea {
int launch_attn6(const ea_attn_args* g, void* stream);
}  // namespace ea

extern "C" int ea_attn_generations(void) { return 1 << 6; }

extern "C" int ea_attn_fwd(const ea_attn_args* g, void* stream) {
  EA_REQUIRE(g && g->q && g->k && g->v, "ea_attn_fwd: null pointer");
  EA_REQUIRE(g->B > 0 && g->H > 0 && g->S > 0, "ea_attn_fwd: empty problem");
  EA_REQUIRE(g->head_dim == 64, "ea_attn_fwd: head_dim must be 64");
  EA_REQUIRE(g->S_text >= 0 && g->S_text <= g->S, "ea_attn_fwd: bad S_text");
  EA_REQUIRE(g->peers || g->S_text == 0 || g->out_text, "ea_attn_fwd: out_text missing");
  EA_REQUIRE(g->peers || g->S_text == g->S || g->out_video, "ea_attn_fwd: out_video missing");
  EA_REQUIRE(g->B * g->H <= 65535, "ea_attn_fwd: B*H exceeds grid.y");
  EA_REQUIRE((g->variant & 0x1100) == 0x100, "ea_attn_fwd: this build carries the sixth-generation kernel only (variant 0x1?c)");
  return ea::launch_attn6(g, stream);
}
