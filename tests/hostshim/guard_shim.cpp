// guard_shim.cpp — test shim: the library's own pdb and cdp votes compiled by g++ for the CPU tests: the host vote
// (vch::EvictSession::tier_victims with one voter, used by preempt's normal reading and by reclaim) and the dry run's vote
// (vct::topo_vote<true> on the bits vch::VictimGuards::device_bits derives, as vcalloc.cu stages them). Not part of the
// product; nothing here is an alternative compute path.
#include "../../volcano_b200/csrc/vc_evict.hpp"

#include <cstring>

extern "C" {

// plugin: VC_PLUGIN_PDB or VC_PLUGIN_CDP; the table as vc_victim_guards; cands: running-task indices in node.Tasks order.
// host_out / dev_out [m]: 1 when the host vote / the dry run's vote returns cands[i]. Returns 0.
int gs_votes(int plugin, const vc_victim_guards *vg, const int32_t *cands, int m, uint8_t *host_out, uint8_t *dev_out) {
  const int n = vg->n_running;
  vch::VictimGuards g;
  g.n_running = n; g.now_ns = vg->now_ns;
  g.allowed.assign(vg->pdb_allowed, vg->pdb_allowed + vg->n_pdb);
  g.off.assign(vg->rt_pdb_off, vg->rt_pdb_off + n + 1);
  g.pdb.assign(vg->rt_pdb, vg->rt_pdb + g.off[n]);
  g.flags.assign(vg->rt_flags, vg->rt_flags + n);
  g.until.assign(vg->rt_cooldown_until_ns, vg->rt_cooldown_until_ns + n);
  vc_conf conf;
  std::memset(&conf, 0, sizeof conf);
  conf.n_plugins = 1;
  conf.plugins[0].plugin = plugin; conf.plugins[0].tier = 0; conf.plugins[0].enabled = VC_EN_PREEMPTABLE;
  vch::EvictSession e;
  e.conf = &conf;
  e.g = &g;
  const std::vector<int> c(cands, cands + m);
  const std::vector<int> v = e.tier_victims(0, c, false);
  for (int i = 0; i < m; ++i) host_out[i] = std::find(v.begin(), v.end(), c[i]) != v.end() ? 1 : 0;
  std::vector<uint8_t> bits((size_t)std::max(n, 1));
  for (int r = 0; r < n; ++r) bits[r] = g.device_bits(r);
  std::vector<int32_t> job((size_t)std::max(n, 1), 0);
  vct::TopoView tv;
  std::memset(&tv, 0, sizeof tv);
  tv.rt_job = job.data(); tv.rt_guard = bits.data(); tv.pdb_off = g.off.data(); tv.pdb = g.pdb.data();
  tv.pdb_allowed = g.allowed.data();
  vct::TopoTask tt;
  std::memset(&tt, 0, sizeof tt);
  vct::topo_vote<true>(tv, tt, plugin, cands, m, dev_out);
  return 0;
}

}  // extern "C"
