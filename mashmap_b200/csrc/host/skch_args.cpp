#include "skch_args.hpp"

#include <cstdlib>
#include <fstream>
#include <iostream>
#include <map>
#include <sstream>

#include "skch_index.hpp"
#include "skch_stats.hpp"

namespace skch {

namespace {

struct OptDef {
  const char *name;   // canonical long name
  const char *alt;    // alternative (short) name or nullptr
  bool has_value;
};

const OptDef kOptions[] = {
    {"help", "h", false}, {"version", "v", false}, {"ref", "r", true}, {"refList", "rl", true}, {"query", "q", true},
    {"queryList", "ql", true}, {"segLength", "s", true}, {"sketchSize", "J", true}, {"dense", nullptr, false},
    {"blockLength", "l", true}, {"chainGap", "c", true}, {"numMappingsForSegment", "n", true},
    {"numMappingsForShortSeq", nullptr, true}, {"saveIndex", nullptr, true}, {"loadIndex", nullptr, true},
    {"noSplit", nullptr, false}, {"perc_identity", "pi", true}, {"dropLowMapId", "K", false}, {"threads", "t", true},
    {"output", "o", true}, {"kmer", "k", true}, {"kmerThreshold", nullptr, true}, {"kmerComplexity", nullptr, true},
    {"noHgFilter", nullptr, false}, {"hgFilterAniDiff", nullptr, true}, {"hgFilterConf", nullptr, true},
    {"filterLengthMismatches", nullptr, false}, {"lowerTriangular", nullptr, false}, {"skipSelf", "X", false},
    {"skipPrefix", "Y", true}, {"targetPrefix", nullptr, true}, {"targetList", nullptr, true},
    {"sparsifyMappings", "x", true}, {"filter_mode", "f", true}, {"noMerge", "M", false}, {"legacy", nullptr, false},
    {"reportPercentage", nullptr, false},
    // B200-specific
    {"device", nullptr, true}, {"devices", nullptr, true}, {"hostIndex", nullptr, false}, {"batchBases", nullptr, true}, {"subBatchBases", nullptr, true},
    {"align", nullptr, false}, {"alignMaxLen", nullptr, true}, {"eqx", nullptr, false}, {"cs", nullptr, false},
    {"indexShards", nullptr, true},
};

[[noreturn]] void usage_error(const std::string &msg)
{
  std::cerr << msg << std::endl;
  exit(1);
}

void parseFileList(const std::string &listFile, std::vector<std::string> &out)
{  // parseCmdArgs.hpp:141-160
  std::ifstream in(listFile);
  if (!in) usage_error("ERROR, skch::parseFileList, Could not open " + listFile);
  std::string line;
  while (std::getline(in, line))
    if (!line.empty()) out.push_back(line);
}

template <typename T>
T to(const std::string &s)
{
  std::stringstream str;
  str << s;
  T v{};
  str >> v;
  return v;
}

}  // namespace

void printCmdOptions(const Parameters &p)
{  // parseCmdArgs.hpp:209-250
  auto list = [](const std::vector<std::string> &v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? ", " : "") + v[i];
    return s + "]";
  };
  std::cerr << "[mashmap-b200] MashMap v" << fixed::VERSION << std::endl;
  std::cerr << "[mashmap-b200] Reference = " << list(p.refSequences) << std::endl;
  std::cerr << "[mashmap-b200] Query = " << list(p.querySequences) << std::endl;
  std::cerr << "[mashmap-b200] Kmer size = " << p.kmerSize << std::endl;
  std::cerr << "[mashmap-b200] Sketch size = " << p.sketchSize << std::endl;
  std::cerr << "[mashmap-b200] Segment length = " << p.segLength << (p.split ? " (read split allowed)" : " (read split disabled)") << std::endl;
  std::cerr << "[mashmap-b200] Chaining gap max = " << p.chain_gap << std::endl;
  std::cerr << "[mashmap-b200] Mappings per segment = " << p.numMappingsForSegment << std::endl;
  std::cerr << "[mashmap-b200] Percentage identity threshold = " << 100 * p.percentageIdentity << "%" << std::endl;
  std::cerr << "[mashmap-b200] Mapping output file = " << p.outFileName << std::endl;
  std::cerr << "[mashmap-b200] Filter mode = " << p.filterMode << " (1 = map, 2 = one-to-one, 3 = none)" << std::endl;
  std::cerr << "[mashmap-b200] Host threads = " << p.threads << ", CUDA device = " << p.device << std::endl;
  if (p.index_shards > 1) std::cerr << "[mashmap-b200] Index shards = " << p.index_shards << std::endl;
  if (p.align)
    std::cerr << "[mashmap-b200] Alignment = NM:i and cg:Z from edlib NW over each mapping's region, regions up to "
              << p.align_max_len << " bp" << std::endl;
}

void parseandSave(int argc, char **argv, Parameters &parameters)
{
  std::map<std::string, std::string> opt;  // canonical name -> value ("" for flags)
  for (int i = 1; i < argc; i++) {
    std::string a = argv[i];
    if (a.size() < 2 || a[0] != '-') usage_error("ERROR, unexpected argument " + a);
    a = a.substr(a[1] == '-' ? 2 : 1);
    std::string val;
    bool have_val = false;
    const size_t eq = a.find('=');
    if (eq != std::string::npos) { val = a.substr(eq + 1); a = a.substr(0, eq); have_val = true; }
    const OptDef *def = nullptr;
    for (const auto &o : kOptions)
      if (a == o.name || (o.alt && a == o.alt)) { def = &o; break; }
    if (!def) usage_error("ERROR, unknown option " + std::string(argv[i]));
    if (def->has_value && !have_val) {
      if (i + 1 >= argc) usage_error("ERROR, option " + std::string(argv[i]) + " requires a value");
      val = argv[++i];
    }
    opt[def->name] = val;
  }
  auto found = [&](const char *n) { return opt.find(n) != opt.end(); };

  if (found("version")) { std::cerr << fixed::VERSION << std::endl; exit(0); }
  if (found("help")) {
    std::cerr << "mashmap-b200 -r ref.fa -q seq.fq [OPTIONS]   (options as in MashMap v3.1.3, plus --device N | --devices 0-7, --batchBases N,\n"
                 "    --align [--alignMaxLen N, default 100000]: append NM:i and cg:Z (edlib NW over each mapping's region, on the GPU),\n"
                 "    --eqx (with --align): cg:Z with =/X for matches and mismatches instead of M, --cs (with --align): also append\n"
                 "    minimap2's short cs:Z difference string (relative to the target's forward strand, bases in lower case),\n"
                 "    --indexShards N [default 1]: cut the reference index by contig into N device images (shard i on the i-th device of\n"
                 "    --devices, round robin), for references whose index does not fit one GPU; the output is the same)" << std::endl;
    exit(0);
  }
  parameters.align = found("align");
  if (parameters.align && found("legacy"))
    usage_error("ERROR, --align writes PAF tags and cannot be combined with --legacy (mashmap-b200-align aligns --legacy mapping files)");
  if (found("alignMaxLen")) {
    const std::string &v = opt["alignMaxLen"];
    if (!parameters.align) usage_error("ERROR, --alignMaxLen is given without --align");
    if (v.empty() || v.size() > 10 || v.find_first_not_of("0123456789") != std::string::npos || std::stoll(v) < 1)
      usage_error("ERROR, --alignMaxLen needs a positive whole number of bases, not '" + v + "'");
    parameters.align_max_len = std::stoll(v);
  }
  for (const char *o : {"eqx", "cs"})
    if (found(o) && !parameters.align) usage_error(std::string("ERROR, --") + o + " is given without --align");
  parameters.align_eqx = found("eqx");
  parameters.align_cs = found("cs");
  if (!found("ref") && !found("refList")) usage_error("ERROR, skch::parseandSave, Provide reference file(s)");

  if (found("ref")) parameters.refSequences.push_back(opt["ref"]);
  else parseFileList(opt["refList"], parameters.refSequences);
  parameters.referenceSize = (offset_t)CommonFunc::getReferenceSize(parameters.refSequences);  // truncates like the reference (:304)

  if (found("query")) parameters.querySequences.push_back(opt["query"]);
  else if (found("queryList")) parseFileList(opt["queryList"], parameters.querySequences);
  else { parameters.skip_self = true; parameters.querySequences = parameters.refSequences; }

  parameters.lower_triangular = found("lowerTriangular");
  parameters.skip_self = found("skipSelf");  // overwrites the no-query default, as the reference does (:340-345)
  if (found("skipPrefix")) { parameters.prefix_delim = opt["skipPrefix"].empty() ? '\0' : opt["skipPrefix"][0]; parameters.skip_prefix = true; }
  else { parameters.skip_prefix = false; parameters.prefix_delim = '\0'; }
  if (found("targetList")) parameters.target_list = opt["targetList"];
  if (found("targetPrefix")) parameters.target_prefix = opt["targetPrefix"];
  parameters.saveIndexFilename = found("saveIndex") ? opt["saveIndex"] : "";
  parameters.loadIndexFilename = found("loadIndex") ? opt["loadIndex"] : "";

  parameters.alphabetSize = 4;
  parameters.filterLengthMismatches = found("filterLengthMismatches");
  parameters.stage1_topANI_filter = !found("noHgFilter");

  if (found("filter_mode")) {
    const std::string &f = opt["filter_mode"];
    if (f == "map") parameters.filterMode = filter::MAP;
    else if (f == "one-to-one") parameters.filterMode = filter::ONETOONE;
    else if (f == "none") { parameters.stage1_topANI_filter = false; parameters.filterMode = filter::NONE; }
    else usage_error("ERROR, skch::parseandSave, Invalid option given for filter_mode");
  } else {
    parameters.filterMode = filter::MAP;
  }
  parameters.split = !found("noSplit");
  parameters.mergeMappings = !found("noMerge");
  parameters.kmerSize = found("kmer") ? to<int>(opt["kmer"]) : 19;

  if (found("segLength")) {
    parameters.segLength = to<offset_t>(opt["segLength"]);
    if (parameters.segLength < 100)
      usage_error("ERROR, skch::parseandSave, minimum segment length is required to be >= 100 bp.\n"
                  "          This is because Mashmap is not designed for computing short local alignments.\n");
  } else {
    parameters.segLength = 5000;
  }
  if (found("blockLength")) {
    parameters.block_length = to<offset_t>(opt["blockLength"]);
    if (parameters.block_length < 0) usage_error("[mashmap] ERROR, skch::parseandSave, min block length has to be a float value greater than or equal to 0.");
  } else {
    parameters.block_length = parameters.segLength;
  }
  if (found("chainGap")) {
    int64_t l = to<int64_t>(opt["chainGap"]);
    if (l < 0) usage_error("[mashmap] ERROR, skch::parseandSave, chain gap has to be a float value greater than or equal to 0.");
    parameters.chain_gap = l;
  } else {
    parameters.chain_gap = parameters.segLength;
  }
  parameters.keep_low_pct_id = !found("dropLowMapId");
  parameters.kmer_pct_threshold = found("kmerThreshold") ? to<float>(opt["kmerThreshold"]) : 0.001;

  if (found("numMappingsForSegment")) {
    uint32_t n = to<uint32_t>(opt["numMappingsForSegment"]);
    if (n > 0) parameters.numMappingsForSegment = n;
    else usage_error("[mashmap] ERROR, skch::parseandSave, the number of mappings to retain for each segment has to be greater than 0.");
  } else {
    parameters.numMappingsForSegment = 1;
  }
  if (found("numMappingsForShortSeq")) {
    uint32_t n = to<uint32_t>(opt["numMappingsForShortSeq"]);
    if (n > 0) parameters.numMappingsForShortSequence = n;
    else usage_error("[mashmap] ERROR, skch::parseandSave, the number of mappings to retain for each sequence shorter than segment length has to be grater than 0.");
  } else {
    parameters.numMappingsForShortSequence = 1;
  }
  if (found("perc_identity")) {
    parameters.percentageIdentity = to<float>(opt["perc_identity"]);
    if (parameters.percentageIdentity < 50) usage_error("ERROR, skch::parseandSave, minimum nucleotide identity requirement should be >= 50%\n");
    parameters.percentageIdentity /= 100.0;
  } else {
    parameters.percentageIdentity = 0.85;
  }
  parameters.kmerComplexityThreshold = found("kmerComplexity") ? to<float>(opt["kmerComplexity"]) : 0.0;

  if (found("hgFilterAniDiff")) {
    parameters.ANIDiff = to<float>(opt["hgFilterAniDiff"]);
    if (parameters.ANIDiff < 0 || parameters.ANIDiff > 100) usage_error("ERROR, skch::parseandSave, ANI difference must be between 0 and 100");
    parameters.ANIDiff /= 100;
  } else {
    parameters.ANIDiff = fixed::ANIDiff;
  }
  if (found("hgFilterConf")) {
    parameters.ANIDiffConf = to<float>(opt["hgFilterConf"]);
    if (parameters.ANIDiffConf < 0 || parameters.ANIDiffConf > 100) usage_error("ERROR, skch::parseandSave, hypergeometric confidence must be between 0 and 100");
    parameters.ANIDiffConf /= 100;
  } else {
    parameters.ANIDiffConf = fixed::ANIDiffConf;
  }
  parameters.stage2_full_scan = true;  // --shortenCandidateRegions is not defined by the reference either (:101,:590)

  if (found("sparsifyMappings")) {
    double frac = to<double>(opt["sparsifyMappings"]);
    if (frac == 1) parameters.sparsity_hash_threshold = std::numeric_limits<uint64_t>::max();
    else parameters.sparsity_hash_threshold = frac * std::numeric_limits<uint64_t>::max();
  } else {
    parameters.sparsity_hash_threshold = std::numeric_limits<uint64_t>::max();
  }
  parameters.threads = found("threads") ? to<int>(opt["threads"]) : 1;

  if (found("sketchSize")) {
    parameters.sketchSize = to<int>(opt["sketchSize"]);
  } else if (found("dense")) {  // :626-631
    const double md = 1 - parameters.percentageIdentity;
    double dens = 0.02 * (1 + (md / 0.05));
    parameters.sketchSize = dens * (parameters.segLength - parameters.kmerSize);
  } else {
    parameters.sketchSize = Stat::recommendedSketchSize(fixed::pval_cutoff, fixed::confidence_interval, parameters.kmerSize,
                                                        parameters.alphabetSize, parameters.percentageIdentity,
                                                        parameters.segLength, parameters.referenceSize);
  }
  parameters.outFileName = found("output") ? opt["output"] : "mashmap.out";
  parameters.legacy_output = found("legacy");
  parameters.report_ANI_percentage = found("reportPercentage");
  parameters.host_index = found("hostIndex");
  if (found("device")) parameters.device = to<int>(opt["device"]);
  if (found("devices")) {  // "0-7", "0,2,5", "1": the GPUs this process drives; reads are sharded across them by batch parts
    parameters.devices.clear();
    std::stringstream ss(opt["devices"]);
    std::string item;
    while (std::getline(ss, item, ',')) {
      const size_t dash = item.find('-');
      if (dash == std::string::npos) parameters.devices.push_back(to<int>(item));
      else
        for (int d = to<int>(item.substr(0, dash)); d <= to<int>(item.substr(dash + 1)); d++) parameters.devices.push_back(d);
    }
    if (parameters.devices.empty()) usage_error("ERROR, --devices needs a list such as 0-7 or 0,2,5");
    parameters.device = parameters.devices[0];
  }
  if (found("indexShards")) {
    const std::string &v = opt["indexShards"];
    if (v.empty() || v.size() > 9 || v.find_first_not_of("0123456789") != std::string::npos || std::stoll(v) < 1)
      usage_error("ERROR, --indexShards needs a whole number of shards >= 1, not '" + v + "'");
    parameters.index_shards = (int)std::stoll(v);
    if (parameters.index_shards > 1) {
      if (parameters.host_index || !parameters.saveIndexFilename.empty() || !parameters.loadIndexFilename.empty())
        usage_error("ERROR, --indexShards builds every shard on its device: it cannot be combined with --hostIndex, --saveIndex or "
                    "--loadIndex, which build, save or load one unsharded index");
      if (parameters.devices.size() > (size_t)parameters.index_shards)
        usage_error("ERROR, --indexShards " + v + " with " + std::to_string(parameters.devices.size()) +
                    " devices: every device must hold a shard (read-parallel copies of a sharded index are not supported)");
    }
  }
  if (found("batchBases")) parameters.batch_bases = to<uint64_t>(opt["batchBases"]);
  if (found("subBatchBases")) parameters.sub_batch_bases = to<uint64_t>(opt["subBatchBases"]);

  printCmdOptions(parameters);

  for (const auto &f : parameters.querySequences)  // validateInputFiles, parseCmdArgs.hpp:166-203
    if (!std::ifstream(f)) usage_error("ERROR, skch::validateInputFiles, Could not open " + f);
  for (const auto &f : parameters.refSequences)
    if (!std::ifstream(f)) usage_error("ERROR, skch::validateInputFiles, Could not open " + f);
}

}  // namespace skch
