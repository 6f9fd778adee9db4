// Lighthouse server: heartbeat table, participants of the in-flight round, tick loop, quorum broadcast,
// dashboard + kill endpoint. Behavioural reference: src/lighthouse.rs (State :57-66, _quorum_tick :292-343,
// RPC quorum :484-551 incl. "a quorum request counts as a heartbeat", heartbeat :553-566, get_status :415-452,
// kill :454-479). Differences: waiters replay missed generations from a short history (the reference uses a
// tokio broadcast channel), the dashboard is plain JS polling /status, and /status.json + quorum_id_base exist.
#include "lighthouse.h"

#include <algorithm>
#include <cstdio>
#include <sstream>

#include "manager_server.h"

namespace tft {

static void log_info(const std::string& msg) {
  static const bool quiet = [] {
    const char* e = getenv("TORCHFT_B200_LOG");
    return !(e && (std::string(e) == "info" || std::string(e) == "debug"));
  }();
  if (!quiet) fprintf(stderr, "[torchft_b200 lighthouse] %s\n", msg.c_str());
}

Lighthouse::Lighthouse(LighthouseOpt opt) : opt_(std::move(opt)) {
  if (opt_.quorum_id_base < 0) opt_.quorum_id_base = (unix_ms() - 1735689600000ll) / 250;  // quarter seconds since 2025-01-01
  state_.quorum_id = opt_.quorum_id_base;
  start(opt_.bind, "tft-lighths");
  tick_thread_ = std::thread([this] {
    name_this_thread("tft-lighths-tick");
    tick_loop();
  });
}

Lighthouse::~Lighthouse() { shutdown(); }

void Lighthouse::shutdown() {
  {
    std::lock_guard<std::mutex> g(mu_);
    if (shutdown_) return;
    shutdown_ = true;
  }
  cv_.notify_all();
  if (tick_thread_.joinable()) tick_thread_.join();
  stop();
}

std::string Lighthouse::address() const { return "http://" + local_hostname() + ":" + std::to_string(port()); }

void Lighthouse::tick_loop() {
  std::unique_lock<std::mutex> lk(mu_);
  while (!shutdown_) {
    tick_locked();
    cv_.wait_for(lk, Millis(opt_.quorum_tick_ms), [this] { return shutdown_; });
  }
}

// Decide; when a quorum is valid: bump the id if membership changed or anyone
// reported commit failures, publish it to all waiters, and start a fresh round.
void Lighthouse::tick_locked() {
  QuorumDecision d = quorum_compute(monotonic_ms(), state_, opt_);
  if (d.reason != last_reason_) {  // change-only logging
    log_info("Quorum status: " + d.reason);
    last_reason_ = d.reason;
  }
  if (!d.participants.has_value()) return;
  std::vector<QuorumMember>& parts = *d.participants;
  bool commit_failures = false;
  for (const auto& p : parts) commit_failures = commit_failures || p.commit_failures > 0;
  if (!state_.prev_quorum.has_value() || quorum_changed(parts, state_.prev_quorum->participants)) {
    state_.quorum_id += 1;
    log_info("Detected quorum change, bumping quorum_id to " + std::to_string(state_.quorum_id));
  } else if (commit_failures) {
    state_.quorum_id += 1;
    log_info("Detected commit failures, bumping quorum_id to " + std::to_string(state_.quorum_id));
  }
  Quorum q;
  q.quorum_id = state_.quorum_id;
  q.participants = std::move(parts);
  q.created_ms = unix_ms();
  state_.prev_quorum = q;
  state_.participants.clear();
  Formed f;
  f.gen = ++gen_;
  {
    Writer w;
    q.encode(w);
    f.wire = std::make_shared<const std::string>(w.take());
  }
  for (const auto& p : q.participants) f.members.insert(p.replica_id);
  f.quorum = std::move(q);
  history_.push_back(std::move(f));
  while (history_.size() > 64) history_.pop_front();
  cv_.notify_all();
}

uint32_t Lighthouse::handle_rpc(uint32_t method, const std::string& req, TimePoint deadline, std::string* resp) {
  Reader r(req);
  if (method == kLighthouseHeartbeat) {
    std::string id = r.str();
    std::lock_guard<std::mutex> g(mu_);
    state_.heartbeats[id] = monotonic_ms();
    return kStatusOk;
  }
  if (method != kLighthouseQuorum) {
    *resp = "unknown lighthouse method";
    return kStatusInvalid;
  }
  QuorumMember requester = QuorumMember::decode(r);
  if (requester.replica_id.empty()) {
    *resp = "missing requester";
    return kStatusInvalid;
  }
  std::unique_lock<std::mutex> lk(mu_);
  const int64_t now = monotonic_ms();
  state_.heartbeats[requester.replica_id] = now;  // a quorum request is an implicit heartbeat
  state_.participants[requester.replica_id] = ParticipantDetails{now, requester};
  uint64_t seen = gen_;  // subscribe BEFORE the eager tick so its quorum is not missed
  // Eager tick (reference: every request ticks, lighthouse.rs:292-343) -- but only when this request can have completed a
  // quorum. Without the join timeout (which the periodic tick serves) a quorum needs every member of the previous quorum
  // (fast path) or every healthy replica among the participants, so fewer participants than both cannot decide anything.
  // quorum_compute sorts and formats over all replicas: running it for each of N simultaneous joiners made forming a
  // quorum O(N^2 log N) under the global lock; the counting pre-check below skips it for joiners that cannot decide.
  bool may_decide = true;
  {
    const size_t np = state_.participants.size();
    const size_t prev = state_.prev_quorum.has_value() ? state_.prev_quorum->participants.size() : (size_t)-1;
    if (np < prev) {
      size_t healthy = 0;
      for (const auto& hb : state_.heartbeats)
        if (now - hb.second < (int64_t)opt_.heartbeat_timeout_ms) ++healthy;
      may_decide = np >= healthy;
    }
  }
  if (may_decide) tick_locked();
  while (true) {
    // replay every quorum formed since we subscribed, oldest first
    for (const auto& f : history_) {
      if (f.gen <= seen) continue;
      seen = f.gen;
      if (f.members.count(requester.replica_id)) {
        std::shared_ptr<const std::string> wire = f.wire;
        lk.unlock();  // copy the (shared, immutable) encoding outside the lock
        *resp = *wire;
        return kStatusOk;
      }
      // formed without us (e.g. shrink_only round): rejoin the next round
      state_.participants[requester.replica_id] = ParticipantDetails{monotonic_ms(), requester};
    }
    if (shutdown_ || stopping()) {
      *resp = "lighthouse shutting down";
      return kStatusCancelled;
    }
    if (cv_.wait_until(lk, deadline) == std::cv_status::timeout && gen_ <= seen) {
      *resp = "lighthouse quorum timed out for replica " + requester.replica_id + ": " + last_reason_;
      return kStatusDeadline;
    }
  }
}

Quorum LighthouseClient::quorum(const QuorumMember& requester, Millis timeout) {
  Writer w;
  requester.encode(w);
  std::string resp = rpc_.call(kLighthouseQuorum, w.data(), timeout);
  Reader r(resp);
  return Quorum::decode(r);
}

void LighthouseClient::heartbeat(const std::string& replica_id, Millis timeout) {
  Writer w;
  w.str(replica_id);
  rpc_.call(kLighthouseHeartbeat, w.data(), timeout);
}

// ------------------------------------------------------------- dashboard
static std::string html_escape(const std::string& s) {
  std::string o;
  for (char c : s) {
    switch (c) {
      case '&': o += "&amp;"; break;
      case '<': o += "&lt;"; break;
      case '>': o += "&gt;"; break;
      case '"': o += "&quot;"; break;
      default: o += c;
    }
  }
  return o;
}

static const char* kIndexHtml = R"HTML(<!doctype html>
<html><head><meta charset="utf-8"><title>torchft_b200 lighthouse</title>
<style>
body{font-family:system-ui,sans-serif;margin:2em;background:#fafafa;color:#222}
h1{font-size:1.4em} .member{display:inline-block;border:1px solid #bbb;border-radius:6px;padding:.6em 1em;margin:.4em;background:#fff}
.recovering{background:#ffe0b3;border-color:#e69500} .old{color:#c00;font-weight:bold}
table{border-collapse:collapse} td,th{border:1px solid #ccc;padding:.3em .7em} button{cursor:pointer}
</style></head><body>
<h1>torchft_b200 Lighthouse</h1>
<div id="status">loading…</div>
<script>
async function refresh(){try{const r=await fetch('/status');document.getElementById('status').innerHTML=await r.text();}catch(e){}}
async function kill(id){if(!confirm('Kill replica '+id+'?'))return;await fetch('/replica/'+encodeURIComponent(id)+'/kill',{method:'POST'});refresh();}
refresh();setInterval(refresh,1000);
</script></body></html>)HTML";

std::string Lighthouse::status_html() {
  std::lock_guard<std::mutex> g(mu_);
  const int64_t now = monotonic_ms();
  QuorumDecision d = quorum_compute(now, state_, opt_);
  std::ostringstream os;
  int64_t max_step = -1, n = -1;
  if (state_.prev_quorum) {
    n = (int64_t)state_.prev_quorum->participants.size();
    for (const auto& p : state_.prev_quorum->participants) max_step = std::max(max_step, p.step);
  }
  os << "<h2>Quorum status</h2><p>Current quorum_id: " << state_.quorum_id << "</p><p>Next quorum status: "
     << html_escape(d.reason) << "</p>";
  os << "<h2>Previous quorum</h2>";
  if (state_.prev_quorum) {
    os << "<p>Previous quorum id: " << state_.prev_quorum->quorum_id << "<br>Num participants: " << n
       << "<br>Quorum age: " << (unix_ms() - state_.prev_quorum->created_ms) / 1000.0 << "s</p><div>";
    for (const auto& p : state_.prev_quorum->participants) {
      os << "<div class=\"member" << (p.step != max_step ? " recovering" : "") << "\"><b>" << html_escape(p.replica_id)
         << "</b><br>Step: " << p.step << "<br>Manager: " << html_escape(p.address)
         << "<br>TCPStore: " << html_escape(p.store_address) << "<br>World size: " << p.world_size
         << "<br><button onclick=\"kill('" << html_escape(p.replica_id) << "')\">Kill</button></div>";
    }
    os << "</div>";
  } else {
    os << "<p>None</p>";
  }
  os << "<h2>Heartbeats</h2><table><tr><th>replica</th><th>age (s)</th></tr>";
  for (const auto& [id, last] : state_.heartbeats) {
    const double age = (now - last) / 1000.0;
    os << "<tr><td>" << html_escape(id) << "</td><td" << ((now - last) >= (int64_t)opt_.heartbeat_timeout_ms ? " class=\"old\"" : "")
       << ">" << age << "</td></tr>";
  }
  os << "</table>";
  return os.str();
}

static std::string json_escape(const std::string& s) {
  std::string o;
  o.reserve(s.size() + 2);
  for (unsigned char c : s) {
    switch (c) {
      case '"': o += "\\\""; break;
      case '\\': o += "\\\\"; break;
      case '\n': o += "\\n"; break;
      case '\r': o += "\\r"; break;
      case '\t': o += "\\t"; break;
      default:
        if (c < 0x20) {
          char buf[8];
          std::snprintf(buf, sizeof(buf), "\\u%04x", c);
          o += buf;
        } else {
          o += (char)c;
        }
    }
  }
  return o;
}

// Machine-readable twin of the dashboard (GET /status.json): what monitoring and chaos tools poll.
std::string Lighthouse::status_json() {
  std::lock_guard<std::mutex> g(mu_);
  const int64_t now = monotonic_ms();
  QuorumDecision d = quorum_compute(now, state_, opt_);
  std::ostringstream os;
  os << "{\"quorum_id\": " << state_.quorum_id << ", \"next_quorum_status\": \"" << json_escape(d.reason)
     << "\", \"next_quorum_ready\": " << (d.participants.has_value() ? "true" : "false")
     << ", \"min_replicas\": " << opt_.min_replicas << ", \"heartbeat_timeout_ms\": " << opt_.heartbeat_timeout_ms
     << ", \"prev_quorum\": ";
  if (state_.prev_quorum) {
    int64_t max_step = -1;
    for (const auto& p : state_.prev_quorum->participants) max_step = std::max(max_step, p.step);
    os << "{\"quorum_id\": " << state_.prev_quorum->quorum_id << ", \"age_s\": "
       << (unix_ms() - state_.prev_quorum->created_ms) / 1000.0 << ", \"max_step\": " << max_step << ", \"participants\": [";
    bool first = true;
    for (const auto& p : state_.prev_quorum->participants) {
      os << (first ? "" : ", ") << "{\"replica_id\": \"" << json_escape(p.replica_id) << "\", \"address\": \""
         << json_escape(p.address) << "\", \"store_address\": \"" << json_escape(p.store_address) << "\", \"step\": " << p.step
         << ", \"world_size\": " << p.world_size << ", \"recovering\": " << (p.step != max_step ? "true" : "false")
         << ", \"commit_failures\": " << p.commit_failures << "}";
      first = false;
    }
    os << "]}";
  } else {
    os << "null";
  }
  os << ", \"waiting\": [";
  bool first = true;
  for (const auto& [id, det] : state_.participants) {
    os << (first ? "" : ", ") << "\"" << json_escape(id) << "\"";
    first = false;
  }
  os << "], \"heartbeats\": {";
  first = true;
  for (const auto& [id, last] : state_.heartbeats) {
    os << (first ? "" : ", ") << "\"" << json_escape(id) << "\": {\"age_s\": " << (now - last) / 1000.0 << ", \"alive\": "
       << ((now - last) < (int64_t)opt_.heartbeat_timeout_ms ? "true" : "false") << "}";
    first = false;
  }
  os << "}}";
  return os.str();
}

HttpResponse Lighthouse::kill_replica(const std::string& replica_id) {
  std::string addr;
  {
    std::lock_guard<std::mutex> g(mu_);
    if (state_.prev_quorum)
      for (const auto& p : state_.prev_quorum->participants)
        if (p.replica_id == replica_id) addr = p.address;
  }
  if (addr.empty()) return {500, "text/plain", "Something went wrong: failed to find replica"};
  try {
    ManagerClient c(addr, Millis(10000));
    c.kill("killed from dashboard");
  } catch (const std::exception& e) {
    // the target exits before answering; a dropped connection is the expected outcome
  }
  return {200, "text/plain", "ok"};
}

static std::string url_decode(const std::string& s) {
  std::string o;
  for (size_t i = 0; i < s.size(); ++i) {
    if (s[i] == '%' && i + 2 < s.size()) {
      o += (char)std::stoi(s.substr(i + 1, 2), nullptr, 16);
      i += 2;
    } else {
      o += s[i];
    }
  }
  return o;
}

HttpResponse Lighthouse::handle_http(const HttpRequest& req) {
  if (req.method == "GET" && (req.path == "/" || req.path == "/index.html")) return {200, "text/html; charset=utf-8", kIndexHtml};
  if (req.method == "GET" && req.path == "/status") return {200, "text/html; charset=utf-8", status_html()};
  if (req.method == "GET" && req.path == "/status.json") return {200, "application/json", status_json()};
  const std::string pre = "/replica/", suf = "/kill";
  if (req.method == "POST" && req.path.rfind(pre, 0) == 0 && req.path.size() > pre.size() + suf.size() &&
      req.path.compare(req.path.size() - suf.size(), suf.size(), suf) == 0) {
    return kill_replica(url_decode(req.path.substr(pre.size(), req.path.size() - pre.size() - suf.size())));
  }
  return {404, "text/plain", "not found"};
}

}  // namespace tft
