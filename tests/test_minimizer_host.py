"""The three minimizer scans of chromap_b200/csrc/minimizers.cuh (run-time body, static-ring body, packed-key body used by the
tier-0 front end) compiled for the HOST and compared with each other on random, low-complexity, tandem-repeat and N-bearing
reads.  (The run-time body is compared with the oracle on the GPU by the stage tests; this keeps the fast paths honest on
machines without one.)"""
from tests import emu

MAIN = r'''
int main(){
  srand(5); long bad=0, tot=0, ties=0;
  // Hash64 on 32-bit halves == the 64-bit formulation
  { u64 x=88172645463325252ull; for(long i=0;i<3000000;i++){ x^=x<<13; x^=x>>7; x^=x<<17; const u64 m=(1ull<<34)-1; if(mix64(x&m,m)!=mix64_k<17>(x&m)) bad++; } }
  for(int it=0; it<120000; ++it){
    int len = 20 + rand()%140;
    std::string r(len,'A');
    int mode = rand()%10;
    for(int i=0;i<len;i++){
      if(mode<5) r[i]="ACGT"[rand()%4];
      else if(mode<7) r[i]="ACGT"[(i/(1+rand()%3))%4];
      else if(mode<8) r[i]= (rand()%20==0)?'N':"ACGT"[rand()%4];
      else if(mode<9) r[i]="AC"[rand()%2];
      else { int per=1+it%6; r[i]="ACGT"[(i%per)%4]; }
    }
    if(mode==7 && rand()%2) for(int i=0;i<len;i++) if(rand()%3==0) r[i]=tolower(r[i]);
    std::vector<std::pair<u64,u32>> A,B,C;
    minimizer_scan<0,0>([&](int i){return (u8)r[i];}, len, 17, 7, [&](u64 h,u32 p){A.push_back({h,p});});
    minimizer_scan_packed<17,7>([&](int i){return (u8)r[i];}, len, [&](u64 h,u32 p){B.push_back({h,p});});
    minimizer_scan<17,7>([&](int i){return (u8)r[i];}, len, 17, 7, [&](u64 h,u32 p){C.push_back({h,p});});
    tot++;
    if(A!=B || A!=C) bad++;
    for(size_t i=1;i<A.size();i++) if(A[i].first==A[i-1].first) {ties++; break;}
  }
  printf("reads=%ld bad=%ld ties=%ld\n",tot,bad,ties); return bad!=0;
}
'''


def test_minimizer_scans_agree_on_the_host(tmp_path):
    out = emu.run(tmp_path, ["device_common.cuh", "minimizers.cuh"], MAIN)
    assert out.returncode == 0, out.stdout
    assert "bad=0" in out.stdout and "ties=0" not in out.stdout, out.stdout
